"""pytorch_volumetric_b200 -- H100-native (sm_90a) drop-in for pytorch_volumetric's batched SDF query path.

The public names of the reference package (`pytorch_volumetric/__init__.py`) that belong to that path are
re-exported here, so `import pytorch_volumetric_b200 as pv` reads like the original.
"""
from . import chamfer as _chamfer, distributed, kinematics as _kin, model_to_sdf as _robot, sdf as _sdf, \
    transforms as _tf, voxel as _voxel

_EXPORTS = {
    _sdf: ("BoxSDF", "CachedSDF", "ComposedSDF", "CylinderSDF", "MeshObjectFactory", "MeshSDF", "ObjectFactory",
           "ObjectFrameSDF", "OccupancyMap", "OccupancySDF", "OutOfBoundsStrategy", "SDFQuery", "SphereSDF", "depth_occupancy",
           "depth_to_points", "occupancy_distance_transform", "ray_occupancy", "sample_mesh_points"),
    _robot: ("RobotSDF", "aabb_to_ordered_end_points", "cache_link_sdf_factory"),
    _chamfer: ("PlausibleDiversity", "batch_chamfer_dist", "pairwise_distance", "pairwise_distance_chamfer"),
    _voxel: ("ExpandingVoxelGrid", "VoxelGrid", "VoxelSet", "Voxels", "get_coordinates_and_points_in_grid",
             "get_divisible_range_by_resolution", "voxel_down_sample"),
    _tf: ("Transform3d", "Translate"),
    _kin: ("Chain", "SerialChain", "build_chain_from_urdf", "build_serial_chain_from_urdf"),
}
for _module, _names in _EXPORTS.items():
    for _name in _names:
        globals()[_name] = getattr(_module, _name)

__all__ = sorted(n for names in _EXPORTS.values() for n in names) + ["distributed"]
del _module, _names, _name
