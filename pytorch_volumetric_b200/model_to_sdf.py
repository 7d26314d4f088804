"""RobotSDF: one SDF per link mesh, posed by batched forward kinematics, min over links in one fused kernel.

API mirror of the reference's src/pytorch_volumetric/model_to_sdf.py (RobotSDF :12-125,
cache_link_sdf_factory :128-133, aabb_to_ordered_end_points :136-171): same constructor arguments, attributes,
output shapes and state semantics.  `chain` is duck-typed on the pytorch_kinematics Chain surface listed in
kinematics.py; every query is a single pvb_composed_query launch.
"""
import logging
import typing

import numpy as np
import torch

from . import sdf
from .transforms import Transform3d, invert_rigid, matrix_of

logger = logging.getLogger(__file__)


def _mesh_visuals(chain, frame_names):
    """(link name, visual) for every mesh visual along the chain, in frame order; other geometry types are
    reported and skipped, like the reference does (model_to_sdf.py:41-56)."""
    for fname in frame_names:
        link = chain.find_frame(fname).link
        for vis in link.visuals:
            if vis.geom_type == "mesh":
                yield link.name, vis
            else:
                logger.warning("Cannot handle non-mesh link visual type %s for %s", vis, link.name)


class RobotSDF(sdf.ObjectFrameSDF):
    """SDF of an articulated robot in its base frame.

    The joint configuration -- a single vector or an arbitrarily batched set of them -- is state: it is installed
    with `set_joint_configuration` and determines both the values and the leading shape of what `__call__` returns.
    """

    def __init__(self, chain, default_joint_config=None, path_prefix='',
                 link_sdf_cls: typing.Callable[[sdf.ObjectFactory], sdf.ObjectFrameSDF] = sdf.MeshSDF):
        """
        :param chain: kinematic description; only mesh visuals become SDFs
        :param default_joint_config: joint values installed at construction (zeros when None)
        :param path_prefix: directory the relative mesh paths of the description are resolved against
        :param link_sdf_cls: callable turning a link's ObjectFactory into its ObjectFrameSDF
        """
        self.chain = chain
        self.dtype, self.device = chain.dtype, chain.device
        self.q = None
        self.configuration_batch = None
        self.object_to_link_frames = None
        self.joint_names = chain.get_joint_parameter_names()
        self.frame_names = chain.get_frame_names(exclude_fixed=False)

        visuals = list(_mesh_visuals(chain, self.frame_names))
        self.sdf_to_link_name = [name for name, _ in visuals]
        link_sdfs = []
        for name, vis in visuals:
            mesh_file, mesh_scale = vis.geom_param[0], vis.geom_param[1]
            logger.info("%s offset %s", name, vis.offset)
            link_sdfs.append(link_sdf_cls(sdf.MeshObjectFactory(mesh_file, scale=mesh_scale, path_prefix=path_prefix)))
        # visual origin of every mesh inside its link frame, stacked link-major
        self.offset_transforms = Transform3d(
            matrix=torch.cat([matrix_of(vis.offset) for _, vis in visuals]).to(device=self.device, dtype=self.dtype))
        # inverse of the visual offsets, once (general inverse: a scaled <visual><origin> is not rigid)
        self._mesh_from_link = self.offset_transforms.inverse().get_matrix()
        self.sdf: typing.Optional[sdf.ComposedSDF] = sdf.ComposedSDF(link_sdfs, None)
        self._fk_plan = self._make_fk_plan()
        self.set_joint_configuration(default_joint_config)

    #: set False to force the eager forward_kinematics of the chain object (what foreign pk chains always get)
    native_fk = True

    def _make_fk_plan(self):
        """(pvb_fk_frame[], pvb_fk_link[]) for pvb_fk_serial when the chain is this package's SerialChain in
        float32 on a CUDA device; None otherwise (duck-typed pytorch_kinematics chains keep their own FK)."""
        from . import _native as nat
        from .kinematics import SerialChain
        if not isinstance(self.chain, SerialChain) or self.dtype != torch.float32 or \
                torch.device(self.device).type != "cuda" or not (1 <= len(self.sdf_to_link_name) <= nat.FK_MAX_LINKS):
            return None
        frames = self.chain.native_fk_frames()
        if frames is None:
            return None
        frame_of = {f.link.name: i for i, f in enumerate(self.chain._frames)}
        inv = self._mesh_from_link.detach().to("cpu", torch.float32)
        if not bool((inv[:, 3] == torch.tensor([0.0, 0.0, 0.0, 1.0])).all()):
            return None                       # a projective visual offset: not an [A | t] matrix
        order = sorted(range(len(self.sdf_to_link_name)), key=lambda s: frame_of[self.sdf_to_link_name[s]])
        links = (nat.FkLink * len(order))()
        for k, s_idx in enumerate(order):
            for r in range(3):
                for c in range(4):
                    links[k].mesh_from_link[4 * r + c] = float(inv[s_idx, r, c])
            links[k].frame = frame_of[self.sdf_to_link_name[s_idx]]
            links[k].slot = s_idx
        return frames, links

    # ------------------------------------------------------------------ state
    def set_joint_configuration(self, joint_config=None):
        """Install joint values of shape [*A, n_joints]; A (possibly empty) becomes the leading shape of results."""
        n_joints = len(self.joint_names)
        if joint_config is None:
            joint_config = torch.zeros(n_joints, device=self.device, dtype=self.dtype)
        batched = joint_config.dim() > 1
        self.configuration_batch = tuple(joint_config.shape[:-1]) if batched else None
        if self.configuration_batch is not None:
            self.configuration_batch = torch.Size(self.configuration_batch)
        flat_q = joint_config.reshape(-1, n_joints) if batched else joint_config
        self.q = flat_q
        if self.native_fk and self._fk_plan is not None:
            # one kernel: FK along the chain + (FK @ visual_offset)^-1 per mesh link, written link-major
            from . import _native as nat
            import ctypes
            frames, links = self._fk_plan
            dev = nat.compute_device(self.device)
            with torch.cuda.device(dev):
                qd = flat_q.detach().reshape(-1, n_joints).to(device=dev, dtype=torch.float32).contiguous()
                n_cfg = qd.shape[0]
                out = torch.empty(len(links) * n_cfg, 4, 4, dtype=torch.float32, device=dev)
                nat.check(nat.lib().pvb_fk_serial(ctypes.cast(frames, ctypes.c_void_p), len(frames),
                                                  ctypes.cast(links, ctypes.c_void_p), len(links), nat.ptr(qd), n_cfg,
                                                  n_joints, nat.ptr(out), nat.stream_ptr(dev)), "pvb_fk_serial")
            self.object_to_link_frames = Transform3d(matrix=out)
            if self.sdf is not None:
                self.sdf.set_transforms(self.object_to_link_frames, batch_dim=self.configuration_batch)
            return
        poses = self.chain.forward_kinematics(flat_q, end_only=False)
        world_from_link = torch.stack([matrix_of(poses[name]) for name in self.sdf_to_link_name])   # (S, |A|, 4, 4)
        n_links, n_cfg = world_from_link.shape[:2]
        mesh_from_link = self._mesh_from_link.to(world_from_link)                                   # (S, 4, 4)
        # base frame -> mesh frame of each link: (FK @ visual_offset)^-1, link-major like the reference's stack
        mesh_from_world = mesh_from_link[:, None] @ invert_rigid(world_from_link)
        self.object_to_link_frames = Transform3d(matrix=mesh_from_world.reshape(n_links * n_cfg, 4, 4))
        if self.sdf is not None:
            self.sdf.set_transforms(self.object_to_link_frames, batch_dim=self.configuration_batch)

    # ---------------------------------------------------------------- queries
    def __call__(self, points_in_object_frame):
        """points [*B, N, 3] in the robot frame -> (values [*A, *B, N], gradients [*A, *B, N, 3])."""
        return self.sdf(points_in_object_frame)

    def surface_bounding_box(self, **kwargs):
        return self.sdf.surface_bounding_box(**kwargs)

    def link_bounding_boxes(self):
        """Corner points (8 x 3, robot frame) of every link's box under the installed configuration(s)."""
        world_from_mesh = Transform3d(matrix=sdf._affine_inverse(matrix_of(self.sdf.obj_frame_to_link_frame)))
        per_link = []
        for i, link_sdf in enumerate(self.sdf.sdfs):
            corners = aabb_to_ordered_end_points(np.asarray(link_sdf.surface_bounding_box(padding=0)))
            corners = torch.tensor(corners, device=world_from_mesh.device, dtype=world_from_mesh.dtype)
            per_link.append(world_from_mesh.transform_points(corners)[self.sdf.ith_transform_slice(i)])
        return torch.stack(per_link).squeeze()


class _CachedLinkFactory:
    """Picklable callable behind `cache_link_sdf_factory`."""

    def __init__(self, resolution, padding, kwargs):
        self.resolution, self.padding, self.kwargs = resolution, padding, kwargs

    def __call__(self, obj_factory: sdf.ObjectFactory):
        box = obj_factory.bounding_box(padding=self.padding)
        return sdf.CachedSDF(obj_factory.name, self.resolution, box, sdf.MeshSDF(obj_factory), **self.kwargs)


def cache_link_sdf_factory(resolution=0.01, padding=0.1, **kwargs):
    """`link_sdf_cls` that wraps every link mesh in a CachedSDF over its padded bounding box."""
    return _CachedLinkFactory(resolution, padding, kwargs)


def aabb_to_ordered_end_points(aabb, arrange_in_sequential_order=False):
    """8 corners of a (3,2) box, or (sequential order) a 16-point closed walk over its edges for line drawing."""
    lo, hi = aabb[:, 0], aabb[:, 1]
    if arrange_in_sequential_order:
        code = ["000", "100", "110", "010", "000", "001", "101", "100", "101", "111", "110", "111", "011", "010",
                "011", "001"]
    else:
        code = ["000", "100", "010", "001", "011", "101", "110", "111"]
    arr = [[(hi if c[k] == "1" else lo)[k] for k in range(3)] for c in code]
    if torch.is_tensor(aabb):
        return torch.tensor(arr, device=aabb.device, dtype=aabb.dtype)
    return np.array(arr)
