"""Signed-distance objects with the reference's Python API, computed by libpvb.so on H100.

Mirrors the reference's src/pytorch_volumetric/sdf.py (same class names, constructor
arguments, shapes, dtypes and exceptions) for the batched query path:

  ObjectFactory / MeshObjectFactory   sdf.py:30-214   mesh load, AABB, closest point + sign
  ObjectFrameSDF                      sdf.py:217-282  the operator interface
  SphereSDF                           sdf.py:285-299
  MeshSDF                             sdf.py:302-329
  ComposedSDF                         sdf.py:332-433
  OutOfBoundsStrategy, CachedSDF      sdf.py:436-614
  sample_mesh_points                  sdf.py:617-670

All arithmetic on the query path runs in hand-written sm_90a kernels behind the
C ABI of include/pvb.h; there is no CPU fallback.  Host tensors are accepted
(copied to the GPU, results copied back to the input's device) so that the
classes drop in for CPU callers of the reference.
"""
import abc
import ctypes
import enum
import logging
import math
import os
import typing
from functools import partial
from typing import NamedTuple, Union

import numpy as np
import torch

from . import _native as nat
from . import meshio
from .transforms import Transform3d, invert_rigid, matrix_of
from .voxel import (GridView, VoxelGrid, get_coordinates_and_points_in_grid, get_divisible_range_by_resolution,
                    nonempty_indices, range_dtype)

logger = logging.getLogger(__name__)


class SDFQuery(NamedTuple):
    closest: torch.Tensor
    distance: torch.Tensor
    gradient: torch.Tensor
    normal: Union[torch.Tensor, None]


class TriMesh:
    """fp64 vertices + int32 triangles (+ unit face normals): what `ObjectFactory._mesh` holds."""

    def __init__(self, vertices, triangles):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.triangles = np.ascontiguousarray(triangles, dtype=np.int32).reshape(-1, 3)
        self.triangle_normals = None

    def compute_triangle_normals(self):
        v, f = self.vertices, self.triangles
        n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        with np.errstate(invalid="ignore", divide="ignore"):
            n = n / np.linalg.norm(n, axis=1, keepdims=True)
        n[~np.isfinite(n).all(axis=1)] = (0.0, 0.0, 1.0)
        self.triangle_normals = n
        return self

    def triangle_areas(self):
        v, f = self.vertices, self.triangles
        return 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1)

    def get_center(self):
        return self.vertices.mean(axis=0)


def _as_trimesh(mesh):
    if isinstance(mesh, TriMesh):
        return mesh
    if isinstance(mesh, (tuple, list)) and len(mesh) == 2:
        return TriMesh(mesh[0], mesh[1])
    if hasattr(mesh, "vertices") and hasattr(mesh, "triangles"):     # e.g. an open3d legacy TriangleMesh
        return TriMesh(np.asarray(mesh.vertices), np.asarray(mesh.triangles))
    raise TypeError("mesh= expects (vertices, faces) or an object with .vertices and .triangles")


def _winding_moments(nodes_u8, tris):
    """Per BVH4 node and child: area-weighted centroid + bounding radius and the sum of area vectors -- the
    first-order data of the hierarchical winding-number evaluation (EXTENSION, see pvb.h PVB_MESH_WINDING).
    nodes_u8 (n,128) uint8 and tris (F,12) float32 are the arrays pvb_bvh_build returned.  -> float32 (n, 8, 4)."""
    n = nodes_u8.shape[0]
    nf = nodes_u8.view(np.float32).reshape(n, 32).astype(np.float64)
    child = nodes_u8.view(np.int32).reshape(n, 32)[:, 24:28].astype(np.int64)
    lo = np.stack([nf[:, 0:4], nf[:, 4:8], nf[:, 8:12]], axis=-1)          # (n, 4, 3)
    hi = np.stack([nf[:, 12:16], nf[:, 16:20], nf[:, 20:24]], axis=-1)
    t = tris.astype(np.float64)
    v0, v1, v2 = t[:, 0:3], t[:, 4:7], t[:, 8:11]
    avec = 0.5 * np.cross(v1 - v0, v2 - v0)                                # area vectors
    area = np.linalg.norm(avec, axis=1)
    acen = area[:, None] * (v0 + v1 + v2) / 3.0
    cs = lambda a: np.concatenate([np.zeros((1,) + a.shape[1:]), np.cumsum(a, axis=0)])   # prefix sums, leaf order
    cs_vec, cs_area, cs_cen = cs(avec), cs(area), cs(acen)
    empty = child == -2 ** 31
    leaf = (child < 0) & ~empty
    inner = child >= 0
    code = np.where(leaf, ~child, 0)
    first, cnt = code >> 2, (code & 3) + 1
    N = np.zeros((n, 4, 3)); A = np.zeros((n, 4)); C = np.zeros((n, 4, 3))
    N[leaf] = (cs_vec[(first + cnt)[leaf]] - cs_vec[first[leaf]])
    A[leaf] = (cs_area[(first + cnt)[leaf]] - cs_area[first[leaf]])
    C[leaf] = (cs_cen[(first + cnt)[leaf]] - cs_cen[first[leaf]])
    # inner children: totals of the child node; children have larger indices (BFS layout), so sweep by depth
    depth = np.zeros(n, dtype=np.int64)
    for i in range(n):                       # parents precede children
        ch = child[i][inner[i]]
        depth[ch] = depth[i] + 1
    for dlev in range(int(depth.max()), -1, -1):
        idx = np.nonzero(depth == dlev)[0]
        if dlev < depth.max():
            sel = inner[idx]
            ii, kk = np.nonzero(sel)
            cidx = child[idx[ii], kk]
            N[idx[ii], kk] = N[cidx].sum(axis=1)
            A[idx[ii], kk] = A[cidx].sum(axis=1)
            C[idx[ii], kk] = C[cidx].sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        cen = C / A[..., None]
    with np.errstate(invalid="ignore"):
        box_c = 0.5 * (lo + hi)
    bad = ~np.isfinite(cen).all(axis=-1) | (A <= 0)
    cen[bad] = np.where(np.isfinite(box_c[bad]), box_c[bad], 0.0)
    with np.errstate(invalid="ignore"):
        rad = np.linalg.norm(np.maximum(np.abs(cen - lo), np.abs(hi - cen)), axis=-1)
    rad[empty] = 0.0
    out = np.zeros((n, 8, 4), dtype=np.float32)
    out[:, 0:4, 0:3] = np.where(empty[..., None], 0.0, cen)
    out[:, 0:4, 3] = np.where(np.isfinite(rad), rad, 0.0)
    out[:, 4:8, 0:3] = np.where(empty[..., None], 0.0, N)
    return out


class _HostChunkStream:
    """Host batch in, pinned host results out, PCIe busy in both directions at once: chunk i is copied in on `s_in`
    while chunk i-1 is computed on the current stream and chunk i-2 is copied out on `s_out`; two device slots per
    direction, events order the reuse of a slot.  `tails` are the trailing shapes of the per-point outputs, e.g.
    ((), (3,)) for value + gradient; `launch(d_in, m, d_outs)` enqueues the computation of one chunk of m points on
    the current stream.

    (Chunks of a few million points: much smaller ones are dominated by per-chunk stream/event bookkeeping.)"""

    def __init__(self, device, chunk, tails):
        self.device, self.chunk, self.tails = device, chunk, tuple(tails)
        with torch.cuda.device(device):
            self.s_in, self.s_out = torch.cuda.Stream(device), torch.cuda.Stream(device)
            self.d_in = [torch.empty(chunk, 3, dtype=torch.float32, device=device) for _ in range(2)]
            self.d_out = [[torch.empty(chunk, *t, dtype=torch.float32, device=device) for t in self.tails]
                          for _ in range(2)]

    def run(self, points, launch):
        device, C = self.device, self.chunk
        src = points.detach().reshape(-1, 3)
        if src.dtype != torch.float32:
            src = src.float()
        src = src.contiguous()
        n = src.shape[0]
        with torch.cuda.device(device):
            cur = torch.cuda.current_stream(device)
            outs_h = [torch.empty(n, *t, dtype=torch.float32, pin_memory=True) for t in self.tails]
            self.s_in.wait_stream(cur)
            self.s_out.wait_stream(cur)
            ev_comp = [None, None]      # computation finished reading d_in[b] / writing d_out[b]
            ev_out = [None, None]       # copy-out finished reading d_out[b]
            for i, lo in enumerate(range(0, n, C)):
                hi = min(lo + C, n)
                m = hi - lo
                b = i & 1
                with torch.cuda.stream(self.s_in):
                    if ev_comp[b] is not None:
                        self.s_in.wait_event(ev_comp[b])
                    self.d_in[b][:m].copy_(src[lo:hi], non_blocking=True)
                    ev_in = torch.cuda.Event()
                    ev_in.record(self.s_in)
                cur.wait_event(ev_in)
                if ev_out[b] is not None:
                    cur.wait_event(ev_out[b])
                launch(self.d_in[b], m, self.d_out[b])
                ev_comp[b] = torch.cuda.Event()
                ev_comp[b].record(cur)
                with torch.cuda.stream(self.s_out):
                    self.s_out.wait_event(ev_comp[b])
                    for h, d in zip(outs_h, self.d_out[b]):
                        h[lo:hi].copy_(d[:m], non_blocking=True)
                    ev_out[b] = torch.cuda.Event()
                    ev_out[b].record(self.s_out)
            self.s_out.synchronize()
            cur.wait_stream(self.s_in)
        return outs_h


class ObjectFactory(abc.ABC):
    def __init__(self, name='', scale=1.0, vis_frame_pos=(0, 0, 0), vis_frame_rot=(0, 0, 0, 1),
                 plausible_suboptimality=0.001, mesh=None, ray_seed=0, **kwargs):
        """
        :param name: path to the mesh obj if loading from file
        :param scale: scaling factor for the mesh
        :param vis_frame_pos: position of the mesh in the object frame
        :param vis_frame_rot: quaternion rotation (xyzw) of the mesh in the object frame
        :param plausible_suboptimality: how much error to tolerate in the SDF
        :param mesh: (vertices, faces) or an object with .vertices/.triangles, given instead of a path;
        scale, vis_frame_pos and vis_frame_rot are then ignored (as in the reference)
        :param ray_seed: seed of the deterministic per-point jitter of the inside/outside ray direction
        (the reference draws it from the unseeded numpy global generator, sdf.py:149)
        """
        self.name = name
        self.scale = scale if scale is not None else 1.0
        self.vis_frame_pos = vis_frame_pos
        self.vis_frame_rot = vis_frame_rot
        self.other_load_kwargs = kwargs
        self.plausible_suboptimality = plausible_suboptimality
        self.ray_seed = int(ray_seed)

        self._mesh = _as_trimesh(mesh) if mesh is not None else None
        self._mesh_given = mesh is not None
        self._face_normals = None
        self._bvh_host = None      # (nodes uint8[n,128], tris float32[F,12], depth)
        self._dev = {}             # device -> dict of device buffers
        self._closed = None
        self._aabb = None
        self.precompute_sdf()

    def __reduce__(self):
        if self._mesh_given:
            return partial(self.__class__, scale=self.scale, vis_frame_pos=self.vis_frame_pos,
                           vis_frame_rot=self.vis_frame_rot, plausible_suboptimality=self.plausible_suboptimality,
                           mesh=(self._mesh.vertices, self._mesh.triangles), **self.other_load_kwargs), (self.name,)
        return partial(self.__class__, scale=self.scale, vis_frame_pos=self.vis_frame_pos,
                       vis_frame_rot=self.vis_frame_rot,
                       plausible_suboptimality=self.plausible_suboptimality, **self.other_load_kwargs), \
            (self.name,)

    @abc.abstractmethod
    def make_collision_obj(self, z, rgba=None):
        """Create collision object of fixed and position along x-y; returns the object ID and bounding box"""

    @abc.abstractmethod
    def get_mesh_resource_filename(self):
        """Return the path to the mesh resource file (.obj, .stl, ...)"""

    def get_mesh_high_poly_resource_filename(self):
        return self.get_mesh_resource_filename()

    def bounding_box(self, padding=0., padding_ratio=0):
        if self._aabb is None:      # the vertices never change after construction
            self._aabb = (self._mesh.vertices.min(axis=0), self._mesh.vertices.max(axis=0))
        ranges = np.stack(self._aabb, axis=1)
        extents = ranges[:, 1] - ranges[:, 0]
        ranges[:, 0] -= padding + padding_ratio * extents
        ranges[:, 1] += padding + padding_ratio * extents
        return ranges

    def center(self):
        if self._mesh is None:
            self.precompute_sdf()
        return self._mesh.get_center()

    @property
    def is_closed(self):
        if self._closed is None:
            self._closed = meshio.is_closed_manifold(self._mesh.triangles)
        return self._closed

    def precompute_sdf(self):
        if self._mesh is None:
            full_path = os.path.expanduser(self.get_mesh_high_poly_resource_filename())
            if not os.path.exists(full_path):
                raise RuntimeError(f"Expected mesh file does not exist: {full_path}")
            v, f = meshio.read_triangle_mesh(full_path)
            v = v * np.asarray(self.scale, dtype=np.float64)                       # sdf.py:105-107
            v = v @ meshio.quaternion_xyzw_to_matrix(self.vis_frame_rot).T         # sdf.py:110-112
            v = v + np.array(self.vis_frame_pos, dtype=np.float64) * self.scale    # sdf.py:113
            self._mesh = TriMesh(v, f)
        if self._bvh_host is None:
            self._mesh.compute_triangle_normals()
            self._face_normals = self._mesh.triangle_normals                       # fp64, sdf.py:119-120
            # the query structure holds fp32 vertices, like the Embree scene built from the
            # float32 tensor mesh at sdf.py:116-118
            self._bvh_host = nat.bvh_build(self._mesh.vertices.astype(np.float32), self._mesh.triangles)

    # -- device residency -------------------------------------------------------
    def _device_state(self, device):
        device = nat.compute_device(device)
        st = self._dev.get(device)
        if st is None:
            nodes, tris, depth = self._bvh_host
            if 3 * depth + 2 > 64:
                raise nat.NativeLibraryError(f"BVH too deep for the traversal stack (depth {depth})")
            st = {
                "nodes": torch.from_numpy(nodes).to(device),
                "tris": torch.from_numpy(tris).to(device),
                "fn32": torch.from_numpy(self._face_normals.astype(np.float32)).contiguous().to(device),
                "v64": torch.from_numpy(self._mesh.vertices).to(device),
                "faces": torch.from_numpy(self._mesh.triangles).to(device),
            }
            self._dev[device] = st
        return st

    def native_desc(self, device):
        """pvb_sdf_desc (kind MESH) for this object on `device`."""
        st = self._device_state(device)
        d = nat.SdfDesc()
        d.kind = nat.PVB_KIND_MESH
        d.flags = 0
        self._fill_mesh_part(d, st)
        return d

    def _winding_state(self, device):
        st = self._device_state(device)
        if "wn" not in st:
            nodes, tris, _ = self._bvh_host
            st["wn"] = torch.from_numpy(_winding_moments(nodes, tris)).to(st["nodes"].device)
        return st["wn"]

    #: set False to force the reference's diagonal ray (sdf.py:147-153) even on closed meshes
    axis_ray_when_closed = True
    #: "parity" (the reference's rule: odd number of ray crossings => inside) or "winding" -- an EXTENSION that
    #: classifies by the generalized winding number |w| > 1/2, robust on open / self-intersecting meshes
    sign_mode = "parity"

    def _fill_mesh_part(self, d, st):
        d.nodes = st["nodes"].data_ptr()
        d.n_nodes = st["nodes"].shape[0]
        d.tris = st["tris"].data_ptr()
        d.n_tris = st["tris"].shape[0]
        d.face_normals = st["fn32"].data_ptr()
        far = self.bounding_box(padding=1.0)[:, 1]                                  # sdf.py:147
        bb = self.bounding_box()
        for k in range(3):
            d.ray_far[k] = float(np.float32(far[k]))
            d.bb_min[k] = float(np.float32(bb[k, 0]))
            d.bb_max[k] = float(np.float32(bb[k, 1]))
        d.ray_seed = self.ray_seed & 0xFFFFFFFF
        if self.axis_ray_when_closed and self.is_closed:
            d.flags |= nat.PVB_MESH_CLOSED
        # slack of the "value >= distance to the AABB" bound used by the composed kernels (fp32 rounding only)
        d.prune_margin = 1e-5 * max(1.0, float(np.abs(bb).max()))

    # -- the query (sdf.py:122-172) ----------------------------------------------
    #: host batches at least this large are streamed through the GPU in chunks (_HostChunkStream); every chunk is
    #: binned and walked on its own
    host_pipeline_min_points = 1 << 22
    host_pipeline_chunk = 1 << 21

    def _do_object_frame_closest_point(self, points_in_object_frame, compute_normal=False, device=None,
                                       mode=nat.PVB_MESH_DEFAULT, want_closest=True):
        """-> (closest | None, distance, gradient, normal | None); want_closest=False (MeshSDF.__call__ needs distance
        and gradient only) skips the closest-point output and its copy to the host."""
        if torch.is_tensor(points_in_object_frame):
            dtype = points_in_object_frame.dtype
            out_device = points_in_object_frame.device
            if device is None and out_device.type == "cuda":
                device = out_device
        else:
            points_in_object_frame = np.asarray(points_in_object_frame)
            dtype = torch.float
            out_device = torch.device("cpu")
        lead = tuple(points_in_object_frame.shape[:-1])
        device = nat.compute_device(device)
        if self.sign_mode not in ("parity", "winding"):
            raise ValueError(f"sign_mode must be 'parity' or 'winding', got {self.sign_mode!r}")
        winding = self.sign_mode == "winding" and bool(mode & nat.PVB_MESH_SIGNED)
        L = nat.lib()
        if (torch.is_tensor(points_in_object_frame) and out_device.type == "cpu" and dtype == torch.float32
                and not winding and points_in_object_frame.shape[-1] == 3
                and points_in_object_frame.numel() // 3 >= self.host_pipeline_min_points
                and (self.axis_ray_when_closed and self.is_closed or not (mode & nat.PVB_MESH_SIGNED))):
            # large host batch: copy-in / tree walk / copy-out overlapped chunk by chunk.  (Only where the sign test is
            # the exact axis-aligned walk: the jittered diagonal ray of open meshes is seeded by the point's index in
            # the call, so chunking would change which ray a point gets.)
            tails = ((3,),) * bool(want_closest) + ((), (3,)) + ((3,),) * bool(compute_normal)
            key = (device, self.host_pipeline_chunk, tails)
            st = getattr(self, "_pipe_state", None)
            if st is None or st[0] != key:
                with torch.cuda.device(device):
                    st = self._pipe_state = (key, _HostChunkStream(device, self.host_pipeline_chunk, tails),
                                             nat.query_workspace(self.host_pipeline_chunk, device))
            desc = self.native_desc(device)
            ws = st[2]

            def launch(d_in, m, d_out):
                o = list(d_out)
                closest = o.pop(0) if want_closest else None
                dist, grad = o.pop(0), o.pop(0)
                normal = o.pop(0) if compute_normal else None
                nat.check(L.pvb_mesh_query(ctypes.byref(desc), nat.ptr(d_in), m, mode, nat.ptr(dist), nat.ptr(grad),
                                           nat.ptr(closest), None, nat.ptr(normal), nat.ptr(ws),
                                           ws.numel() if ws is not None else 0, nat.stream_ptr(device)),
                          "pvb_mesh_query")

            o = list(st[1].run(points_in_object_frame, launch))
            closest = o.pop(0).reshape(*lead, 3) if want_closest else None
            dist, grad = o.pop(0).reshape(lead), o.pop(0).reshape(*lead, 3)
            normal = o.pop(0).reshape(*lead, 3) if compute_normal else None
            return closest, dist, grad, normal
        with torch.cuda.device(device):
            p = nat.as_f32_points(points_in_object_frame, device)
            n = p.shape[0]
            dist = torch.empty(n, dtype=torch.float32, device=device)
            grad = torch.empty(n, 3, dtype=torch.float32, device=device)
            closest = torch.empty(n, 3, dtype=torch.float32, device=device) if want_closest else None
            normal = torch.empty(n, 3, dtype=torch.float32, device=device) if compute_normal else None
            desc = self.native_desc(device)
            face = None
            if winding:
                mode |= nat.PVB_MESH_WINDING
                desc.wn_nodes = self._winding_state(device).data_ptr()
                face = torch.empty(n, dtype=torch.int32, device=device)
            ws = nat.query_workspace(n, device)
            nat.check(L.pvb_mesh_query(ctypes.byref(desc), nat.ptr(p), n, mode, nat.ptr(dist), nat.ptr(grad),
                                       nat.ptr(closest), nat.ptr(face), nat.ptr(normal), nat.ptr(ws),
                                       ws.numel() if ws is not None else 0, nat.stream_ptr(device)),
                      "pvb_mesh_query")

        def fin(t, tail):
            return nat.deliver(t, out_device, dtype).reshape(*lead, *tail)

        return (fin(closest, (3,)) if want_closest else None, fin(dist, ()), fin(grad, (3,)),
                fin(normal, (3,)) if compute_normal else None)

    def object_frame_closest_point(self, points_in_object_frame, compute_normal=False) -> SDFQuery:
        """
        :param points_in_object_frame: N x 3 points in the object frame (arbitrary batch dimensions in front of N)
        :param compute_normal: whether to also return the surface normal at the closest point
        :return: SDFQuery(closest N x 3, signed distance N, gradient N x 3, normal N x 3 | None)
        """
        return SDFQuery(*self._do_object_frame_closest_point(points_in_object_frame, compute_normal=compute_normal))


class MeshObjectFactory(ObjectFactory):
    def __init__(self, mesh_name='', path_prefix='', **kwargs):
        self.path_prefix = path_prefix
        # strip the package:// prefix when a path prefix is given (loading the mesh manually)
        self.strip_package_prefix = path_prefix != ''
        super(MeshObjectFactory, self).__init__(mesh_name, **kwargs)

    def __reduce__(self):
        fn, args = super().__reduce__()
        return partial(fn.func, path_prefix=self.path_prefix, **fn.keywords), args

    def make_collision_obj(self, z, rgba=None):
        return None, None

    def get_mesh_resource_filename(self):
        mesh_path = self.name
        if self.strip_package_prefix:
            mesh_path = mesh_path.replace("package://", "")
        return os.path.join(self.path_prefix, mesh_path)


class ObjectFrameSDF(abc.ABC):
    @abc.abstractmethod
    def __call__(self, points_in_object_frame):
        """
        Evaluate the signed distance function at given points in the object frame
        :param points_in_object_frame: B x N x d points; located in object frame
        :return: tuple of B x N signed distance (m) and B x N x d SDF gradient pointing towards higher SDF values
        """

    @abc.abstractmethod
    def surface_bounding_box(self, padding=0., padding_ratio=0.):
        """(min,max) per dimension of the 0-level set, inflated by padding + padding_ratio * extent"""

    def outside_surface(self, points_in_object_frame, surface_level=0):
        sdf_values, _ = self.__call__(points_in_object_frame)
        return sdf_values > surface_level

    def get_voxel_view(self, voxels: VoxelGrid = None, dtype=torch.float, device='cpu') -> GridView:
        if voxels is None:
            voxels = VoxelGrid(0.01, self.surface_bounding_box(padding=0.1).cpu().numpy(), dtype=dtype, device=device)
        pts = voxels.get_voxel_center_points()
        sdf_val, sdf_grad = self.__call__(pts.unsqueeze(0))
        cached_underlying_sdf = sdf_val.reshape([len(coord) for coord in voxels.coords])
        return GridView(cached_underlying_sdf, voxels.range_per_dim,
                        invalid_value=lambda p: self.__call__(p)[0])

    def get_filtered_points(self, unary_filter, voxels: VoxelGrid = None, dtype=torch.float,
                            device='cpu') -> torch.tensor:
        model_voxels = self.get_voxel_view(voxels, dtype=dtype, device=device)
        interior = unary_filter(model_voxels.raw_data)
        flat = nonempty_indices(interior.reshape(-1))
        idx = torch.stack(torch.unravel_index(flat, tuple(model_voxels.shape)), dim=-1)
        return model_voxels.ensure_value_key(idx)

    # hook for the fused composition kernels: a pvb_sdf_desc on `device`, or None if this SDF has to be
    # evaluated through its Python __call__
    def native_desc(self, device):
        return None


def _result_like(points, lead, tensors_tails, out_device=None):
    dtype = points.dtype if torch.is_tensor(points) and points.dtype.is_floating_point else torch.float
    dev = out_device if out_device is not None else (points.device if torch.is_tensor(points) else torch.device("cpu"))
    return tuple(nat.deliver(t, dev, dtype).reshape(*lead, *tail) for t, tail in tensors_tails)


def _config_count(tsf_batch):
    """The number of configurations a composition's transforms hold: prod(tsf_batch), 1 without a batch (None)."""
    return 1 if tsf_batch is None else math.prod(list(tsf_batch))


class _query_points:
    """`with _query_points(points) as (device, p)`: enter the device a query of `points` runs on -- theirs when they
    are a CUDA tensor, else the current device -- with p the points as contiguous fp32 (M, 3) on it.  (A class rather
    than a contextlib generator: it is entered on every query call.)"""
    __slots__ = ("points", "guard")

    def __init__(self, points):
        self.points = points

    def __enter__(self):
        device = nat.compute_device(self.points.device if torch.is_tensor(self.points) else None)
        self.guard = torch.cuda.device(device)
        self.guard.__enter__()
        try:
            return device, nat.as_f32_points(self.points, device)
        except BaseException:
            self.guard.__exit__(None, None, None)
            raise

    def __exit__(self, *exc):
        return self.guard.__exit__(*exc)


class SphereSDF(ObjectFrameSDF):
    """SDF for a geometric primitive, the sphere centered at the origin"""

    def __init__(self, radius):
        self.radius = radius

    def __call__(self, points_in_object_frame):
        lead = tuple(points_in_object_frame.shape[:-1])
        with _query_points(points_in_object_frame) as (device, p):
            n = p.shape[0]
            val = torch.empty(n, dtype=torch.float32, device=device)
            grad = torch.empty(n, 3, dtype=torch.float32, device=device)
            nat.check(nat.lib().pvb_sphere_query(float(self.radius), nat.ptr(p), n, nat.ptr(val), nat.ptr(grad),
                                                 nat.stream_ptr(device)), "pvb_sphere_query")
        return _result_like(points_in_object_frame, lead, ((val, ()), (grad, (3,))))

    def surface_bounding_box(self, padding=0., padding_ratio=0.):
        length = self.radius + padding + padding_ratio * self.radius
        return torch.tensor([[-length, length], [-length, length], [-length, length]])

    def native_desc(self, device):
        d = nat.SdfDesc()
        d.kind = nat.PVB_KIND_SPHERE
        d.radius = float(self.radius)
        r = float(np.float32(self.radius))
        _set_primitive_bound(d, [r] * 3, r)
        return d


def _set_primitive_bound(d, half, inradius):
    """Box -half..half and the pruning bound of an analytic primitive descriptor (SPHERE / BOX / CYLINDER).

    The fused kernels skip a sub-SDF when dist(q, bb) - prune_margin exceeds the running minimum, so the value must
    never be below that.  The shape is convex and lies inside its box, so its exact value is >= dist(q, bb) outside
    the shape and >= -inradius inside.  In fp32: inside the box every per-axis term (|q_k| - h_k, rho - r, |q| - r)
    is >= -h_k, -r resp. by monotone rounding, so the value is never below -inradius; outside, the value is the fp32
    rounding of a distance >= dist(q, bb), a few ulp of |q| low at most, and the kernels' own fp32 dist(q, bb) a few
    ulp high.  The slack 1e-5 * max(1, |bb|) (the one MeshSDF uses for the same bound) covers those roundings for
    |q| up to ~30 max(1, |bb|) in the primitive's frame (tests/test_primitive_cpu.py checks it densely)."""
    h = [float(np.float32(v)) for v in half]
    for k in range(3):
        d.bb_min[k] = -h[k]
        d.bb_max[k] = h[k]
    d.prune_margin = float(inradius) + 1e-5 * max(1.0, max(h))
    d.flags = nat.PVB_GRID_PRUNE_OK


def _check_extent(name, v):
    v = float(v)
    if not math.isfinite(v) or v < 0:
        raise ValueError(f"{name} must be finite and >= 0, got {v}")
    return v


class _PrimitiveSDF(ObjectFrameSDF):
    """Analytic primitive evaluated by the fused composition kernels: __call__ is a one-sub-SDF ComposedSDF under
    the identity transform (exact up to the sign of zero), so it shares their arithmetic bit for bit."""
    _half = None      # per-axis half extents of the primitive's box

    def __call__(self, points_in_object_frame):
        comp = self.__dict__.get("_self_composed")
        if comp is None:
            comp = self._self_composed = ComposedSDF([self], Transform3d(matrix=torch.eye(4).unsqueeze(0)))
        lead = tuple(points_in_object_frame.shape[:-1])
        vv, gg = comp(points_in_object_frame)
        return vv.reshape(lead), gg.reshape(*lead, 3)

    def surface_bounding_box(self, padding=0., padding_ratio=0.):
        return torch.tensor([[-(h + padding + padding_ratio * h), h + padding + padding_ratio * h]
                             for h in self._half])


class BoxSDF(_PrimitiveSDF):
    """EXTENSION (the reference has no primitive SDFs): exact SDF of the box with full edge lengths `size`, centred
    at the origin (URDF <box size=...>).

    Outside: the distance to the box, gradient the unit vector from the closest box point.  Inside or on the
    surface: max_k(|q_k| - h_k) with h = size / 2, gradient +-e_k for that axis -- the first axis on ties, + where
    q_k >= 0 (-0 included)."""

    def __init__(self, size):
        size = [_check_extent("BoxSDF size", s) for s in np.asarray(size, dtype=np.float64).reshape(-1)]
        if len(size) != 3:
            raise ValueError(f"BoxSDF size needs 3 edge lengths, got {len(size)}")
        self.size = size
        self._half = [0.5 * s for s in size]

    def native_desc(self, device):
        d = nat.SdfDesc()
        d.kind = nat.PVB_KIND_BOX
        _set_primitive_bound(d, self._half, min(float(np.float32(h)) for h in self._half))
        return d


class CylinderSDF(_PrimitiveSDF):
    """EXTENSION (the reference has no primitive SDFs): exact SDF of the cylinder of `radius` r and total `length`
    along the local z axis, centred at the origin (URDF <cylinder radius=... length=...>).

    With rho = |(x, y)|, u = (x, y) / rho ((1, 0) on the axis) and d = (rho - r, |z| - length / 2): outside,
    w = max(d, 0), value |w| and gradient (w_0 u, w_1 sign z) / |w|; inside or on the surface, value max(d) and
    gradient (u, 0) when d_0 >= d_1 (radial wins ties), else (0, 0, sign z), with sign z = +1 for z >= 0 (-0
    included)."""

    def __init__(self, radius, length):
        self.radius = _check_extent("CylinderSDF radius", radius)
        self.length = _check_extent("CylinderSDF length", length)
        self._half = [self.radius, self.radius, 0.5 * self.length]

    def native_desc(self, device):
        d = nat.SdfDesc()
        d.kind = nat.PVB_KIND_CYLINDER
        d.radius = self.radius
        r, h = float(np.float32(self.radius)), float(np.float32(0.5 * self.length))
        _set_primitive_bound(d, self._half, min(r, h))
        return d


class MeshSDF(ObjectFrameSDF):
    """SDF from direct BVH closest-point + ray-parity queries against the mesh."""

    def __init__(self, obj_factory: ObjectFactory, vis=None):
        if vis is not None:
            raise NotImplementedError("debug drawing (vis=) is outside the query path; pass vis=None")
        self.obj_factory = obj_factory
        self.vis = vis

    def surface_bounding_box(self, **kwargs):
        return torch.tensor(self.obj_factory.bounding_box(**kwargs))

    def __call__(self, points_in_object_frame):
        of = self.obj_factory
        if (type(of).object_frame_closest_point is ObjectFactory.object_frame_closest_point
                and type(of)._do_object_frame_closest_point is ObjectFactory._do_object_frame_closest_point):
            # stock factory: distance and gradient only -- no closest-point output, no copy of it to a host caller
            _, dist, grad, _ = of._do_object_frame_closest_point(points_in_object_frame, want_closest=False)
            return dist, grad
        res = of.object_frame_closest_point(points_in_object_frame)
        return res.distance, res.gradient

    def native_desc(self, device):
        if self.obj_factory.sign_mode != "parity":
            return None      # the fused composition kernels implement the reference's parity rule only
        return self.obj_factory.native_desc(device)


def _affine_inverse(m):
    """Inverse of (n,4,4) affine matrices [A|t; 0 0 0 1] in closed form (adjugate of the 3x3)."""
    A = m[:, :3, :3]
    t = m[:, :3, 3:]
    c0 = torch.linalg.cross(A[:, :, 1], A[:, :, 2], dim=-1)
    c1 = torch.linalg.cross(A[:, :, 2], A[:, :, 0], dim=-1)
    c2 = torch.linalg.cross(A[:, :, 0], A[:, :, 1], dim=-1)
    det = (A[:, :, 0] * c0).sum(-1)
    Ainv = torch.stack([c0, c1, c2], dim=1) / det[:, None, None]
    out = torch.zeros_like(m)
    out[:, :3, :3] = Ainv
    out[:, :3, 3:] = -(Ainv @ t)
    out[:, 3, 3] = 1
    return out


class ComposedSDF(ObjectFrameSDF):
    def __init__(self, sdfs: typing.Sequence[ObjectFrameSDF], obj_frame_to_each_frame):
        """
        :param sdfs: S Object frame SDFs
        :param obj_frame_to_each_frame: [B*]S x 4 x 4 transforms (a Transform3d-like with get_matrix()) from the
        shared object frame to the frame of each SDF, flattened SDF-major when batched over configurations
        """
        self.sdfs = sdfs
        self.obj_frame_to_link_frame = None
        self._link_to_obj = None
        self.tsf_batch = None
        self._desc_cache = {}
        self.set_transforms(obj_frame_to_each_frame)

    # the reference exposes the inverted transforms as a list; build it on demand
    @property
    def link_frame_to_obj_frame(self):
        if self._link_to_obj is None and self.obj_frame_to_link_frame is not None:
            inv = _affine_inverse(matrix_of(self.obj_frame_to_link_frame))
            self._link_to_obj = [Transform3d(matrix=inv[self.ith_transform_slice(i)]) for i in range(len(self.sdfs))]
        return self._link_to_obj if self._link_to_obj is not None else []

    def surface_bounding_box(self, **kwargs):
        # transforms only the (min, max) corner pair of every sub-box, as the reference does (sdf.py:347-368)
        m_inv = _affine_inverse(matrix_of(self.obj_frame_to_link_frame))
        bounds = []
        for i, sdf in enumerate(self.sdfs):
            pts = sdf.surface_bounding_box(**kwargs)
            tsf = Transform3d(matrix=m_inv[self.ith_transform_slice(i)])
            pts = tsf.transform_points(pts.to(dtype=m_inv.dtype, device=m_inv.device).transpose(0, 1))
            if self.tsf_batch is not None and len(pts.shape) == 2:
                pts = pts.unsqueeze(0)
            bounds.append(pts)
        bounds = torch.stack(bounds)
        if self.tsf_batch is not None:
            dims = (0,) + tuple(range(2, len(bounds.shape) - 1))
        else:
            dims = tuple(range(len(bounds.shape) - 1))
        mins = bounds.amin(dim=dims)
        maxs = bounds.amax(dim=dims)
        return torch.stack((mins, maxs), dim=-1)

    def set_transforms(self, tsf, batch_dim=None):
        self.obj_frame_to_link_frame = tsf
        self._link_to_obj = None
        self._xf_dev = {}
        self._inv_xf_dev = {}
        self.tsf_batch = batch_dim
        if tsf is not None:
            S = len(self.sdfs)
            S_tsf = matrix_of(tsf).shape[0]
            if self.tsf_batch is None and (S_tsf != S):
                self.tsf_batch = (S_tsf // S,)
            if S_tsf % S != 0:
                raise ValueError(f"{S_tsf} transforms cannot be split over {S} SDFs")

    def ith_transform_slice(self, i):
        n_cfg = _config_count(self.tsf_batch)
        return slice(i * n_cfg, (i + 1) * n_cfg)

    def _slab(self, cfg_begin, cfg_count):
        """(n_cfg, cfg_count) of the configuration slab [cfg_begin, cfg_begin + cfg_count) of the n_cfg installed
        configurations; cfg_count None runs to the last one."""
        n_cfg = _config_count(self.tsf_batch)
        return n_cfg, n_cfg - cfg_begin if cfg_count is None else cfg_count

    def _check_leading_batch(self, pts_shape, form, tail, n_tail, separate_mismatch=False):
        """The shape rule of a paired form: points of shape pts_shape are [*A, <tail>], the configuration batch A
        leading, then at least n_tail dimensions, the last of size 3.  Otherwise ValueError "<form>: points ... must
        be [*A, <tail>] with the configuration batch A = ... leading"; with separate_mismatch, points with enough
        dimensions but other leading ones get "<form>: points ... must have the configuration batch A = ... leading"
        instead."""
        batch = tuple(int(a) for a in self.tsf_batch or ())
        fits = len(pts_shape) >= len(batch) + n_tail and pts_shape[-1:] == (3,)
        leads = pts_shape[:len(batch)] == batch
        if separate_mismatch and fits and not leads:
            raise ValueError(f"{form}: points {pts_shape} must have the configuration batch A = {batch} leading")
        if not (fits and leads):
            raise ValueError(f"{form}: points {pts_shape} must be [*A, {tail}] with the configuration batch "
                             f"A = {batch} leading")

    @staticmethod
    def _paired_block(lead, cfg_count):
        """The size of each of the cfg_count blocks, one per configuration, that a paired form's `lead` leading points
        split into (0 for an empty slab without points); None when they do not split."""
        if (lead % cfg_count) if cfg_count > 0 else lead:
            return None
        return lead // cfg_count if cfg_count > 0 else 0

    @staticmethod
    def _deliver(points, outs, shape, device=None):
        """Flat query results as a public form returns them: values and gradients in the points' dtype (fp32 for
        non-tensors), index outputs as int64, on `device` -- by default the points' device, CPU for non-tensors --
        and each reshaped to `shape` followed by its own trailing dimensions."""
        dtype = points.dtype if torch.is_tensor(points) else torch.float
        if device is None:
            device = points.device if torch.is_tensor(points) else "cpu"
        res = []
        for t in outs:      # a plain loop and argument-list reshapes: this runs on every call of every public form
            d = nat.deliver(t, device, dtype if t.is_floating_point() else torch.int64)
            res.append(d.reshape(shape) if t.dim() == 1 else d.reshape(*shape, *t.shape[1:]))
        return tuple(res)

    # -- fused path ---------------------------------------------------------------
    #: most sub-SDFs one fused-kernel launch takes (pvb_composed_query* refuse more)
    max_fused_sdfs = 128

    def _native_descs(self, device):
        """(descriptor array, needs_mesh) for the fused kernels, or (None, False) when the set must take the generic
        per-sub-SDF path: some sub-SDF has no native descriptor, or there are more than `max_fused_sdfs` of them."""
        key = (device, tuple(id(s) for s in self.sdfs))
        hit = self._desc_cache.get(key)
        if hit is None:
            descs = None if len(self.sdfs) > self.max_fused_sdfs else [s.native_desc(device) for s in self.sdfs]
            if descs is None or any(d is None for d in descs):
                hit = (None, False, None)
            else:
                needs_mesh = any(d.kind == nat.PVB_KIND_MESH or (d.flags & nat.PVB_GRID_OOB_GT) for d in descs)
                hit = (nat.desc_array(descs), needs_mesh, descs)
            self._desc_cache = {key: hit}
        return hit[0], hit[1]

    def _fused_descs(self, device, form):
        """`_native_descs` of a form only the fused kernels run; NotImplementedError when the set is generic."""
        descs_arr, needs_mesh = self._native_descs(device)
        if descs_arr is None:
            raise NotImplementedError(f"{form} needs the fused kernels: at most 128 sub-SDFs, all with native "
                                      "descriptors")
        return descs_arr, needs_mesh

    def _xforms_on(self, device):
        xf = self._xf_dev.get(device)
        if xf is None:
            xf = matrix_of(self.obj_frame_to_link_frame).detach().to(device=device, dtype=torch.float32).contiguous()
            self._xf_dev = {device: xf}
        return xf

    def _inv_xforms_on(self, device):
        """W = _affine_inverse(M) of the fp32 transforms `_xforms_on` returns: sub-frame -> object frame, [S * A, 4, 4]
        fp32 on `device`, computed once per installed transform set."""
        inv = self._inv_xf_dev.get(device)
        if inv is None:
            inv = _affine_inverse(self._xforms_on(device)).contiguous()
            self._inv_xf_dev = {device: inv}
        return inv

    def query(self, points_in_object_frame, cfg_begin=0, cfg_count=None, return_which=False):
        """__call__ restricted to the configuration slab [cfg_begin, cfg_begin + cfg_count) (multi-GPU sharding
        over configurations).  Returns flat (cfg_count * P,) / (cfg_count * P, 3) fp32 tensors on the GPU."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        with _query_points(points_in_object_frame) as (device, p):
            P = p.shape[0]
            descs_arr, needs_mesh = self._native_descs(device)
            if descs_arr is None:
                return self._generic_query(p, cfg_begin, cfg_count, n_cfg, return_which)
            xf = self._xforms_on(device)
            val = torch.empty(cfg_count * P, dtype=torch.float32, device=device)
            grad = torch.empty(cfg_count * P, 3, dtype=torch.float32, device=device)
            which = torch.empty(cfg_count * P, dtype=torch.int32, device=device) if return_which else None
            nat.check(nat.lib().pvb_composed_query(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg,
                                                   cfg_begin, cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                   nat.ptr(val), nat.ptr(grad), nat.ptr(which),
                                                   nat.stream_ptr(device)), "pvb_composed_query")
        return (val, grad, which) if return_which else (val, grad)

    def query_paired(self, points_in_object_frame, cfg_begin=0, cfg_count=None, return_which=False):
        """Paired form of `query`: configuration cfg_begin + c is evaluated at its own points only.  The points
        reshape to [cfg_count, P, 3]; entry c * P + i of the result is configuration cfg_begin + c at points[c, i].
        Bit-identical to query(points[c], cfg_begin=cfg_begin + c, cfg_count=1) for every c, mesh ray jitter
        included.  Returns flat (cfg_count * P,) / (cfg_count * P, 3) fp32 tensors on the GPU."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        shape = tuple(points_in_object_frame.shape)
        P = self._paired_block(math.prod(shape[:-1]), cfg_count)
        if shape[-1:] != (3,) or P is None:
            raise ValueError(f"paired query: points {shape} do not split into {cfg_count} blocks of [P, 3]")
        with _query_points(points_in_object_frame) as (device, p):
            descs_arr, needs_mesh = self._native_descs(device)
            if descs_arr is None:
                return self._generic_query(p, cfg_begin, cfg_count, n_cfg, return_which, paired=True)
            xf = self._xforms_on(device)
            val = torch.empty(cfg_count * P, dtype=torch.float32, device=device)
            grad = torch.empty(cfg_count * P, 3, dtype=torch.float32, device=device)
            which = torch.empty(cfg_count * P, dtype=torch.int32, device=device) if return_which else None
            nat.check(nat.lib().pvb_composed_query_paired(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg,
                                                          cfg_begin, cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                          nat.ptr(val), nat.ptr(grad), nat.ptr(which),
                                                          nat.stream_ptr(device)), "pvb_composed_query_paired")
        return (val, grad, which) if return_which else (val, grad)

    def paired(self, points_in_object_frame):
        """Every installed configuration at its own points: points [*A, *B, N, 3], with A the configuration batch
        (`tsf_batch`), give (values [*A, *B, N], gradients [*A, *B, N, 3]) in the points' dtype and on their device;
        entry [a, ...] is configuration a evaluated at points[a, ...].

        For GRID and SPHERE sub-SDFs this equals the diagonal of __call__ over the same points, without computing
        the |A|-fold cross product.  For mesh sub-SDFs it equals the per-configuration slab query
        query(points[a], cfg_begin=a, cfg_count=1), ray jitter included.  Without a configuration batch it is
        __call__.  Not a reference operator (an extension); raises ValueError before any device work when the
        leading dimensions of the points are not A."""
        if self.tsf_batch is None:
            return self(points_in_object_frame)
        pts_shape = tuple(points_in_object_frame.shape)
        self._check_leading_batch(pts_shape, "paired query", "..., 3", 1)
        return self._deliver(points_in_object_frame, self.query_paired(points_in_object_frame), pts_shape[:-1])

    #: configurations per chunk of every composition route (bounds its chunk x P temporaries)
    composition_chunk = 64

    def _composition_chunks(self, p, cfg_begin, cfg_count, paired=False):
        """The walk of the composition routes: (c0, cc, points, v, g, w) of every chunk of the slab, ascending, with
        (v, g, w) = query(points, c0, cc, return_which=True) at points = p -- paired (p holds one block of points
        per configuration), query_paired at the chunk's own blocks.  Nothing when there are no points."""
        n_pts = p.shape[0] // max(cfg_count, 1) if paired else p.shape[0]
        for c0 in range(cfg_begin, cfg_begin + (cfg_count if n_pts > 0 else 0), self.composition_chunk):
            cc = min(self.composition_chunk, cfg_begin + cfg_count - c0)
            pts = p[(c0 - cfg_begin) * n_pts:(c0 - cfg_begin + cc) * n_pts] if paired else p
            query = self.query_paired if paired else self.query
            yield (c0, cc, pts, *query(pts, cfg_begin=c0, cfg_count=cc, return_which=True))

    def query_swept(self, points_in_object_frame, cfg_begin=0, cfg_count=None, return_which=False):
        """Swept form of `query`: at every point, the result of the configuration of the slab
        [cfg_begin, cfg_begin + cfg_count) with the smallest value -- the first such configuration on ties -- without
        the cfg_count-fold cross product.  Bit-identical to that reduction of query(..., return_which=True): (value,
        configuration, sub-SDF index) minimised lexicographically.  Returns flat (P,) / (P, 3) fp32 tensors on the GPU,
        and with return_which also the int32 absolute configuration index and sub-SDF index."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        shape = tuple(points_in_object_frame.shape)
        if shape[-1:] != (3,):
            raise ValueError(f"swept query: points {shape} must be [..., 3]")
        if cfg_count < 1 and math.prod(shape[:-1]) > 0:
            raise ValueError(f"swept query: no minimum over an empty configuration slab (cfg_count={cfg_count})")
        with _query_points(points_in_object_frame) as (device, p):
            P = p.shape[0]
            descs_arr, needs_mesh = self._native_descs(device)
            if descs_arr is None:
                return self._composed_swept(p, cfg_begin, cfg_count, return_which)
            xf = self._xforms_on(device)
            val = torch.empty(P, dtype=torch.float32, device=device)
            grad = torch.empty(P, 3, dtype=torch.float32, device=device)
            cfg = torch.empty(P, dtype=torch.int32, device=device) if return_which else None
            which = torch.empty(P, dtype=torch.int32, device=device) if return_which else None
            nat.check(nat.lib().pvb_composed_query_swept(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg,
                                                         cfg_begin, cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                         nat.ptr(val), nat.ptr(grad), nat.ptr(cfg), nat.ptr(which),
                                                         nat.stream_ptr(device)), "pvb_composed_query_swept")
        return (val, grad, cfg, which) if return_which else (val, grad)

    def _composed_swept(self, p, cfg_begin, cfg_count, return_which):
        """query_swept for sub-SDFs without native descriptors, over `_composition_chunks`: within a chunk the first
        configuration attaining the minimum, across chunks a strictly smaller value -- the same (value, configuration,
        sub-SDF) order as the fused kernels."""
        P = p.shape[0]
        best = torch.full((P,), float("inf"), dtype=torch.float32, device=p.device)
        bgrad = torch.zeros(P, 3, dtype=torch.float32, device=p.device)
        bcfg = torch.full((P,), -1, dtype=torch.int32, device=p.device)
        bwhich = torch.full((P,), -1, dtype=torch.int32, device=p.device)
        for c0, cc, _, v, g, w in self._composition_chunks(p, cfg_begin, cfg_count):
            v, g, w = v.reshape(cc, P), g.reshape(cc, P, 3), w.reshape(cc, P)
            first = (v == v.amin(dim=0)).int().argmax(dim=0)          # first configuration attaining the minimum
            cv = v.gather(0, first[None])[0]
            better = (cv < best) | (bcfg < 0)
            best = torch.where(better, cv, best)
            bgrad = torch.where(better[:, None], g.gather(0, first[None, :, None].expand(1, P, 3))[0], bgrad)
            bcfg = torch.where(better, (first + c0).to(torch.int32), bcfg)
            bwhich = torch.where(better, w.gather(0, first[None])[0], bwhich)
        return (best, bgrad, bcfg, bwhich) if return_which else (best, bgrad)

    def swept(self, points_in_object_frame, return_argmin=False):
        """The minimum over every installed configuration at every point (the SDF of the swept volume of a
        trajectory or a set of poses): points [*B, N, 3] give (values [*B, N], gradients [*B, N, 3]) in the points'
        dtype and on their device.  Entry i is configuration c*'s result at point i, c* the first configuration
        attaining the minimum value: bit-identical to __call__ followed by that reduction over the configuration
        dimensions, without materialising the |A| x N cross product.  With return_argmin, also the configuration
        index c* (int64, flat row-major into A) and the sub-SDF index, each [*B, N].  Without a configuration batch
        it is __call__ (configuration 0).  Not a reference operator (an extension); raises ValueError before any
        device work when the points are not [..., 3]."""
        pts_shape = tuple(points_in_object_frame.shape)
        if len(pts_shape) < 1 or pts_shape[-1] != 3:
            raise ValueError(f"swept query: points {pts_shape} must be [..., 3]")
        out = self.query_swept(points_in_object_frame, return_which=return_argmin)
        return self._deliver(points_in_object_frame, out, pts_shape[:-1])

    @staticmethod
    def _clearance_segments(shape):
        """(n_seg, seg_len) of points [*B, N, 3]; ValueError when they are not [..., N, 3]."""
        if len(shape) < 2 or shape[-1] != 3:
            raise ValueError(f"clearance query: points {shape} must be [..., N, 3]")
        return math.prod(shape[:-2]), shape[-2]

    def query_clearance(self, points_in_object_frame, cfg_begin=0, cfg_count=None, return_which=False):
        """Clearance form of `query`: points [*B, N, 3] are n_seg = prod(B) segments of N points; for configuration
        cfg_begin + c and segment b, the per-configuration result at the FIRST point of the segment attaining the
        minimum value, without the cfg_count-fold cross product.  Bit-identical to that reduction of
        query(..., return_which=True) over the flat points: (value, point) minimised lexicographically, -0 == +0, a NaN
        value above every number.  Returns flat (cfg_count * n_seg,) / (cfg_count * n_seg, 3) fp32 tensors on the GPU,
        configuration-major, and with return_which also the int32 point index within the segment and sub-SDF index."""
        _, cfg_count = self._slab(cfg_begin, cfg_count)
        n_seg, seg_len = self._clearance_segments(tuple(points_in_object_frame.shape))
        if n_seg > 0 and seg_len == 0 and cfg_count > 0:
            raise ValueError("clearance query: no minimum over an empty segment (N = 0)")
        if cfg_count < 1 and n_seg * seg_len > 0:
            raise ValueError(f"clearance query: no minimum over an empty configuration slab (cfg_count={cfg_count})")
        return self._clearance_query(points_in_object_frame, cfg_begin, cfg_count, n_seg, seg_len, return_which)

    def _clearance_query(self, points, cfg_begin, cfg_count, n_seg, seg_len, return_which, paired=False):
        """query_clearance (paired=False) or query_paired_clearance (paired=True) once their checks have passed: the
        form's fused entry point, or `_composed_clearance` for the sets the fused kernels do not take."""
        S, n_cfg = len(self.sdfs), _config_count(self.tsf_batch)
        with _query_points(points) as (device, p):
            descs_arr, needs_mesh = self._native_descs(device)
            if descs_arr is None:
                return self._composed_clearance(p, cfg_begin, cfg_count, n_seg, seg_len, return_which, paired=paired)
            xf = self._xforms_on(device)
            R = max(cfg_count, 0) * n_seg
            keys = torch.empty(R, dtype=torch.int64, device=device)
            val = torch.empty(R, dtype=torch.float32, device=device)
            grad = torch.empty(R, 3, dtype=torch.float32, device=device)
            point = torch.empty(R, dtype=torch.int32, device=device) if return_which else None
            which = torch.empty(R, dtype=torch.int32, device=device) if return_which else None
            lib = nat.lib()
            entry = lib.pvb_composed_query_paired_clearance if paired else lib.pvb_composed_query_clearance
            nat.check(entry(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg, cfg_begin, cfg_count, nat.ptr(p),
                            n_seg, seg_len, nat.PVB_MESH_DEFAULT, nat.ptr(keys), nat.ptr(val), nat.ptr(grad),
                            nat.ptr(point), nat.ptr(which), nat.stream_ptr(device)), entry.__name__)
        return (val, grad, point, which) if return_which else (val, grad)

    @staticmethod
    def _clearance_keys(v):
        """The kernels' clearance_key (pvb_device.cuh) of values v [..., N] and their index along the last dimension,
        as int64 in the same order (the unsigned key minus 2^63): its minimum names the first point attaining the
        minimum value, with -0 == +0 and a NaN value above every number."""
        v = torch.where(v == 0, torch.zeros_like(v), v)
        b = v.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
        h = torch.where(b >= 1 << 31, 0xFFFFFFFF - b, b + (1 << 31))
        h = torch.where(torch.isnan(v), torch.full_like(h, 0xFFFFFFFF), h)
        i = torch.arange(v.shape[-1], device=v.device, dtype=torch.int64)
        return ((h - (1 << 31)) << 32) | i

    @classmethod
    def _first_minimum(cls, v):
        """The index (int64) along the last dimension of v of the first minimum in `_clearance_keys` order."""
        return cls._clearance_keys(v).amin(dim=-1) & 0xFFFFFFFF

    def _composed_clearance(self, p, cfg_begin, cfg_count, n_seg, seg_len, return_which, paired=False):
        """query_clearance (paired: query_paired_clearance) for sub-SDFs without native descriptors, over
        `_composition_chunks`: each chunk reduced over the points of every segment by the kernels' key order."""
        R = max(cfg_count, 0) * n_seg
        val = torch.empty(R, dtype=torch.float32, device=p.device)
        grad = torch.empty(R, 3, dtype=torch.float32, device=p.device)
        point = torch.empty(R, dtype=torch.int32, device=p.device)
        which = torch.empty(R, dtype=torch.int32, device=p.device)
        for c0, cc, _, v, g, w in self._composition_chunks(p, cfg_begin, cfg_count, paired):
            v, g, w = v.reshape(cc, n_seg, seg_len), g.reshape(cc, n_seg, seg_len, 3), w.reshape(cc, n_seg, seg_len)
            i = self._first_minimum(v)[..., None]
            out = slice((c0 - cfg_begin) * n_seg, (c0 - cfg_begin + cc) * n_seg)
            val[out] = v.gather(-1, i).reshape(-1)
            grad[out] = g.gather(-2, i[..., None].expand(cc, n_seg, 1, 3)).reshape(-1, 3)
            point[out] = i.reshape(-1).to(torch.int32)
            which[out] = w.gather(-1, i).reshape(-1)
        return (val, grad, point, which) if return_which else (val, grad)

    def clearance(self, points_in_object_frame, return_argmin=False):
        """For every installed configuration, the minimum over the points of every segment (the clearance of the
        configuration to a cloud): points [*B, N, 3] give (values [*A, *B], gradients [*A, *B, 3]) in the points'
        dtype and on their device, A the configuration batch.  Entry [a, b] is configuration a's result at the first
        point of points[b] attaining the minimum value: bit-identical to __call__ followed by that reduction over the
        point dimension, without materialising the |A| x N cross product.  With return_argmin, also that point's index
        into N (int64) and the sub-SDF index, each [*A, *B].  Without a configuration batch the result is [*B].  Not a
        reference operator (an extension); raises ValueError before any device work when the points are not
        [..., N, 3] or N = 0 with segments to reduce."""
        pts_shape = tuple(points_in_object_frame.shape)
        n_seg, seg_len = self._clearance_segments(pts_shape)
        if n_seg > 0 and seg_len == 0:
            raise ValueError("clearance query: no minimum over an empty segment (N = 0)")
        out = self.query_clearance(points_in_object_frame, return_which=return_argmin)
        return self._deliver(points_in_object_frame, out, (*(self.tsf_batch or ()), *pts_shape[:-2]))

    def query_paired_clearance(self, points_in_object_frame, cfg_begin=0, cfg_count=None, return_which=False):
        """Paired form of `query_clearance`: configuration cfg_begin + c against its own points only.  The points
        reshape to [cfg_count, n_seg, N, 3], N = points.shape[-2]; entry c * n_seg + b of the result is
        query_clearance(points[c], cfg_begin=cfg_begin + c, cfg_count=1)[b], bit for bit in all four outputs, mesh
        ray jitter included -- equivalently the first-point (value, point) minimum of query_paired(...,
        return_which=True) over each segment.  Returns flat (cfg_count * n_seg,) / (cfg_count * n_seg, 3) fp32
        tensors on the GPU, configuration-major, and with return_which also the int32 point index within the segment
        and sub-SDF index."""
        _, cfg_count = self._slab(cfg_begin, cfg_count)
        shape = tuple(points_in_object_frame.shape)
        lead, seg_len = self._clearance_segments(shape)
        n_seg = self._paired_block(lead, cfg_count)
        if n_seg is None:
            raise ValueError(f"paired clearance query: points {shape} do not split into {cfg_count} blocks of "
                             f"[n_seg, N, 3]")
        if n_seg > 0 and seg_len == 0:
            raise ValueError("paired clearance query: no minimum over an empty segment (N = 0)")
        return self._clearance_query(points_in_object_frame, cfg_begin, cfg_count, n_seg, seg_len, return_which,
                                     paired=True)

    def paired_clearance(self, points_in_object_frame, return_argmin=False):
        """Every installed configuration against its own cloud: points [*A, *B, N, 3], A the configuration batch, give
        (values [*A, *B], gradients [*A, *B, 3]) in the points' dtype and on their device.  Entry [a, b] is
        configuration a's result at the first point of points[a, b] attaining the minimum value: bit-identical to
        paired() followed by that reduction over N, and to clearance(points[a]) of configuration a alone, without
        |A| times the work of clearance() over every cloud.  With return_argmin, also that point's index into N and
        the sub-SDF index, int64 [*A, *B].  Without a configuration batch it is clearance().  Not a reference
        operator (an extension); raises ValueError before any device work when the leading dimensions of the points
        are not A, when they are not [..., N, 3], or when N = 0 with segments to reduce."""
        if self.tsf_batch is None:
            return self.clearance(points_in_object_frame, return_argmin=return_argmin)
        pts_shape = tuple(points_in_object_frame.shape)
        self._check_leading_batch(pts_shape, "paired clearance query", "..., N, 3", 2, separate_mismatch=True)
        if math.prod(pts_shape[:-2]) > 0 and pts_shape[-2] == 0:
            raise ValueError("paired clearance query: no minimum over an empty segment (N = 0)")
        out = self.query_paired_clearance(points_in_object_frame, return_which=return_argmin)
        return self._deliver(points_in_object_frame, out, pts_shape[:-2])

    def _self_clearance_args(self, link_points, allowed):
        """(K, allowed rows as S lists of bools with the diagonal cleared) of a self-clearance query; ValueError when
        link_points is not [S, K, 3] with 1 <= K < 2^24 or allowed is not an [S, S] bool matrix."""
        S = len(self.sdfs)
        shape = tuple(link_points.shape)
        if len(shape) != 3 or shape[0] != S or shape[2] != 3 or not 1 <= shape[1] < (1 << 24):
            raise ValueError(f"self-clearance query: link_points {shape} must be [S, K, 3] with S = {S} sub-SDFs and "
                             f"1 <= K < 2^24")
        a = allowed if torch.is_tensor(allowed) else torch.as_tensor(np.asarray(allowed))
        if a.dtype != torch.bool or tuple(a.shape) != (S, S):
            raise ValueError(f"self-clearance query: allowed must be an [S, S] = [{S}, {S}] bool matrix, got "
                             f"{tuple(a.shape)} {a.dtype}")
        rows = a.detach().cpu().tolist()
        for i in range(S):
            rows[i][i] = False
        return shape[1], rows

    def _self_clearance_fused(self, device):
        """Whether pvb_composed_query_self_clearance takes this set: native descriptors, at most 8 sub-SDFs, no mesh and
        no LOOKUP_GT_SDF grid (the sets robot_paired_clearance_kernel takes)."""
        descs_arr, needs_mesh = self._native_descs(device)
        return descs_arr is not None and len(self.sdfs) <= 8 and not needs_mesh

    def query_self_clearance(self, link_points, allowed, cfg_begin=0, cfg_count=None, return_which=False):
        """Self-clearance of configurations [cfg_begin, cfg_begin + cfg_count): for configuration a, the smallest
        sdf_j(M_j(a) x) over every source sub-SDF i, every j that `allowed[i, j]` lets i be tested against (the
        diagonal is ignored) and every point x = W_i(a) link_points[i, k], W_i = _affine_inverse(M_i) -- points that
        belong to sub-SDF i, given in its own frame, posed with it.  The minimum is taken over (value, i, k)
        lexicographically, and for that point the first allowed j attaining the value wins; -0 == +0 and a NaN value
        ranks above every number.  The gradient is the object-frame gradient query_paired of the allowed
        sub-composition reports at x.  A configuration without an allowed pair gets +inf, a zero gradient and indices
        -1.

        The definition is the composition route (`_composed_self_clearance`): for every source i, its points posed by
        pvb_transform_points_paired and query_paired_clearance of the composition of its allowed sub-SDFs.  Sets of
        at most 8 grid (bounding-box rule) or primitive sub-SDFs run fused in one kernel and its finish
        (pvb_composed_query_self_clearance), bit-identical to that route; every other set takes the route itself.

        link_points [S, K, 3], 1 <= K < 2^24; allowed [S, S] bool.  Returns flat (cfg_count,) / (cfg_count, 3) fp32
        tensors on the GPU, and with return_which also int32 source sub-SDF i, point k and sub-SDF j.  Raises
        ValueError before any device work on wrong shapes or an empty slab."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        K, rows = self._self_clearance_args(link_points, allowed)
        if cfg_count < 1 or cfg_begin < 0 or cfg_begin + cfg_count > n_cfg:
            raise ValueError(f"self-clearance query: empty or invalid configuration slab [{cfg_begin}, +{cfg_count}) "
                             f"of {n_cfg}")
        with _query_points(link_points) as (device, p):
            if not self._self_clearance_fused(device):
                return self._composed_self_clearance(p, K, rows, cfg_begin, cfg_count, return_which)
            descs_arr, _ = self._native_descs(device)
            xf, inv = self._xforms_on(device), self._inv_xforms_on(device)
            masks = (ctypes.c_uint8 * S)(*[sum(1 << j for j in range(S) if rows[i][j]) for i in range(S)])
            keys = torch.empty(cfg_count, dtype=torch.int64, device=device)
            val = torch.empty(cfg_count, dtype=torch.float32, device=device)
            grad = torch.empty(cfg_count, 3, dtype=torch.float32, device=device)
            src, point, which = (torch.empty(cfg_count, dtype=torch.int32, device=device) if return_which else None
                                 for _ in range(3))
            nat.check(nat.lib().pvb_composed_query_self_clearance(descs_arr, S, nat.ptr(xf), nat.ptr(inv), n_cfg,
                                                                  cfg_begin, cfg_count, nat.ptr(p), K, masks,
                                                                  nat.ptr(keys), nat.ptr(val), nat.ptr(grad),
                                                                  nat.ptr(src), nat.ptr(point), nat.ptr(which),
                                                                  nat.stream_ptr(device)),
                      "pvb_composed_query_self_clearance")
        return (val, grad, src, point, which) if return_which else (val, grad)

    def _self_sources(self, rows, device):
        """The sources of the self routes: (i, js, sub) for every sub-SDF i with an allowed row, js the sub-SDFs
        rows[i] allows and sub = ComposedSDF([sdfs[j] for j in js]) with their transform rows on `device`."""
        S, n_cfg = len(self.sdfs), _config_count(self.tsf_batch)
        xf = self._xforms_on(device).reshape(S, n_cfg, 4, 4)
        for i in range(S):
            js = [j for j in range(S) if rows[i][j]]
            if js:
                sub = ComposedSDF([self.sdfs[j] for j in js], None)
                sub.set_transforms(Transform3d(matrix=xf[js].reshape(len(js) * n_cfg, 4, 4)), batch_dim=(n_cfg,))
                yield i, js, sub

    def _posed_link_points(self, lp, i, c0, cc):
        """link_points[i] of lp [S, K, 3] fp32, posed by W_i of configurations [c0, c0 + cc): [cc, K, 3] fp32 from
        pvb_transform_points_paired."""
        (S, K, _), device = lp.shape, lp.device
        w_i = self._inv_xforms_on(device).reshape(S, -1, 4, 4)[i, c0:c0 + cc].contiguous()
        own = lp[i].expand(cc, K, 3).contiguous()
        x = torch.empty(cc, K, 3, dtype=torch.float32, device=device)
        nat.check(nat.lib().pvb_transform_points_paired(nat.ptr(w_i), cc, nat.ptr(own), K, nat.ptr(x),
                                                        nat.stream_ptr(device)), "pvb_transform_points_paired")
        return x

    def _composed_self_clearance(self, p, K, rows, cfg_begin, cfg_count, return_which):
        """query_self_clearance by composition, the definition of its result: for every source, its points posed over
        the slab and query_paired_clearance(..., return_which=True) of its sub-composition, the sub-SDF index mapped
        back; then the minimum over the sources by (value, source)."""
        device = p.device
        lp = p.reshape(len(self.sdfs), K, 3)
        per_src = []
        for i, js, sub in self._self_sources(rows, device):
            x = self._posed_link_points(lp, i, cfg_begin, cfg_count)
            v, g, pt, w = sub.query_paired_clearance(x, cfg_begin=cfg_begin, cfg_count=cfg_count, return_which=True)
            w = torch.tensor(js, dtype=torch.int32, device=device)[w.long()]
            per_src.append((i, v, g, pt, w))
        if not per_src:
            val = torch.full((cfg_count,), float("inf"), dtype=torch.float32, device=device)
            grad = torch.zeros(cfg_count, 3, dtype=torch.float32, device=device)
            idx = [torch.full((cfg_count,), -1, dtype=torch.int32, device=device) for _ in range(3)]
            return (val, grad, *idx) if return_which else (val, grad)
        v = torch.stack([r[1] for r in per_src], dim=1)                                   # [cfg_count, n_src]
        pos = self._first_minimum(v)[:, None]                                              # first source on ties
        val = v.gather(1, pos).reshape(-1)
        grad = torch.stack([r[2] for r in per_src], dim=1).gather(1, pos[..., None].expand(cfg_count, 1, 3))
        grad = grad.reshape(-1, 3)
        if not return_which:
            return val, grad
        srcs = torch.tensor([r[0] for r in per_src], dtype=torch.int32, device=device)[pos.reshape(-1)]
        point = torch.stack([r[3] for r in per_src], dim=1).gather(1, pos).reshape(-1)
        which = torch.stack([r[4] for r in per_src], dim=1).gather(1, pos).reshape(-1)
        return val, grad, srcs, point, which

    def self_clearance(self, link_points, allowed, return_argmin=False):
        """For every installed configuration, the smallest distance between its own sub-SDFs: link_points [S, K, 3]
        holds K points of every sub-SDF in its own frame (its surface, say), and allowed [S, S] bool says which
        sub-SDFs the points of each one are tested against (the diagonal is ignored).  Returns (values [*A],
        gradients [*A, 3]) in link_points' dtype on the composition's device -- 0-d / [3] without a configuration
        batch -- and with return_argmin also the source sub-SDF i, point k and sub-SDF j, int64 [*A].  Negative
        values mean the two sub-SDFs intersect.  The semantics, tie rule and routes are those of
        `query_self_clearance`; a configuration without an allowed pair gets +inf and indices -1.  Not a reference
        operator (an extension); raises ValueError before any device work on wrong shapes."""
        shape = () if self.tsf_batch is None else tuple(int(a) for a in self.tsf_batch)
        out = self.query_self_clearance(link_points, allowed, return_which=return_argmin)
        return self._deliver(link_points, out, shape, device=matrix_of(self.obj_frame_to_link_frame).device)

    @staticmethod
    def _collision_cost_margin(margin):
        """The margin rounded to fp32 (every route computes with that value), as a Python float; ValueError unless it
        is one number that stays finite in fp32."""
        try:
            m = float(np.float32(float(margin)))
        except (TypeError, ValueError, RuntimeError):
            raise ValueError(f"collision-cost query: the margin must be one finite number, got {margin!r}") from None
        if not math.isfinite(m):
            raise ValueError(f"collision-cost query: the margin must be finite, got {m}")
        return m

    def query_collision_cost(self, points_in_object_frame, margin, cfg_begin=0, cfg_count=None):
        """Collision cost of configurations [cfg_begin, cfg_begin + cfg_count) against points [*B, N, 3], n_seg =
        prod(B) segments of N points.  For configuration a, segment b and margin m (rounded to fp32), with (d, g, s) what
        query(..., return_which=True) gives at point p (value, object-frame gradient, first sub-SDF attaining it):
        cost = sum_p max(0, m - d)^2, and for every sub-SDF s, twist[s] = sum over the p with argmin s and d < m of
        (2 (m - d) g, 2 (m - d) (p x g)) -- the derivative of the cost when sub-SDF s alone moves by an object-frame
        twist (v, w) about the origin.  A segment without points costs 0.

        Sets of at most 8 grid (bounding-box rule) or primitive sub-SDFs run in one fused kernel
        (pvb_composed_query_collision_cost); every other set is composed from `query` in chunks of
        `composition_chunk` configurations and reduced in torch.  Both are deterministic, and the fused route's
        rows do not depend on the slab: a configuration split reproduces the full call bit for bit.  Returns flat
        (cfg_count * n_seg,) / (cfg_count * n_seg, S, 6) fp32 tensors on the GPU, configuration-major.  Raises
        ValueError before any device work on malformed points, a margin that is not finite, or a slab without
        configurations when there are points."""
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        m = self._collision_cost_margin(margin)
        shape = tuple(points_in_object_frame.shape)
        if len(shape) < 2 or shape[-1] != 3:
            raise ValueError(f"collision-cost query: points {shape} must be [..., N, 3]")
        n_seg, seg_len = math.prod(shape[:-2]), shape[-2]
        if cfg_begin < 0 or cfg_count < 0 or cfg_begin + cfg_count > n_cfg or (cfg_count < 1 and n_seg * seg_len > 0):
            raise ValueError(f"collision-cost query: invalid configuration slab [{cfg_begin}, +{cfg_count}) of {n_cfg}")
        return self._collision_cost_query(points_in_object_frame, m, cfg_begin, cfg_count, n_seg, seg_len)

    def _collision_cost_query(self, points, m, cfg_begin, cfg_count, n_seg, seg_len, paired=False):
        """query_collision_cost (paired=False) or query_paired_collision_cost (paired=True) once their checks have
        passed: the form's fused entry point, or `_composed_collision_cost` for the sets the fused kernels refuse."""
        S, n_cfg = len(self.sdfs), _config_count(self.tsf_batch)
        with _query_points(points) as (device, p):
            R = cfg_count * n_seg
            if not self._self_clearance_fused(device):
                return self._composed_collision_cost(p, m, cfg_begin, cfg_count, n_seg, seg_len, paired=paired)
            descs_arr, _ = self._native_descs(device)
            xf = self._xforms_on(device)
            cost = torch.empty(R, dtype=torch.float32, device=device)
            twist = torch.empty(R, S, 6, dtype=torch.float32, device=device)
            lib = nat.lib()
            need = lib.pvb_collision_cost_workspace(S, cfg_count, n_seg, seg_len)
            ws = torch.empty(max(need, 0) // 4, dtype=torch.float32, device=device)
            entry = lib.pvb_composed_query_paired_collision_cost if paired else lib.pvb_composed_query_collision_cost
            nat.check(entry(descs_arr, S, nat.ptr(xf), n_cfg, cfg_begin, cfg_count, nat.ptr(p), n_seg, seg_len, m,
                            nat.ptr(ws) if need > 0 else None, need, nat.ptr(cost), nat.ptr(twist),
                            nat.stream_ptr(device)), entry.__name__)
        return cost, twist

    @staticmethod
    def _hinge_terms(v, g, x, m):
        """The terms of a collision cost in fp64 at values v [...], gradients g [..., 3] and points x (broadcast to
        g) for margin m: (h, tau) with h = max(0, m - v), 0 exactly where v >= m, and tau = 2h (g, x x g) [..., 6]."""
        h = (m - v.double()).clamp_min(0.0)
        g = g.double()
        return h, torch.cat([g, torch.linalg.cross(x.double().expand_as(g), g, dim=-1)], dim=-1) * (2.0 * h)[..., None]

    def _composed_collision_cost(self, p, m, cfg_begin, cfg_count, n_seg, seg_len, paired=False):
        """query_collision_cost (paired: query_paired_collision_cost) by composition, for the sets the fused kernel
        refuses: `_composition_chunks`, the `_hinge_terms` grouped by sub-SDF with one mask and one sum per sub-SDF
        (torch's sums are deterministic; scatter_add / index_add on CUDA are not)."""
        S = len(self.sdfs)
        R = cfg_count * n_seg
        cost = torch.zeros(R, dtype=torch.float32, device=p.device)
        twist = torch.zeros(R, S, 6, dtype=torch.float32, device=p.device)
        shared = None if paired else p.double().reshape(n_seg, seg_len, 3)
        for c0, cc, x, v, g, w in self._composition_chunks(p, cfg_begin, cfg_count, paired):
            pts = x.double().reshape(cc, n_seg, seg_len, 3) if paired else shared
            v, g, w = v.reshape(cc, n_seg, seg_len), g.reshape(cc, n_seg, seg_len, 3), w.reshape(cc, n_seg, seg_len)
            h, terms = self._hinge_terms(v, g, pts, m)
            out = slice((c0 - cfg_begin) * n_seg, (c0 - cfg_begin + cc) * n_seg)
            cost[out] = (h * h).sum(dim=-1).reshape(-1).float()
            for s in range(S):
                twist[out, s] = (terms * (w == s)[..., None]).sum(dim=-2).reshape(-1, 6).float()
        return cost, twist

    def collision_cost(self, points_in_object_frame, margin):
        """For every installed configuration and every segment of points [*B, N, 3], the soft collision cost
        sum_p max(0, margin - d)^2 over the points within `margin` of the composition, and its twist gradient per
        sub-SDF: returns (cost [*A, *B], twist_grad [*A, *B, S, 6]) in the points' dtype and on their device, A the
        configuration batch (no A without one).  twist_grad[..., s, :] = (dC/dv_s, dC/dw_s), the derivative of the cost
        when sub-SDF s alone moves by an object-frame twist (v, w) about the origin; a point contributes to the
        sub-SDF that attains its minimum, with the gradient `__call__` reports there.  Margins <= 0 count penetration
        only; a segment with N = 0 costs 0.  Semantics and routes are those of `query_collision_cost`.  Not a
        reference operator (an extension); raises ValueError before any device work on malformed points or a margin
        that is not finite."""
        pts_shape = tuple(points_in_object_frame.shape)
        if len(pts_shape) < 2 or pts_shape[-1] != 3:
            raise ValueError(f"collision-cost query: points {pts_shape} must be [..., N, 3]")
        m = self._collision_cost_margin(margin)
        out = self.query_collision_cost(points_in_object_frame, m)
        return self._deliver(points_in_object_frame, out, (*(self.tsf_batch or ()), *pts_shape[:-2]))

    def query_paired_collision_cost(self, points_in_object_frame, margin, cfg_begin=0, cfg_count=None):
        """Paired form of `query_collision_cost`: configuration cfg_begin + c against its own points only.  The points
        reshape to [cfg_count, n_seg, N, 3], N = points.shape[-2]; entry c * n_seg + b of the result, cost and twist,
        is query_collision_cost(points[c], margin, cfg_begin=cfg_begin + c, cfg_count=1)[b] -- the margin rounded to
        fp32, the terms of the (d, g, s) query_paired(..., return_which=True) gives at each point, object-frame twists
        about the origin, and 0 with all-zero twists for N = 0.

        Sets of at most 8 grid (bounding-box rule) or primitive sub-SDFs run in one fused kernel
        (pvb_composed_query_paired_collision_cost), bit-identical to that definition; every other set is composed from
        `query_paired` in chunks of `composition_chunk` configurations and reduced in torch, equal to it within
        fp32 rounding.  Returns flat (cfg_count * n_seg,) / (cfg_count * n_seg, S, 6) fp32 tensors on the GPU,
        configuration-major.  Raises ValueError before any device work on malformed points, points that do not split
        into cfg_count blocks, an invalid slab or a margin that is not finite."""
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        m = self._collision_cost_margin(margin)
        shape = tuple(points_in_object_frame.shape)
        if len(shape) < 2 or shape[-1] != 3:
            raise ValueError(f"paired collision-cost query: points {shape} must be [..., N, 3]")
        lead, seg_len = math.prod(shape[:-2]), shape[-2]
        if cfg_begin < 0 or cfg_count < 0 or cfg_begin + cfg_count > n_cfg:
            raise ValueError(f"paired collision-cost query: invalid configuration slab [{cfg_begin}, +{cfg_count}) of "
                             f"{n_cfg}")
        n_seg = self._paired_block(lead, cfg_count)
        if n_seg is None:
            raise ValueError(f"paired collision-cost query: points {shape} do not split into {cfg_count} blocks of "
                             f"[n_seg, N, 3]")
        return self._collision_cost_query(points_in_object_frame, m, cfg_begin, cfg_count, n_seg, seg_len,
                                          paired=True)

    def paired_collision_cost(self, points_in_object_frame, margin):
        """Every installed configuration against its own cloud: points [*A, *B, N, 3], A the configuration batch, give
        (cost [*A, *B], twist_grad [*A, *B, S, 6]) in the points' dtype and on their device.  Entry [a, b] is
        configuration a's collision cost over points[a, b] and its twist gradient per sub-SDF: what collision_cost of
        configuration a alone gives over points[a] (bit for bit on the fused sets), without |A| times the work of
        collision_cost over every cloud.  Without a configuration batch it is collision_cost.  Semantics and routes are
        those of `query_paired_collision_cost`.  Not a reference operator (an extension), and not autograd: the
        gradient is an output of the query.  Raises ValueError before any device work when the leading dimensions of
        the points are not A, when they are not [..., N, 3], or when the margin is not finite."""
        if self.tsf_batch is None:
            return self.collision_cost(points_in_object_frame, margin)
        pts_shape = tuple(points_in_object_frame.shape)
        self._check_leading_batch(pts_shape, "paired collision-cost query", "..., N, 3", 2, separate_mismatch=True)
        m = self._collision_cost_margin(margin)
        out = self.query_paired_collision_cost(points_in_object_frame, m)
        return self._deliver(points_in_object_frame, out, pts_shape[:-2])

    def query_self_collision_cost(self, link_points, allowed, margin, cfg_begin=0, cfg_count=None):
        """Self-collision cost of configurations [cfg_begin, cfg_begin + cfg_count) and its twist gradient per
        sub-SDF.

        Inputs: a composition of S sub-SDFs with transforms M_s(a), and W_s = _affine_inverse(M_s); link_points
        [S, K, 3], each row in its own sub-SDF's frame; allowed [S, S] bool (the diagonal is ignored); a margin m,
        rounded to fp32 exactly as _collision_cost_margin does.  For configuration a, every source i and every
        point k:
          - x = W_i(a) . link_points[i, k], posed with composed_xform.  This is the same posed point as in
            pvb_transform_points_paired and self_clearance.
          - (d, g, j) is what query_paired(..., return_which=True) of the composition of row i's allowed sub-SDFs
            gives at x: the value, the object-frame gradient, and the first allowed sub-SDF attaining the value.  These
            are the per-point values _composed_self_clearance already uses.
          - When d < m, with h = m - d and tau = 2h (g, x x g):
              - cost[a] += h^2
              - twist[a, j] += tau.  The target moves.  This is the same term and sign as collision_cost_term.
              - twist[a, i] -= tau.  The source moves.  Its point travels with it, so d changes by +g . (v + w x x).
          - twist[a, s] is therefore the derivative of the cost when sub-SDF s alone moves by an object-frame twist
            (v, w) about the origin.  This is the convention of collision_cost, so RobotSDF.joint_gradient applies
            unchanged.
          - A configuration with no allowed pair, or with no point below m, costs exactly 0 and has all-zero twists.

        Sets of at most 8 grid (bounding-box rule) or primitive sub-SDFs run in one fused kernel
        (pvb_composed_query_self_collision_cost); every other set takes the composition route
        (`_composed_self_collision_cost`), against which the fused route is checked.  Both are deterministic, and the
        fused route's rows do not depend on the slab: a configuration split reproduces the full call bit for bit.
        Returns flat (cfg_count,) / (cfg_count, S, 6) fp32 tensors on the GPU.  Raises ValueError before any device
        work on wrong shapes, a margin that is not finite, or an empty slab."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        K, rows = self._self_clearance_args(link_points, allowed)
        m = self._collision_cost_margin(margin)
        if cfg_count < 1 or cfg_begin < 0 or cfg_begin + cfg_count > n_cfg:
            raise ValueError(f"self-collision-cost query: empty or invalid configuration slab [{cfg_begin}, "
                             f"+{cfg_count}) of {n_cfg}")
        with _query_points(link_points) as (device, p):
            if not self._self_clearance_fused(device):
                return self._composed_self_collision_cost(p, K, rows, m, cfg_begin, cfg_count)
            descs_arr, _ = self._native_descs(device)
            xf, inv = self._xforms_on(device), self._inv_xforms_on(device)
            masks = (ctypes.c_uint8 * S)(*[sum(1 << j for j in range(S) if rows[i][j]) for i in range(S)])
            cost = torch.empty(cfg_count, dtype=torch.float32, device=device)
            twist = torch.empty(cfg_count, S, 6, dtype=torch.float32, device=device)
            nat.check(nat.lib().pvb_composed_query_self_collision_cost(descs_arr, S, nat.ptr(xf), nat.ptr(inv), n_cfg,
                                                                       cfg_begin, cfg_count, nat.ptr(p), K, masks, m,
                                                                       nat.ptr(cost), nat.ptr(twist),
                                                                       nat.stream_ptr(device)),
                      "pvb_composed_query_self_collision_cost")
        return cost, twist

    def _composed_self_collision_cost(self, p, K, rows, m, cfg_begin, cfg_count):
        """query_self_collision_cost by composition, the definition of its result: for every source and chunk, its
        points posed and query_paired(..., return_which=True) of its sub-composition; the `_hinge_terms`, one masked
        sum per target, and the source's total subtracted (torch's sums are deterministic; scatter_add / index_add
        on CUDA are not)."""
        S = len(self.sdfs)
        device = p.device
        lp = p.reshape(S, K, 3)
        cost = torch.zeros(cfg_count, dtype=torch.float64, device=device)
        twist = torch.zeros(cfg_count, S, 6, dtype=torch.float64, device=device)
        for i, js, sub in self._self_sources(rows, device):
            js_t = torch.tensor(js, dtype=torch.long, device=device)
            for c0 in range(cfg_begin, cfg_begin + cfg_count, self.composition_chunk):
                cc = min(self.composition_chunk, cfg_begin + cfg_count - c0)
                x = self._posed_link_points(lp, i, c0, cc)
                v, g, w = sub.query_paired(x, cfg_begin=c0, cfg_count=cc, return_which=True)
                h, tau = self._hinge_terms(v.reshape(cc, K), g.reshape(cc, K, 3), x, m)
                w = js_t[w.long()].reshape(cc, K)
                rs = slice(c0 - cfg_begin, c0 - cfg_begin + cc)
                cost[rs] += (h * h).sum(dim=-1)
                for j in js:
                    twist[rs, j] += (tau * (w == j)[..., None]).sum(dim=-2)
                twist[rs, i] -= tau.sum(dim=-2)
        return cost.float(), twist.float()

    def self_collision_cost(self, link_points, allowed, margin):
        """For every installed configuration, the soft self-collision cost between its own sub-SDFs and its twist
        gradient per sub-SDF: link_points [S, K, 3] holds K points of every sub-SDF in its own frame (its surface,
        say), allowed [S, S] bool says which sub-SDFs the points of each one are tested against (the diagonal is
        ignored), and every posed point within `margin` of an allowed sub-SDF adds max(0, margin - d)^2.  Returns
        (cost [*A], twist_grad [*A, S, 6]) in link_points' dtype on the composition's device -- 0-d / [S, 6] without a
        configuration batch.  twist_grad[..., s, :] is the derivative of the cost when sub-SDF s alone moves by an
        object-frame twist (v, w) about the origin: a term adds to its target and subtracts from its source, so
        moving both together changes nothing.  The definition and routes are those of `query_self_collision_cost`.
        Not a reference operator (an extension); raises ValueError before any device work on wrong shapes or a margin
        that is not finite."""
        shape = () if self.tsf_batch is None else tuple(int(a) for a in self.tsf_batch)
        out = self.query_self_collision_cost(link_points, allowed, margin)
        return self._deliver(link_points, out, shape, device=matrix_of(self.obj_frame_to_link_frame).device)

    #: most sub-SDFs a composition may hold on the fused scene route (the 8 bits of the source in its key)
    max_scene_sources = 255

    def _scene_args(self, scene, link_points, links, form):
        """(K, links as S bools) of a scene query; ValueError when link_points is not [S, K, 3] with 1 <= K < 2^24,
        links is not an [S] bool mask, or the scene is not an ObjectFrameSDF with one pose."""
        S = len(self.sdfs)
        shape = tuple(link_points.shape)
        if len(shape) != 3 or shape[0] != S or shape[2] != 3 or not 1 <= shape[1] < (1 << 24):
            raise ValueError(f"{form}: link_points {shape} must be [S, K, 3] with S = {S} sub-SDFs and 1 <= K < 2^24")
        if links is None:
            mask = [True] * S
        else:
            lk = links if torch.is_tensor(links) else torch.as_tensor(np.asarray(links))
            if lk.dtype != torch.bool or tuple(lk.shape) != (S,):
                raise ValueError(f"{form}: links must be an [S] = [{S}] bool mask, got {tuple(lk.shape)} {lk.dtype}")
            mask = lk.detach().cpu().tolist()
        if not isinstance(scene, ObjectFrameSDF):
            raise ValueError(f"{form}: the scene must be an ObjectFrameSDF, got {type(scene).__name__}")
        if isinstance(scene, ComposedSDF) and _config_count(scene.tsf_batch) != 1:
            raise ValueError(f"{form}: the scene ComposedSDF holds {_config_count(scene.tsf_batch)} configurations; a "
                             f"static scene has one pose")
        return shape[1], mask

    def _scene_fused(self, scene, device):
        """(descriptor array, n_scene, scene transforms [n_scene, 4, 4] fp32 on `device`) when the fused scene kernels
        take this composition and scene, else None: at most `max_scene_sources` sub-SDFs here, and a scene of grid
        (bounding-box rule) or primitive SDFs -- a CachedSDF, SphereSDF, BoxSDF or CylinderSDF, or a one-configuration
        ComposedSDF of at most 128 of them.  A bare scene is one sub-SDF under the identity."""
        if len(self.sdfs) > self.max_scene_sources:
            return None
        if isinstance(scene, ComposedSDF):
            descs_arr, needs_mesh = scene._native_descs(device)
            if descs_arr is None or needs_mesh:
                return None
            return descs_arr, len(scene.sdfs), scene._xforms_on(device)
        d = scene.native_desc(device)
        if d is None or d.kind == nat.PVB_KIND_MESH or (d.flags & nat.PVB_GRID_OOB_GT):
            return None
        return nat.desc_array([d]), 1, torch.eye(4, dtype=torch.float32, device=device)

    def _scene_slab(self, cfg_begin, cfg_count, form):
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        if cfg_count < 1 or cfg_begin < 0 or cfg_begin + cfg_count > n_cfg:
            raise ValueError(f"{form}: empty or invalid configuration slab [{cfg_begin}, +{cfg_count}) of {n_cfg}")
        return n_cfg, cfg_count

    def query_scene_clearance(self, scene, link_points, links=None, cfg_begin=0, cfg_count=None, return_which=False):
        """Scene clearance of configurations [cfg_begin, cfg_begin + cfg_count): for configuration a, the smallest
        value of the static `scene` over every source sub-SDF i that `links[i]` tests (default: all) and every point
        x = W_i(a) link_points[i, k], W_i = _affine_inverse(M_i) -- points that belong to sub-SDF i, given in its own
        frame, posed with it (pvb_transform_points_paired).  The scene is any ObjectFrameSDF in this composition's
        object frame (place one with ComposedSDF([scene], T)); (d, g) is its value and gradient at x.  The minimum is
        taken over (d, i, k) lexicographically, -0 == +0 and a NaN value above every number.  A configuration without
        a tested source gets +inf, a zero gradient and indices -1.

        The definition is the composition route (`_composed_scene_clearance`: the posed points and scene(x)).  Scenes
        of grid (bounding-box rule) or primitive SDFs -- CachedSDF, SphereSDF, BoxSDF, CylinderSDF, or a
        one-configuration ComposedSDF of at most 128 of them -- run fused in one kernel
        (pvb_composed_query_scene_clearance) for any kind of sub-SDF here, up to 255 of them, bit-identical to that
        route; every other scene takes the route itself.

        link_points [S, K, 3], 1 <= K < 2^24; links [S] bool.  Returns flat (cfg_count,) / (cfg_count, 3) fp32
        tensors on the GPU, and with return_which also the int32 source i and point k.  Raises ValueError before any
        device work on wrong shapes, a scene with more than one pose, or an empty slab."""
        form = "scene-clearance query"
        K, mask = self._scene_args(scene, link_points, links, form)
        n_cfg, cfg_count = self._scene_slab(cfg_begin, cfg_count, form)
        S = len(self.sdfs)
        with _query_points(link_points) as (device, p):
            fused = self._scene_fused(scene, device)
            if fused is None:
                return self._composed_scene_clearance(scene, p, K, mask, cfg_begin, cfg_count, return_which)
            descs_arr, n_scene, sxf = fused
            inv = self._inv_xforms_on(device)
            val = torch.empty(cfg_count, dtype=torch.float32, device=device)
            grad = torch.empty(cfg_count, 3, dtype=torch.float32, device=device)
            link, point = (torch.empty(cfg_count, dtype=torch.int32, device=device) if return_which else None
                           for _ in range(2))
            nat.check(nat.lib().pvb_composed_query_scene_clearance(
                descs_arr, n_scene, nat.ptr(sxf), nat.ptr(inv), S, n_cfg, cfg_begin, cfg_count, nat.ptr(p), K,
                (ctypes.c_uint8 * S)(*mask), nat.ptr(val), nat.ptr(grad), nat.ptr(link), nat.ptr(point),
                nat.stream_ptr(device)), "pvb_composed_query_scene_clearance")
        return (val, grad, link, point) if return_which else (val, grad)

    def _scene_chunks(self, scene, p, K, srcs, cfg_begin, cfg_count):
        """The walk of the scene composition routes: (c0, cc, x, v, g) for every chunk of `composition_chunk`
        configurations, ascending, with x [cc, n_src, K, 3] the tested sources' points posed (`_posed_link_points`)
        and (v [cc, n_src, K], g [..., 3]) = scene(x) as fp32."""
        lp = p.reshape(len(self.sdfs), K, 3)
        for c0 in range(cfg_begin, cfg_begin + cfg_count, self.composition_chunk):
            cc = min(self.composition_chunk, cfg_begin + cfg_count - c0)
            x = torch.stack([self._posed_link_points(lp, i, c0, cc) for i in srcs], dim=1)
            v, g = scene(x)
            yield (c0, cc, x, v.to(device=p.device, dtype=torch.float32).reshape(cc, len(srcs), K),
                   g.to(device=p.device, dtype=torch.float32).reshape(cc, len(srcs), K, 3))

    def _composed_scene_clearance(self, scene, p, K, mask, cfg_begin, cfg_count, return_which):
        """query_scene_clearance by composition, the definition of its result: `_scene_chunks`, then the first
        minimum over (source, point) in clearance-key order."""
        device = p.device
        srcs = [i for i, on in enumerate(mask) if on]
        val = torch.full((cfg_count,), float("inf"), dtype=torch.float32, device=device)
        grad = torch.zeros(cfg_count, 3, dtype=torch.float32, device=device)
        link, point = (torch.full((cfg_count,), -1, dtype=torch.int32, device=device) for _ in range(2))
        src_t = torch.tensor(srcs, dtype=torch.int64, device=device)
        for c0, cc, _, v, g in (self._scene_chunks(scene, p, K, srcs, cfg_begin, cfg_count) if srcs else ()):
            j = self._first_minimum(v.reshape(cc, -1))[:, None]                      # pos * K + k: (i, k) order
            out = slice(c0 - cfg_begin, c0 - cfg_begin + cc)
            val[out] = v.reshape(cc, -1).gather(1, j).reshape(-1)
            grad[out] = g.reshape(cc, -1, 3).gather(1, j[..., None].expand(cc, 1, 3)).reshape(-1, 3)
            link[out] = src_t[j.reshape(-1) // K].to(torch.int32)
            point[out] = (j.reshape(-1) % K).to(torch.int32)
        return (val, grad, link, point) if return_which else (val, grad)

    def scene_clearance(self, scene, link_points, links=None, return_argmin=False):
        """For every installed configuration, the smallest distance from its tested links to a static scene:
        link_points [S, K, 3] holds K points of every sub-SDF in its own frame (its surface, say), links [S] bool says
        which sub-SDFs are tested (default: all), and `scene` is any ObjectFrameSDF in this composition's object frame.
        Returns (values [*A], scene gradients [*A, 3]) in link_points' dtype on the composition's device -- 0-d / [3]
        without a configuration batch -- and with return_argmin also the source sub-SDF i and point k, int64 [*A].
        Negative values mean a link penetrates the scene.  The semantics, tie rule and routes are those of
        `query_scene_clearance`.  Not a reference operator (an extension); raises ValueError before any device work on
        wrong shapes or a scene with more than one pose."""
        shape = () if self.tsf_batch is None else tuple(int(a) for a in self.tsf_batch)
        out = self.query_scene_clearance(scene, link_points, links, return_which=return_argmin)
        return self._deliver(link_points, out, shape, device=matrix_of(self.obj_frame_to_link_frame).device)

    def query_scene_collision_cost(self, scene, link_points, margin, links=None, cfg_begin=0, cfg_count=None):
        """Scene collision cost of configurations [cfg_begin, cfg_begin + cfg_count) and its twist gradient per
        sub-SDF.  The posed points x and the scene's (d, g) at them are those of `query_scene_clearance`; the margin m
        is rounded to fp32 as _collision_cost_margin does.  When d < m, with h = m - d and tau = 2h (g, x x g):
          - cost[a] += h^2
          - twist[a, i] -= tau.  The source moves and its point with it, so d changes by +g . (v + w x x); the scene
            is static and takes no term, so every other twist entry is 0.
        twist[a, s] is the derivative of the cost when sub-SDF s alone moves by an object-frame twist (v, w) about the
        origin: the convention of collision_cost, so RobotSDF.joint_gradient applies unchanged.  A configuration with
        nothing inside the margin costs exactly 0.

        The routes are those of `query_scene_clearance`; the composition route (`_composed_scene_collision_cost`) is
        the definition the fused one is checked against.  Both are deterministic, and the fused route's rows do not
        depend on the slab: a configuration split reproduces the full call bit for bit.  Returns flat (cfg_count,) /
        (cfg_count, S, 6) fp32 tensors on the GPU.  Raises ValueError before any device work on wrong shapes, a
        margin that is not finite, a scene with more than one pose, or an empty slab."""
        form = "scene-collision-cost query"
        K, mask = self._scene_args(scene, link_points, links, form)
        m = self._collision_cost_margin(margin)
        n_cfg, cfg_count = self._scene_slab(cfg_begin, cfg_count, form)
        S = len(self.sdfs)
        with _query_points(link_points) as (device, p):
            fused = self._scene_fused(scene, device)
            if fused is None:
                return self._composed_scene_collision_cost(scene, p, K, mask, m, cfg_begin, cfg_count)
            descs_arr, n_scene, sxf = fused
            inv = self._inv_xforms_on(device)
            cost = torch.empty(cfg_count, dtype=torch.float32, device=device)
            twist = torch.empty(cfg_count, S, 6, dtype=torch.float32, device=device)
            nat.check(nat.lib().pvb_composed_query_scene_collision_cost(
                descs_arr, n_scene, nat.ptr(sxf), nat.ptr(inv), S, n_cfg, cfg_begin, cfg_count, nat.ptr(p), K,
                (ctypes.c_uint8 * S)(*mask), m, nat.ptr(cost), nat.ptr(twist), nat.stream_ptr(device)),
                "pvb_composed_query_scene_collision_cost")
        return cost, twist

    def _composed_scene_collision_cost(self, scene, p, K, mask, m, cfg_begin, cfg_count):
        """query_scene_collision_cost by composition, the definition of its result: `_scene_chunks`, the
        `_hinge_terms`, and one sum per tested source (torch's sums are deterministic; scatter_add / index_add on
        CUDA are not)."""
        device = p.device
        srcs = [i for i, on in enumerate(mask) if on]
        cost = torch.zeros(cfg_count, dtype=torch.float64, device=device)
        twist = torch.zeros(cfg_count, len(self.sdfs), 6, dtype=torch.float64, device=device)
        for c0, cc, x, v, g in (self._scene_chunks(scene, p, K, srcs, cfg_begin, cfg_count) if srcs else ()):
            h, tau = self._hinge_terms(v, g, x, m)
            rs = slice(c0 - cfg_begin, c0 - cfg_begin + cc)
            cost[rs] = (h * h).sum(dim=(-2, -1))
            for pos, i in enumerate(srcs):
                twist[rs, i] = 0.0 - tau[:, pos].sum(dim=-2)       # +0, as the fused kernel, without terms
        return cost.float(), twist.float()

    def scene_collision_cost(self, scene, link_points, margin, links=None):
        """For every installed configuration, the soft collision cost of its tested links against a static scene and
        its twist gradient per sub-SDF: link_points [S, K, 3] holds K points of every sub-SDF in its own frame, links
        [S] bool says which sub-SDFs are tested (default: all), and every posed point within `margin` of `scene` (any
        ObjectFrameSDF in this composition's object frame) adds max(0, margin - d)^2.  Returns (cost [*A],
        twist_grad [*A, S, 6]) in link_points' dtype on the composition's device -- 0-d / [S, 6] without a
        configuration batch.  twist_grad[..., s, :] is the derivative of the cost when sub-SDF s alone moves by an
        object-frame twist (v, w) about the origin.  The definition and routes are those of
        `query_scene_collision_cost`.  Not a reference operator (an extension), and not autograd; raises ValueError
        before any device work on wrong shapes, a margin that is not finite or a scene with more than one pose."""
        shape = () if self.tsf_batch is None else tuple(int(a) for a in self.tsf_batch)
        out = self.query_scene_collision_cost(scene, link_points, margin, links)
        return self._deliver(link_points, out, shape, device=matrix_of(self.obj_frame_to_link_frame).device)

    def query_into(self, points_in_object_frame, targets, cfg_begin=0, cfg_count=None):
        """`query` whose result slab is stored by the kernel epilogue into several full-size result buffers at once
        (pvb_composed_query_multi): `targets` is a list of (val, grad) pairs, each a float32 tensor or a raw device
        address of a buffer holding ALL n_cfg * P results -- typically this rank's buffer and the peer-mapped buffers
        of the other ranks (distributed.PeerResult).  The slab lands at element cfg_begin * P of every buffer."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        if not 1 <= len(targets) <= nat.MAX_TARGETS:
            raise ValueError(f"between 1 and {nat.MAX_TARGETS} targets per launch, got {len(targets)}")
        with _query_points(points_in_object_frame) as (device, p):
            P = p.shape[0]
            descs_arr, needs_mesh = self._fused_descs(device, "query_into")
            arr = (nat.OutTarget * len(targets))()
            for t, (tv, tg) in enumerate(targets):
                for buf, per in ((tv, 1), (tg, 3)):
                    if torch.is_tensor(buf) and (buf.dtype != torch.float32 or not buf.is_contiguous()
                                                 or buf.numel() < per * n_cfg * P):
                        raise ValueError("targets must be contiguous float32 buffers of the full (n_cfg * P) result")
                arr[t].val = (tv.data_ptr() if torch.is_tensor(tv) else int(tv)) + 4 * cfg_begin * P
                arr[t].grad = (tg.data_ptr() if torch.is_tensor(tg) else int(tg)) + 12 * cfg_begin * P
            xf = self._xforms_on(device)
            nat.check(nat.lib().pvb_composed_query_multi(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg, cfg_begin,
                                                         cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                         ctypes.cast(arr, ctypes.c_void_p), len(targets), None,
                                                         nat.stream_ptr(device)), "pvb_composed_query_multi")

    def query_at(self, points_in_object_frame, val_addr, grad_addr, cfg_begin=0, cfg_count=None):
        """`query` that writes the slab into caller-owned device memory: val_addr / grad_addr are the addresses of
        FULL (n_cfg * P) value / gradient buffers (float32); the slab lands at element cfg_begin * P.  Single
        destination, the kernels' fastest store path -- what the copy-engine re-assembly (gather="dma") runs before it
        pushes the slab to the peers."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        with _query_points(points_in_object_frame) as (device, p):
            P = p.shape[0]
            descs_arr, needs_mesh = self._fused_descs(device, "query_at")
            xf = self._xforms_on(device)
            nat.check(nat.lib().pvb_composed_query(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg, cfg_begin,
                                                   cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                   int(val_addr) + 4 * cfg_begin * P, int(grad_addr) + 12 * cfg_begin * P,
                                                   None, nat.stream_ptr(device)), "pvb_composed_query")

    def query_multicast(self, points_in_object_frame, mc_val, mc_grad, cfg_begin=0, cfg_count=None):
        """`query` whose result slab leaves through an NVLS multicast mapping (pvb_composed_query_multicast): mc_val /
        mc_grad are the multicast device addresses of the full (n_cfg * P) value / gradient buffers; one multimem.st
        per 16-byte chunk lands in every bound GPU's copy."""
        S = len(self.sdfs)
        n_cfg, cfg_count = self._slab(cfg_begin, cfg_count)
        with _query_points(points_in_object_frame) as (device, p):
            P = p.shape[0]
            descs_arr, needs_mesh = self._fused_descs(device, "query_multicast")
            xf = self._xforms_on(device)
            nat.check(nat.lib().pvb_composed_query_multicast(descs_arr, S, int(needs_mesh), nat.ptr(xf), n_cfg, cfg_begin,
                                                             cfg_count, nat.ptr(p), P, nat.PVB_MESH_DEFAULT,
                                                             int(mc_val) + 4 * cfg_begin * P,
                                                             int(mc_grad) + 12 * cfg_begin * P,
                                                             nat.stream_ptr(device)), "pvb_composed_query_multicast")

    #: (configuration, point) pairs per chunk of `_generic_query` (bounds its per-sub-SDF temporaries)
    generic_chunk_pairs = 1 << 20

    def _generic_query(self, p, cfg_begin, cfg_count, n_cfg, return_which, paired=False):
        """Sub-SDFs without a native descriptor (user subclasses, nested compositions): per-SDF evaluation through
        their own __call__, with the transform and the running min still on the GPU, over chunks of at most
        `generic_chunk_pairs` pairs (one configuration at least), each written into its rows of the result.  paired:
        p holds cfg_count blocks of P points, block c for configuration cfg_begin + c only (query_paired)."""
        S = len(self.sdfs)
        device = p.device
        P = (p.shape[0] // cfg_count if cfg_count else 0) if paired else p.shape[0]
        M = self._xforms_on(device).reshape(S, n_cfg, 4, 4)
        best = torch.full((cfg_count * P,), float("inf"), dtype=torch.float32, device=device)
        bgrad = torch.zeros(cfg_count * P, 3, dtype=torch.float32, device=device)
        bwhich = torch.full((cfg_count * P,), -1, dtype=torch.int32, device=device)
        transform = nat.lib().pvb_transform_points_paired if paired else nat.lib().pvb_transform_points
        step = max(1, self.generic_chunk_pairs // max(P, 1))
        for c0 in range(0, cfg_count if P > 0 else 0, step):
            cc = min(step, cfg_count - c0)
            rows = slice(c0 * P, (c0 + cc) * P)
            pts = p[rows] if paired else p
            cbest, cgrad, cwhich = best[rows], bgrad[rows], bwhich[rows]        # views: the chunk's result rows
            for i, sdf in enumerate(self.sdfs):
                xf = M[i, cfg_begin + c0:cfg_begin + c0 + cc].contiguous()
                local = torch.empty(cc, P, 3, dtype=torch.float32, device=device)
                nat.check(transform(nat.ptr(xf), cc, nat.ptr(pts), P, nat.ptr(local), nat.stream_ptr(device)),
                          transform.__name__)
                v, g = sdf(local)
                v = v.to(device=device, dtype=torch.float32).reshape(-1)
                g = (g.to(device=device, dtype=torch.float32).reshape(cc, P, 3) @ xf[:, :3, :3]).reshape(-1, 3)
                better = (v < cbest) | (cwhich < 0)
                cbest.copy_(torch.where(better, v, cbest))
                cgrad.copy_(torch.where(better.unsqueeze(-1), g, cgrad))
                cwhich.masked_fill_(better, i)
        return (best, bgrad, bwhich) if return_which else (best, bgrad)

    #: host callers with at least this many result bytes get their result streamed out slab by slab
    host_result_pipeline_min_bytes = 64 << 20

    def _host_result_pipeline(self, points_in_object_frame):
        """Host points in, pinned host results out, for results so large that the device-to-host copy IS the call
        (C4: the PCIe copy takes many times the lookups): the configurations are queried in slabs (a first small one, then 64 at
        a time -- whole 32-configuration tiles) into one device buffer, and each slab starts its copy on a side stream
        as soon as its kernel has finished, so only the first slab's lookups are not hidden behind the copy.
        Returns None when the call does not qualify (then __call__ takes the plain path)."""
        if not (torch.is_tensor(points_in_object_frame) and points_in_object_frame.device.type == "cpu"
                and points_in_object_frame.dtype == torch.float32 and self.tsf_batch is not None):
            return None
        n_cfg = _config_count(self.tsf_batch)
        P = points_in_object_frame.numel() // 3
        if n_cfg < 64 or 16 * n_cfg * P < self.host_result_pipeline_min_bytes:
            return None
        device = nat.compute_device(None)
        if self._native_descs(device)[0] is None:
            return None
        with torch.cuda.device(device):
            cur = torch.cuda.current_stream(device)
            p = nat.as_f32_points(points_in_object_frame, device)
            val_d = torch.empty(n_cfg * P, dtype=torch.float32, device=device)
            grad_d = torch.empty(n_cfg * P, 3, dtype=torch.float32, device=device)
            val_h = torch.empty(n_cfg * P, dtype=torch.float32, pin_memory=True)
            grad_h = torch.empty(n_cfg * P, 3, dtype=torch.float32, pin_memory=True)
            s_out = getattr(self, "_s_out", None)
            if s_out is None or s_out.device != device:
                s_out = self._s_out = torch.cuda.Stream(device)
            b = 0
            while b < n_cfg:
                c = min(32 if b == 0 else 64, n_cfg - b)
                self.query_at(p, val_d.data_ptr(), grad_d.data_ptr(), b, c)
                done = torch.cuda.Event()
                done.record(cur)
                with torch.cuda.stream(s_out):
                    s_out.wait_event(done)
                    val_h[b * P:(b + c) * P].copy_(val_d[b * P:(b + c) * P], non_blocking=True)
                    grad_h[b * P:(b + c) * P].copy_(grad_d[b * P:(b + c) * P], non_blocking=True)
                b += c
            s_out.synchronize()        # the device buffers may be recycled from here on
        return val_h, grad_h

    def __call__(self, points_in_object_frame):
        pts_shape = tuple(points_in_object_frame.shape)
        piped = self._host_result_pipeline(points_in_object_frame)      # fp32 on the host already, like its points
        out = piped if piped is not None else self.query(points_in_object_frame)
        # configuration batch dims first, then the query points' batch dims (sdf.py:428-431); flat without a batch
        shape = (*self.tsf_batch, *pts_shape[:-1]) if self.tsf_batch is not None else (-1,)
        return self._deliver(points_in_object_frame, out, shape)


class OutOfBoundsStrategy(enum.Enum):
    LOOKUP_GT_SDF = 0
    BOUNDING_BOX = 1  # always under-approximates the SDF value, but more accurate than a sphere approximation


def _fp32_ceil(x):
    f = np.float32(x)
    return f if float(f) >= x else np.nextafter(f, np.float32(np.inf))


def _fp32_floor(x):
    f = np.float32(x)
    return f if float(f) <= x else np.nextafter(f, np.float32(-np.inf))


def fast_index_band(lo, hi, n):
    """(inv_res32, idx_certain) of one grid axis for the kernels' fast voxel index.

    The kernels estimate the index as q = (p - fp32(lo)) * inv_res32 in fp32 and accept rint(q) when
    |q - rint(q)| <= idx_certain; closer to a cell boundary than that, they evaluate the reference's formula
    round((p - lo) / res) exactly (fp64 or fp32, by the dtype torch infers for the range).  `err` bounds
    |q - (p - lo) / res| in cells: rounding lo to fp32, the fp32 subtraction, the rounding of inv_res32 and the fp32
    product, with a 4x safety factor; the identity "certain => same index" is checked on adversarial inputs by
    tests/test_index_band.py.  idx_certain = -1 sends every point down the exact path."""
    res = (hi - lo) / (n - 1) if n > 1 else float("inf")
    if not (n > 1 and math.isfinite(res) and res > 0):
        return 0.0, -1.0
    scale = max(abs(lo), abs(hi)) + (hi - lo)
    err = 4.0 * scale * 2.0 ** -24 / res + (n + 4) * 2.0 ** -22
    return float(np.float32(1.0 / res)), max(0.5 - (4.0 * err + 1e-6), -1.0)


def grid_prune_margin(values, lo, hi, bb):
    """Margin m such that a BOUNDING_BOX CachedSDF never returns less than dist(q, bb) - m, for ANY query q.

    The composed kernels skip a sub-SDF when dist(q, bb) - m already exceeds the running minimum, so the bound must
    be exact, not typical.  Out of range the value IS dist(q, bb) (sdf.py:555-571).  In range it is the table entry
    of the nearest voxel c, |q - c| <= half a cell diagonal, dist(., bb) is 1-Lipschitz, and t = max over the table
    of (dist(c, bb) - value(c))+ is measured on the table itself, so the bound holds for any table contents:
    value(c) >= dist(c, bb) - t >= dist(q, bb) - half_diag - t.  (1e-5 absorbs the kernels' fp32 arithmetic.)
    The same margin bounds the trilinear interpolant sum_i w_i value(c_i) over the 8 corners c_i of q's cell:
    value(c_i) >= dist(q, bb) - |q - c_i| - t, and sum_i w_i |q - c_i| <= sqrt(sum_i w_i |q - c_i|^2) (Jensen)
    = sqrt(sum_a r_a^2 f_a (1 - f_a)) <= half_diag, with r_a the cell size and f_a the fraction along axis a.
    values: (nx, ny, nz) table; lo / hi: per-axis range; bb: (3, 2) box the out-of-range rule measures against."""
    shape = tuple(values.shape)
    dev = values.device
    bbt = torch.as_tensor(np.asarray(bb), dtype=torch.float64, device=dev)
    per_axis = []
    for k in range(3):
        c = torch.linspace(lo[k], hi[k], shape[k], dtype=torch.float64, device=dev)
        per_axis.append(torch.clamp(torch.maximum(bbt[k, 0] - c, c - bbt[k, 1]), min=0))
    lb = torch.sqrt(per_axis[0][:, None, None] ** 2 + per_axis[1][None, :, None] ** 2 + per_axis[2][None, None, :] ** 2)
    t = float(torch.clamp(lb - values.double(), min=0).max())
    cell = [(hi[k] - lo[k]) / (shape[k] - 1) for k in range(3) if shape[k] > 1]
    return 0.5 * math.sqrt(sum(r * r for r in cell)) + t + 1e-5


class _TableStore:
    """The on-disk table cache of CachedSDF: one torch.save file holding {name: (val[nx,ny,nz], grad[Nvox,3])} for any
    number of objects -- the layout of the reference's sdf_cache.pkl (sdf.py:487-519), so existing files keep
    loading and files written here load in the reference."""

    def __init__(self, path):
        self.path = path
        self.entries = (torch.load(path) or {}) if os.path.exists(path) else {}

    def get(self, name):
        entry = self.entries.get(name)
        if entry is None:
            return None
        try:
            val, grad = entry
        except (ValueError, TypeError):
            logger.info("cached sdf invalid %s from %s, recreating", name, self.path)
            return None
        logger.info("cached sdf for %s loaded from %s", name, self.path)
        return val, grad

    def put(self, name, tables):
        self.entries[name] = tuple(t.cpu() for t in tables)
        torch.save(self.entries, self.path)
        logger.info("caching sdf for %s to %s", name, self.path)


class CachedSDF(ObjectFrameSDF):
    """SDF via nearest-voxel lookup of precomputed value and gradient tables."""

    def __init__(self, object_name, resolution, range_per_dim, gt_sdf: ObjectFrameSDF,
                 out_of_bounds_strategy=OutOfBoundsStrategy.BOUNDING_BOX,
                 device="cpu", clean_cache=False,
                 debug_check_sdf=False, cache_path="sdf_cache.pkl", interpolation="nearest"):
        """
        :param object_name: readable name of the object; combined with the resolution and range for the cache key
        :param resolution: side length of each voxel cell
        :param range_per_dim: (min, max) sequence for each dimension
        :param gt_sdf: ground truth SDF used to generate the cache and (optionally) for out-of-range queries
        :param out_of_bounds_strategy: LOOKUP_GT_SDF or BOUNDING_BOX (default)
        :param device: device results are returned on (the tables always live on the GPU)
        :param clean_cache: ignore an existing cache entry and recompute
        :param debug_check_sdf: check the generated tables against the ground truth SDF
        :param cache_path: torch.save file holding {name: (val[nx,ny,nz], grad[Nvox,3])}, same format as the reference
        :param interpolation: "nearest" (the reference's behaviour: nearest voxel value and stored gradient) or
        "trilinear" -- an EXTENSION that interpolates the value table trilinearly and returns the gradient of the
        interpolant (cell-wise finite differences); smoother, but O(resolution) away from the reference's output.
        Trilinear needs OutOfBoundsStrategy.BOUNDING_BOX.  It runs on the fused ComposedSDF / RobotSDF kernels like
        "nearest" does (point-serial robot kernel for <= 8 links, configuration-major and point-major kernels
        otherwise); batch_chamfer_dist evaluates a trilinear obj_sdf through its __call__
        """
        if interpolation not in ("nearest", "trilinear"):
            raise ValueError(f"interpolation must be 'nearest' or 'trilinear', got {interpolation!r}")
        self.interpolation = interpolation
        self.device = device
        self.voxels = None
        self.voxels_grad = None
        self.out_of_bounds_strategy = out_of_bounds_strategy
        self.gt_sdf = gt_sdf
        self.resolution = resolution
        self._cdev = nat.compute_device(device)

        span = np.asarray(range_per_dim, dtype=np.float64)
        cells = (span[:, 1] - span[:, 0]) // resolution
        if cells.min() < 10:
            logger.warning(f"Resolution {resolution} is too high for {object_name}, only getting {cells} voxels.")
        self.ranges = get_divisible_range_by_resolution(resolution, range_per_dim)
        range_per_dim = self.ranges
        # cache key: name, resolution and the snapped range, the format existing sdf_cache.pkl files were written with
        self.name = f"{object_name} {resolution} {tuple(self.ranges)}"
        self.debug_check_sdf = debug_check_sdf

        store = _TableStore(cache_path)
        tables = None if clean_cache else store.get(self.name)
        if tables is None:
            if gt_sdf is None:
                raise RuntimeError("Cached SDF did not find the cache and requires an initialize queryable SDF")
            tables = self._build_tables(gt_sdf)
            store.put(self.name, tables)
        cached_underlying_sdf, cached_underlying_sdf_grad = tables

        val = cached_underlying_sdf.to(device=self._cdev, dtype=torch.float32)
        grad = cached_underlying_sdf_grad.to(device=self._cdev, dtype=torch.float32).reshape(-1, 3)
        self._install_tables(val, grad)

    def _install_tables(self, val, grad, table=None):
        """Make val [nx, ny, nz] and grad [Nvox, 3] (fp32, on the compute device) the lookup tables over self.ranges,
        with surface_bounding_box() the box of the bounding-box rule, and build the fused kernels' descriptor.
        table: the [Nvox, 4] records of val and grad when the caller already holds them."""
        self.voxels = GridView(val, self.ranges, invalid_value=self._fallback_sdf_value_func)
        self.voxels_grad = grad
        # one 16-byte record {val, gx, gy, gz} per voxel: each lookup is a single 128-bit load
        self._table = torch.cat([val.reshape(-1, 1), grad], dim=1).contiguous() if table is None else table
        self.bb = self.surface_bounding_box().to(device=self._cdev)
        self._desc = self._make_desc()

    def _build_tables(self, gt_sdf):
        """(val[nx,ny,nz], grad[Nvox,3]): ONE batched ground-truth query over every voxel centre, on the GPU
        (the reference evaluates the same points through its CPU MeshSDF, sdf.py:502-505)."""
        coords, pts = get_coordinates_and_points_in_grid(self.resolution, self.ranges)
        sdf_val, sdf_grad = gt_sdf(pts.to(self._cdev))
        val = sdf_val.reshape([len(coord) for coord in coords])
        grad = sdf_grad.squeeze(0)
        if self.debug_check_sdf:
            debug_view = GridView(val, self.ranges, invalid_value=self._fallback_sdf_value_func)
            query = debug_view[pts.to(val.device)]
            assert torch.allclose(sdf_val.reshape(-1), query.reshape(-1))
        return val, grad

    # -- descriptor -----------------------------------------------------------------
    def _make_desc(self):
        d = nat.SdfDesc()
        d.kind = nat.PVB_KIND_GRID
        flags = 0
        d.table = self._table.data_ptr()
        shape = tuple(self.voxels.shape)
        lo = [float(min(r)) for r in self.ranges]
        hi = [float(max(r)) for r in self.ranges]
        fp32_index = range_dtype(self.ranges) == torch.float32
        if fp32_index:
            flags |= nat.PVB_GRID_INDEX_FP32
        bb = self.bb.detach().cpu().numpy().astype(np.float32)       # fp32 like the cast at sdf.py:556-557
        res_max = 0.0
        for k in range(3):
            d.dims[k] = shape[k]
            d.min64[k] = lo[k]
            d.res64[k] = (hi[k] - lo[k]) / (shape[k] - 1) if shape[k] > 1 else float("inf")
            lo32, hi32 = np.float32(lo[k]), np.float32(hi[k])
            d.min32[k] = float(lo32)
            d.res32[k] = float((hi32 - lo32) / np.float32(shape[k] - 1)) if shape[k] > 1 else float("inf")
            if fp32_index:
                d.valid_lo[k], d.valid_hi[k] = float(lo32), float(hi32)
            else:   # fp32 bounds equivalent to the fp64 comparison min <= double(p) <= max
                d.valid_lo[k], d.valid_hi[k] = float(_fp32_ceil(lo[k])), float(_fp32_floor(hi[k]))
            d.bb_min[k] = float(bb[k, 0])
            d.bb_max[k] = float(bb[k, 1])
            d.inv_res32[k], d.idx_certain[k] = fast_index_band(lo[k], hi[k], shape[k])
            if shape[k] > 1:
                res_max = max(res_max, d.res64[k])
        gt_native = None
        if self.out_of_bounds_strategy == OutOfBoundsStrategy.LOOKUP_GT_SDF:
            gt_native = self.gt_sdf.native_desc(self._cdev) if isinstance(self.gt_sdf, MeshSDF) else None
            if gt_native is not None:
                flags |= nat.PVB_GRID_OOB_GT
                self.gt_sdf.obj_factory._fill_mesh_part(d, self.gt_sdf.obj_factory._device_state(self._cdev))
                flags |= d.flags & nat.PVB_MESH_CLOSED
                for k in range(3):       # _fill_mesh_part rewrote the box from the mesh; keep self.bb
                    d.bb_min[k] = float(bb[k, 0])
                    d.bb_max[k] = float(bb[k, 1])
        self._gt_in_kernel = gt_native is not None
        # Pruning bound for the composed kernels: table value at the nearest voxel of q is never below
        # aabb_distance(q) - prune_margin.  t is measured on the table itself, so the bound holds for any table.
        # It holds for the trilinear interpolant as well (grid_prune_margin).
        if self.out_of_bounds_strategy == OutOfBoundsStrategy.BOUNDING_BOX:
            margin = grid_prune_margin(self.voxels.raw_data.reshape(shape), lo, hi, bb)
            if math.isfinite(margin):
                d.prune_margin = margin
                flags |= nat.PVB_GRID_PRUNE_OK
        if self.interpolation == "trilinear":
            if self.out_of_bounds_strategy != OutOfBoundsStrategy.BOUNDING_BOX:
                raise ValueError("interpolation='trilinear' supports OutOfBoundsStrategy.BOUNDING_BOX only")
            flags |= nat.PVB_GRID_TRILINEAR
        d.flags = flags
        return d

    def native_desc(self, device):
        """Descriptor for the fused kernels on `device` (None: not queryable there natively).  With
        interpolation="trilinear" it carries PVB_GRID_TRILINEAR, which pvb_grid_lookup and the composed kernels
        honour and pvb_chamfer rejects."""
        device = nat.compute_device(device)
        if device != self._cdev:
            return None
        if self.out_of_bounds_strategy == OutOfBoundsStrategy.LOOKUP_GT_SDF and not self._gt_in_kernel:
            return None
        return self._desc

    def surface_bounding_box(self, **kwargs):
        return self.gt_sdf.surface_bounding_box(**kwargs)

    def _fallback_sdf_value_func(self, *args, **kwargs):
        sdf_val, _ = self.gt_sdf(*args, **kwargs)
        return sdf_val.to(device=self._cdev)

    def _lookup(self, points, want_val=True, want_outside=False, surface_level=0., want_index=False):
        device = self._cdev
        with nat.on_device(device):
            p = nat.as_f32_points(points, device)
            n = p.shape[0]
            val = torch.empty(n, dtype=torch.float32, device=device) if want_val else None
            grad = torch.empty(n, 3, dtype=torch.float32, device=device) if want_val else None
            outside = torch.empty(n, dtype=torch.uint8, device=device) if want_outside else None
            index = torch.empty(n, dtype=torch.int64, device=device) if want_index else None
            L = nat.lib()
            if self.interpolation == "trilinear" and (want_outside or want_index):
                # keys / occupancy always follow the reference's nearest-voxel rule; values come from the interpolant
                plain = self._desc.copy()
                plain.flags &= ~nat.PVB_GRID_TRILINEAR
                nat.check(L.pvb_grid_lookup(ctypes.byref(plain), nat.ptr(p), n, None, None, nat.ptr(outside),
                                            float(surface_level), nat.ptr(index), nat.stream_ptr(device)),
                          "pvb_grid_lookup")
                if want_val:
                    nat.check(L.pvb_grid_lookup(ctypes.byref(self._desc), nat.ptr(p), n, nat.ptr(val), nat.ptr(grad),
                                                None, 0.0, None, nat.stream_ptr(device)), "pvb_grid_lookup")
            else:
                nat.check(L.pvb_grid_lookup(ctypes.byref(self._desc), nat.ptr(p), n, nat.ptr(val), nat.ptr(grad),
                                            nat.ptr(outside), float(surface_level), nat.ptr(index),
                                            nat.stream_ptr(device)), "pvb_grid_lookup")
        return p, val, grad, outside, index

    #: host batches at least this large are streamed through the GPU in chunks (_HostChunkStream: copy-in / lookup /
    #: copy-out overlapped on three streams); smaller ones take one H2D copy, one launch, one D2H copy
    host_pipeline_min_points = 1 << 22
    host_pipeline_chunk = 1 << 21

    def _host_pipeline(self, points):
        """Host tensor in, pinned host (values, gradients) out through the chunk pipeline."""
        device = self._cdev
        st = getattr(self, "_pipe_state", None)
        if st is None or st.chunk != self.host_pipeline_chunk or st.device != device:
            st = self._pipe_state = _HostChunkStream(device, self.host_pipeline_chunk, ((), (3,)))
        L = nat.lib()

        def launch(d_in, m, d_out):
            nat.check(L.pvb_grid_lookup(ctypes.byref(self._desc), nat.ptr(d_in), m, nat.ptr(d_out[0]), nat.ptr(d_out[1]),
                                        None, 0.0, None, nat.stream_ptr(device)), "pvb_grid_lookup")

        val_h, grad_h = st.run(points, launch)
        return val_h, grad_h

    def __call__(self, points_in_object_frame):
        lead = tuple(points_in_object_frame.shape[:-1])
        gt_outside_kernel = (self.out_of_bounds_strategy == OutOfBoundsStrategy.LOOKUP_GT_SDF
                             and not self._gt_in_kernel)
        if (torch.is_tensor(points_in_object_frame) and points_in_object_frame.device.type == "cpu"
                and torch.device(self.device).type == "cpu" and not gt_outside_kernel and not self.debug_check_sdf
                and self.interpolation == "nearest"
                and points_in_object_frame.numel() // 3 >= self.host_pipeline_min_points):
            val, grad = self._host_pipeline(points_in_object_frame)
            dtype = points_in_object_frame.dtype
            if dtype != torch.float32:
                val, grad = val.to(dtype), grad.to(dtype)
            return val.reshape(lead), grad.reshape(*lead, 3)
        p, val, grad, _, index = self._lookup(points_in_object_frame, want_index=gt_outside_kernel or
                                              self.debug_check_sdf)
        if gt_outside_kernel:
            # ground-truth SDF without a native descriptor: evaluate it on the out-of-range points (host-synchronous)
            oob = index < 0
            if oob.any():
                v, g = self.gt_sdf(p[oob])
                val[oob] = v.to(device=p.device, dtype=torch.float32)
                grad[oob] = g.to(device=p.device, dtype=torch.float32)
        if self.debug_check_sdf:
            inb = index >= 0
            if self.out_of_bounds_strategy == OutOfBoundsStrategy.BOUNDING_BOX and (~inb).any():
                val_gt, grad_gt = self.gt_sdf(p[~inb])
                assert torch.all(val_gt - val[~inb] > -1e-6)     # under-approximates (sdf.py:578)
                cos = torch.cosine_similarity(grad_gt, grad[~inb], dim=-1)
                assert torch.all(cos > 0.7) and cos.mean() > 0.95
            val_gt = self._fallback_sdf_value_func(p)
            assert torch.all((torch.abs(val - val_gt) < self.resolution)[inb])
        dtype = points_in_object_frame.dtype if torch.is_tensor(points_in_object_frame) else torch.float
        return (nat.deliver(val, self.device, dtype).reshape(lead),
                nat.deliver(grad, self.device, dtype).reshape(*lead, 3))

    def outside_surface(self, points_in_object_frame, surface_level=0):
        lead = tuple(points_in_object_frame.shape[:-1])
        _, _, _, outside, _ = self._lookup(points_in_object_frame, want_val=False, want_outside=True,
                                           surface_level=surface_level)
        return nat.deliver(outside, self.device, torch.bool).reshape(lead)

    def voxel_keys(self, points_in_object_frame):
        """Ravelled nearest-voxel key per point (int64, -1 where out of the cached range): the index/occupancy
        quantity that must be bit-exact against the reference (sdf.py:537-540)."""
        lead = tuple(points_in_object_frame.shape[:-1])
        _, _, _, _, index = self._lookup(points_in_object_frame, want_val=False, want_index=True)
        return nat.deliver(index, self.device).reshape(lead)

    def get_voxel_view(self, voxels: VoxelGrid = None, dtype=torch.float, device='cpu') -> GridView:
        if voxels is None:
            return self.voxels
        pts = voxels.get_voxel_center_points()
        sdf_val, sdf_grad = self.gt_sdf(pts.unsqueeze(0))
        sdf_val = sdf_val.to(device=self._cdev)
        cached_underlying_sdf = sdf_val.reshape([len(coord) for coord in voxels.coords])
        return GridView(cached_underlying_sdf, voxels.range_per_dim, invalid_value=self._fallback_sdf_value_func)


def _occupancy_u8(occupancy):
    """occupancy (bool / uint8 tensor or array [nx, ny, nz]) as a contiguous uint8 tensor on its own device, checked
    for the shape and the two states pvb_occupancy_sdf needs."""
    occ = occupancy if torch.is_tensor(occupancy) else torch.as_tensor(np.asarray(occupancy))
    if occ.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"occupancy must be bool or uint8, got {occ.dtype}")
    if occ.dim() != 3 or not all(2 <= n <= 1024 for n in occ.shape):
        raise ValueError(f"occupancy must be [nx, ny, nz] with 2..1024 voxels per axis, got {tuple(occ.shape)}")
    occ = occ.contiguous()
    occ = occ.view(torch.uint8) if occ.dtype == torch.bool else occ
    n_occ = int(torch.count_nonzero(occ))
    if n_occ == 0 or n_occ == occ.numel():
        raise ValueError("occupancy needs at least one occupied and one free voxel: a grid of one state has no "
                         "distance field")
    return occ


def _occupancy_sdf(occ, resolution, sqdist=False, site=False, table=False):
    """pvb_occupancy_sdf over the uint8 grid `occ` (on its CUDA device): the requested outputs, in the order
    (sqdist int32 [nx, ny, nz], site int32 [nx, ny, nz], table fp32 [Nvox, 4])."""
    dev = occ.device
    dims = (ctypes.c_int32 * 3)(*occ.shape)
    L = nat.lib()
    with nat.on_device(dev):
        ws = torch.empty(int(L.pvb_occupancy_sdf_workspace(dims)), dtype=torch.uint8, device=dev)
        outs = [torch.empty(occ.shape, dtype=torch.int32, device=dev) if sqdist else None,
                torch.empty(occ.shape, dtype=torch.int32, device=dev) if site else None,
                torch.empty(occ.numel(), 4, dtype=torch.float32, device=dev) if table else None]
        nat.check(L.pvb_occupancy_sdf(nat.ptr(occ), dims, float(resolution), nat.ptr(ws), ws.numel(),
                                      *[nat.ptr(t) for t in outs], nat.stream_ptr(dev)), "pvb_occupancy_sdf")
    return tuple(t for t in outs if t is not None)


def occupancy_distance_transform(occupancy):
    """Exact squared Euclidean distance transform of an occupancy grid, with the site of every voxel.

    occupancy: bool / uint8 [nx, ny, nz] (nonzero = occupied), 2..1024 voxels per axis, with both states present.
    Returns (D, site) on the occupancy's device: D int32 [nx, ny, nz] is the squared distance, in cell units, from each
    voxel to the nearest voxel of the other state (free voxels measure to occupied ones and occupied voxels to free
    ones); site int64 [nx, ny, nz] is that voxel's flat C-order index, the smallest index among equally near ones --
    the role of scipy.ndimage.distance_transform_edt's return_indices.  Computed on the GPU, in integer arithmetic."""
    src = occupancy.device if torch.is_tensor(occupancy) else torch.device("cpu")
    occ = _occupancy_u8(occupancy)
    d, site = _occupancy_sdf(occ.to(nat.compute_device(src)), 1.0, sqdist=True, site=True)
    return nat.deliver(d, src), nat.deliver(site.long(), src)


class OccupancySDF(CachedSDF):
    """Signed distance table of an occupancy grid, built on the GPU by an exact Euclidean distance transform.

    Each voxel's value is its distance to the nearest voxel of the other state, minus half a cell, negative inside:
    val = sigma r (sqrt(D) - 1/2) with sigma = -1 for an occupied voxel, so the zero level lies on the faces between
    occupied and free voxels, and the gradient is sigma (c - site) / sqrt(D).  The table is a CachedSDF table on the
    same lattice (range snapped by get_divisible_range_by_resolution, voxel i at lo + i r), looked up with the
    bounding-box rule outside the range, the box being that of the occupied voxel centres widened by r / 2.  So an
    OccupancySDF serves everywhere a CachedSDF does: as a scene (RobotSDF.scene_clearance), as a ComposedSDF
    sub-SDF and as batch_chamfer_dist's obj_sdf, on the fused kernels.

    A cloud sampled on surfaces marks only the surfaces occupied: the inside of a solid stays free and its values are
    positive there.  A signed interior needs filled occupancy.

    :param occupancy: VoxelGrid (its resolution and range are used), or a bool / uint8 tensor [nx, ny, nz] together
        with resolution and range_per_dim; its shape must be the lattice those imply.  Both states must be present.
    :param interpolation: "nearest" or "trilinear", as for CachedSDF
    :param device: device results are returned on (the tables always live on the GPU)
    There is no ground-truth SDF and no cache file; the bounding-box rule is the only out-of-range rule."""

    def __init__(self, occupancy, resolution=None, range_per_dim=None, interpolation="nearest", device="cpu"):
        if interpolation not in ("nearest", "trilinear"):
            raise ValueError(f"interpolation must be 'nearest' or 'trilinear', got {interpolation!r}")
        if isinstance(occupancy, VoxelGrid):
            if resolution is not None or range_per_dim is not None:
                raise ValueError("a VoxelGrid carries its own resolution and range; pass neither")
            resolution, range_per_dim, occupancy = occupancy.resolution, occupancy.range_per_dim, \
                occupancy.get_voxel_values()
        elif resolution is None or range_per_dim is None:
            raise ValueError("an occupancy tensor needs resolution and range_per_dim")
        if not (math.isfinite(float(resolution)) and float(resolution) > 0):
            raise ValueError(f"resolution must be finite and positive, got {resolution}")
        self.interpolation = interpolation
        self.device = device
        self.out_of_bounds_strategy = OutOfBoundsStrategy.BOUNDING_BOX
        self.gt_sdf = None
        self.resolution = resolution
        self.debug_check_sdf = False
        self.ranges = get_divisible_range_by_resolution(resolution, range_per_dim)
        self.name = f"occupancy {resolution} {tuple(self.ranges)}"
        coords, _ = get_coordinates_and_points_in_grid(resolution, self.ranges, get_points=False)
        shape = tuple(len(c) for c in coords)
        if tuple(occupancy.shape) != shape:
            raise ValueError(f"occupancy of shape {tuple(occupancy.shape)} does not match the lattice of resolution "
                             f"{resolution} over {self.ranges}, {shape}")
        occ = _occupancy_u8(occupancy)
        self._cdev = nat.compute_device(device)
        occ = occ.to(self._cdev)
        self.occupancy = occ.view(torch.bool)
        (table,) = _occupancy_sdf(occ, resolution, table=True)
        box = np.empty((3, 2))
        for k in range(3):
            idx = torch.nonzero(self.occupancy.any(dim=tuple(a for a in range(3) if a != k))).reshape(-1)
            lo = float(min(self.ranges[k]))
            box[k] = (lo + int(idx[0]) * resolution - 0.5 * resolution, lo + int(idx[-1]) * resolution + 0.5 * resolution)
        self._surface_box = box
        self._install_tables(table[:, 0].reshape(shape).contiguous(), table[:, 1:].contiguous(), table=table)

    @classmethod
    def from_points(cls, points, resolution, range_per_dim, interpolation="nearest", device="cpu"):
        """OccupancySDF of the voxels the points [N, 3] fall into (pvb_voxel_scatter, as
        VoxelGrid(resolution, range_per_dim, dtype=torch.bool)[points] = True); points outside the range are dropped."""
        cdev = nat.compute_device(device)
        grid = VoxelGrid(resolution, range_per_dim, dtype=torch.bool, device=cdev)
        grid[nat.as_f32_points(points, cdev)] = True
        return cls(grid, interpolation=interpolation, device=device)

    @classmethod
    def from_depth(cls, depth, K, cam_to_world, resolution, range_per_dim, unknown="occupied", max_depth=math.inf,
                   free_margin=None, interpolation="nearest", device="cpu"):
        """OccupancySDF of the scene that depth images see (depth_occupancy's state grid).

        unknown="occupied" (the default) counts the voxels no view saw as occupied, as planners do: solids are
        negative inside.  unknown="free" counts only the voxels a valid pixel's point falls into as occupied, which
        gives the same occupancy and table as from_points(points[valid]) with the same resolution and range.
        The other arguments are depth_occupancy's, plus interpolation and device as for OccupancySDF."""
        if unknown not in ("occupied", "free"):
            raise ValueError(f"unknown must be 'occupied' or 'free', got {unknown!r}")
        if interpolation not in ("nearest", "trilinear"):
            raise ValueError(f"interpolation must be 'nearest' or 'trilinear', got {interpolation!r}")
        views = _depth_views(depth, K, cam_to_world, max_depth)
        lattice = _depth_lattice(resolution, range_per_dim, free_margin)
        cdev = nat.compute_device(device)
        state = _depth_state(views, lattice, cdev)
        grid = VoxelGrid(resolution, range_per_dim, dtype=torch.bool, device=cdev)
        grid.get_voxel_values().copy_(state == 1 if unknown == "free" else state != 0)
        return cls(grid, interpolation=interpolation, device=device)

    @classmethod
    def from_rays(cls, points, origins, resolution, range_per_dim, unknown="occupied", max_range=math.inf,
                  free_margin=None, interpolation="nearest", device="cpu"):
        """OccupancySDF of the scene that point clouds taken from known sensor origins see (ray_occupancy's state
        grid), under from_depth's rules: unknown="occupied" (the default) counts the voxels no ray passed through as
        occupied; unknown="free" counts only the voxels a valid ray's return falls into, which gives the occupancy
        and table of from_points(the returns of the valid rays).  The other arguments are ray_occupancy's, plus
        interpolation and device as for OccupancySDF."""
        if unknown not in ("occupied", "free"):
            raise ValueError(f"unknown must be 'occupied' or 'free', got {unknown!r}")
        if interpolation not in ("nearest", "trilinear"):
            raise ValueError(f"interpolation must be 'nearest' or 'trilinear', got {interpolation!r}")
        rays = _rays(points, origins, max_range)
        lattice = _depth_lattice(resolution, range_per_dim, free_margin)
        cdev = nat.compute_device(device)
        state = _ray_state(rays, lattice, cdev)
        grid = VoxelGrid(resolution, range_per_dim, dtype=torch.bool, device=cdev)
        grid.get_voxel_values().copy_(state == 1 if unknown == "free" else state != 0)
        return cls(grid, interpolation=interpolation, device=device)

    def surface_bounding_box(self, padding=0., padding_ratio=0.):
        """The box of the occupied voxel centres widened by half a cell, inflated by padding + padding_ratio * extent
        (fp64)."""
        box = self._surface_box.copy()
        grow = padding + padding_ratio * (box[:, 1] - box[:, 0])
        box[:, 0] -= grow
        box[:, 1] += grow
        return torch.from_numpy(box)

    def _fallback_sdf_value_func(self, points, *args, **kwargs):
        """Values outside the range (GridView lookups of self.voxels): the bounding-box rule of __call__."""
        return self._lookup(points)[1]

    def get_voxel_view(self, voxels: VoxelGrid = None, dtype=torch.float, device='cpu') -> GridView:
        if voxels is None:
            return self.voxels
        return ObjectFrameSDF.get_voxel_view(self, voxels, dtype=dtype, device=device)


# ---------------------------------------------------------------- depth images
class _DepthViews(NamedTuple):
    depth: torch.Tensor         # fp32 [V, H, W], on the caller's device
    intrinsics: np.ndarray      # fp32 [V, 4] = fx, fy, cx, cy
    cam_to_world: torch.Tensor  # fp64 [V, 4, 4], host
    max_depth: float


def _depth_views(depth, K, cam_to_world, max_depth):
    """Check depth_to_points' / depth_occupancy's view arguments (ValueError, before any device work)."""
    d = depth if torch.is_tensor(depth) else torch.as_tensor(np.asarray(depth))
    if d.dtype != torch.float32:
        raise ValueError(f"depth must be float32 metres, got {d.dtype}")
    if d.dim() != 3 or not (1 <= d.shape[0] <= 64 and 1 <= d.shape[1] <= 32768 and 1 <= d.shape[2] <= 32768):
        raise ValueError(f"depth must be [V, H, W] with V in 1..64 and H, W in 1..32768, got {tuple(d.shape)}")
    V = d.shape[0]
    k = torch.as_tensor(np.asarray(K.detach().cpu() if torch.is_tensor(K) else K, dtype=np.float64))
    if k.shape == (3, 3):
        k = k.expand(V, 3, 3)
    if k.shape != (V, 3, 3):
        raise ValueError(f"K must be [3, 3] or [V, 3, 3] with V = {V}, got {tuple(k.shape)}")
    if (k[:, 0, 1] != 0).any() or (k[:, 1, 0] != 0).any() or (k[:, 2] != torch.tensor([0., 0., 1.],
                                                                                         dtype=k.dtype)).any():
        raise ValueError("K must be a pinhole matrix [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]: no skew, bottom row 0 0 1")
    fx, fy, cx, cy = k[:, 0, 0], k[:, 1, 1], k[:, 0, 2], k[:, 1, 2]
    if not (torch.isfinite(k).all() and (fx > 0).all() and (fy > 0).all()):
        raise ValueError("K must be finite, with positive focal lengths")
    intr = torch.stack([fx, fy, cx, cy], 1).numpy().astype(np.float32)
    if not (np.isfinite(intr).all() and (intr[:, :2] > 0).all()):
        raise ValueError("K's entries must be finite and its focal lengths positive in float32")
    m = matrix_of(cam_to_world) if isinstance(cam_to_world, Transform3d) else cam_to_world
    m = torch.as_tensor(np.asarray(m.detach().cpu() if torch.is_tensor(m) else m, dtype=np.float64))
    if m.shape != (V, 4, 4):
        raise ValueError(f"cam_to_world must hold one 4x4 transform per view, [{V}, 4, 4], got {tuple(m.shape)}")
    R = m[:, :3, :3]
    if not (torch.isfinite(m).all() and (m[:, 3] == torch.tensor([0., 0., 0., 1.], dtype=m.dtype)).all()
            and (R @ R.transpose(1, 2) - torch.eye(3, dtype=m.dtype)).abs().max() < 1e-5
            and (torch.linalg.det(R) > 0).all()):
        raise ValueError("cam_to_world must be finite rigid transforms: a rotation, a translation, bottom row 0 0 0 1")
    max_depth = float(max_depth)
    if not max_depth > 0:
        raise ValueError(f"max_depth must be positive (+inf allowed), got {max_depth}")
    return _DepthViews(d, intr, m, max_depth)


def _depth_lattice(resolution, range_per_dim, free_margin):
    """(resolution, free_margin) checked, free_margin defaulting to half a cell diagonal, sqrt(3) r / 2; the lattice
    must hold 2..1024 voxels per axis."""
    resolution = float(resolution)
    if not (math.isfinite(resolution) and resolution > 0):
        raise ValueError(f"resolution must be finite and positive, got {resolution}")
    margin = math.sqrt(3.0) * resolution / 2 if free_margin is None else float(free_margin)
    if not (math.isfinite(margin) and margin >= 0):
        raise ValueError(f"free_margin must be finite and non-negative, got {free_margin}")
    coords, _ = get_coordinates_and_points_in_grid(resolution, get_divisible_range_by_resolution(resolution,
                                                                                                 range_per_dim),
                                                   get_points=False)
    shape = tuple(len(c) for c in coords)
    if len(shape) != 3 or not all(2 <= n <= 1024 for n in shape):
        raise ValueError(f"the lattice of resolution {resolution} over {range_per_dim} must hold 2..1024 voxels per "
                         f"axis, got {shape}")
    return resolution, range_per_dim, margin


def _depth_points(views, d, cdev):
    """pvb_depth_points of the depth images d (views.depth on cdev): (points fp32 [V, H, W, 3], valid bool
    [V, H, W]), both on cdev."""
    V, H, W = d.shape
    c2w = (ctypes.c_float * (12 * V))(*views.cam_to_world[:, :3].to(torch.float32).reshape(-1).tolist())
    intr = (ctypes.c_float * (4 * V))(*views.intrinsics.reshape(-1).tolist())
    with nat.on_device(cdev):
        out = torch.empty(V, H, W, 3, dtype=torch.float32, device=cdev)
        nat.check(nat.lib().pvb_depth_points(nat.ptr(d), V, H, W, intr, c2w, views.max_depth, nat.ptr(out),
                                             nat.stream_ptr(cdev)), "pvb_depth_points")
    valid = (d > 0) & (d <= views.max_depth) & torch.isfinite(d)
    return out, valid


def _depth_state(views, lattice, cdev):
    """The uint8 state grid [nx, ny, nz] on cdev: pvb_depth_carve writes 0 (free) or 2 (unknown), then the scatter of
    the valid points (VoxelGrid(...)[points] = True, pvb_voxel_scatter) writes 1 (occupied)."""
    resolution, range_per_dim, margin = lattice
    d = views.depth.to(cdev).contiguous()
    points, valid = _depth_points(views, d, cdev)
    V, H, W = d.shape
    grid = VoxelGrid(resolution, range_per_dim, dtype=torch.bool, device=cdev)
    state = grid.get_voxel_values().view(torch.uint8)
    w2c = (ctypes.c_float * (12 * V))(*invert_rigid(views.cam_to_world)[:, :3].to(torch.float32).reshape(-1).tolist())
    intr = (ctypes.c_float * (4 * V))(*views.intrinsics.reshape(-1).tolist())
    lo = (ctypes.c_float * 3)(*[float(min(r)) for r in grid.range_per_dim])
    dims = (ctypes.c_int32 * 3)(*state.shape)
    with nat.on_device(cdev):
        nat.check(nat.lib().pvb_depth_carve(nat.ptr(d), V, H, W, intr, w2c, views.max_depth, margin, lo, resolution,
                                            dims, nat.ptr(state), nat.stream_ptr(cdev)), "pvb_depth_carve")
    grid[points[valid]] = True
    return state


def depth_to_points(depth, K, cam_to_world, max_depth=math.inf):
    """Back-project depth images to world points on the GPU (pvb_depth_points).

    depth: float32 [V, H, W], z-depth in metres, row-major; V up to 64.  K: [3, 3] or [V, 3, 3] pinhole intrinsics
    (fx = K[0, 0], fy = K[1, 1], cx = K[0, 2], cy = K[1, 2]; any skew or a bottom row other than 0 0 1 is refused).
    cam_to_world: Transform3d or [V, 4, 4] rigid camera-to-world transforms.  The camera follows the OpenCV
    convention (x right, y down, z forward) with pixel (row i, column j) centred at u = j, v = i.
    A pixel is valid when its depth d is finite, d > 0 and d <= max_depth; write 0 where a pixel should be ignored
    (the robot's own body, say).  A valid pixel gives p_cam = ((j - cx) d / fx, (i - cy) d / fy, d) and the point
    cam_to_world p_cam, in fp32 (the operation order is in include/pvb.h); an invalid one gives NaN.
    Returns (points float32 [V, H, W, 3], valid bool [V, H, W]) on depth's device."""
    views = _depth_views(depth, K, cam_to_world, max_depth)
    src = views.depth.device
    cdev = nat.compute_device(src)
    points, valid = _depth_points(views, views.depth.to(cdev).contiguous(), cdev)
    return nat.deliver(points, src), nat.deliver(valid, src)


def depth_occupancy(depth, K, cam_to_world, resolution, range_per_dim, max_depth=math.inf, free_margin=None):
    """Fuse depth images into an occupancy state grid on the GPU (pvb_depth_carve, then pvb_voxel_scatter).

    The grid is the lattice OccupancySDF uses (range snapped by get_divisible_range_by_resolution, voxel i centred at
    lo + i r in fp32), 2..1024 voxels per axis.  The depth, K, cam_to_world and max_depth arguments are
    depth_to_points'.  Each voxel is
      1 occupied  when a valid pixel's back-projected point falls into it (the VoxelGrid scatter from_points uses);
      0 free      otherwise, when any view says free: the voxel centre c is in front of the camera, its pixel
                  (floor(fy y / z + cy + 0.5), floor(fx x / z + cx + 0.5)) of c's camera coordinates (x, y, z) lies in
                  the image and is valid, and z < d - free_margin;
      2 unknown   otherwise: no view saw it.
    free_margin defaults to sqrt(3) r / 2, half a cell diagonal, so that a voxel is carved only when its whole cube
    lies in front of the surface along that pixel's ray.  The result depends on neither the view order nor the thread
    order.  Returns uint8 [nx, ny, nz] on depth's device."""
    views = _depth_views(depth, K, cam_to_world, max_depth)
    lattice = _depth_lattice(resolution, range_per_dim, free_margin)
    src = views.depth.device
    return nat.deliver(_depth_state(views, lattice, nat.compute_device(src)), src)


# ---------------------------------------------------------------- ray-cast point clouds
class _Rays(NamedTuple):
    points: torch.Tensor        # fp32 [n_rays, 3], on the caller's device
    origins: torch.Tensor       # fp32 [V, 3], on points' device
    per_origin: int             # rays per origin: N
    max_range: float


def _rays(points, origins, max_range):
    """Check ray_occupancy's / integrate_points' ray arguments (ValueError, before any device work): float32 points
    [N, 3] with origins [3], or [V, N, 3] with origins [V, 3]."""
    p = points if torch.is_tensor(points) else torch.as_tensor(np.asarray(points))
    o = origins if torch.is_tensor(origins) else torch.as_tensor(np.asarray(origins))
    if p.dtype != torch.float32 or o.dtype != torch.float32:
        raise ValueError(f"points and origins must be float32, got {p.dtype} and {o.dtype}")
    shapes = tuple(p.shape), tuple(o.shape)
    if p.dim() == 2 and o.dim() == 1:
        p, o = p.unsqueeze(0), o.unsqueeze(0)
    if p.dim() != 3 or p.shape[2] != 3 or p.shape[0] < 1 or p.shape[1] < 1 or tuple(o.shape) != (p.shape[0], 3):
        raise ValueError(f"points must be [N, 3] with origins [3], or [V, N, 3] with origins [V, 3], N, V >= 1; got "
                         f"{shapes[0]} and {shapes[1]}")
    if p.shape[0] * p.shape[1] >= 2 ** 31:
        raise ValueError(f"at most 2^31 - 1 rays per call, got {p.shape[0] * p.shape[1]}")
    max_range = float(max_range)
    if not max_range > 0:
        raise ValueError(f"max_range must be positive (+inf allowed), got {max_range}")
    return _Rays(p.reshape(-1, 3), o.to(p.device), int(p.shape[1]), max_range)


def _ray_carve(rays, margin, lo, resolution, dims, marks, cdev):
    """pvb_ray_carve of the rays into the uint8 marks on cdev; returns out_points (NaN for an invalid ray)."""
    pts = rays.points.to(cdev).contiguous()
    org = rays.origins.to(cdev).contiguous()
    with nat.on_device(cdev):
        out = torch.empty_like(pts)
        nat.check(nat.lib().pvb_ray_carve(nat.ptr(pts), pts.shape[0], rays.per_origin, nat.ptr(org), rays.max_range,
                                          margin, lo, resolution, dims, nat.ptr(marks), nat.ptr(out),
                                          nat.stream_ptr(cdev)), "pvb_ray_carve")
    return out


def _ray_state(rays, lattice, cdev):
    """The uint8 state grid [nx, ny, nz] on cdev: 2 - marks after pvb_ray_carve writes 2 on the free voxels and the
    scatter of the valid returns (VoxelGrid(...)[points] = True, pvb_voxel_scatter) writes 1."""
    resolution, range_per_dim, margin = lattice
    grid = VoxelGrid(resolution, range_per_dim, dtype=torch.bool, device=cdev)
    marks = grid.get_voxel_values().view(torch.uint8)
    lo = (ctypes.c_float * 3)(*[float(min(r)) for r in grid.range_per_dim])
    out = _ray_carve(rays, margin, lo, resolution, (ctypes.c_int32 * 3)(*marks.shape), marks, cdev)
    grid[out] = True                    # an invalid ray's NaN point falls into no voxel
    return 2 - marks


def ray_occupancy(points, origins, resolution, range_per_dim, max_range=math.inf, free_margin=None):
    """Fuse point clouds taken from known sensor origins into an occupancy state grid on the GPU (pvb_ray_carve, then
    pvb_voxel_scatter), as OctoMap's insertPointCloud does: each ray is walked from its origin towards its return.

    points: float32 [N, 3] with origins [3] (one scan), or [V, N, 3] with origins [V, 3] (V scans), world frame; any
    other dtype or shape raises ValueError.  A ray is valid when its six coordinates are finite and its length l
    satisfies 0 < l <= max_range: NaN rows pad ragged scans, l = 0 is a "no return", and returns beyond max_range are
    dropped.  An invalid ray says nothing.  The grid is depth_occupancy's lattice (range snapped by
    get_divisible_range_by_resolution, voxel i centred at lo + i r), 2..1024 voxels per axis.  Each voxel is
      1 occupied  when the return of a valid ray falls into it (the VoxelGrid scatter from_points uses);
      0 free      otherwise, when the face-connected walk of some valid ray's segment from its origin to
                  (l - free_margin) / l of the way to its return passes through it (nothing when l <= free_margin);
      2 unknown   otherwise.
    free_margin defaults to sqrt(3) r / 2, half a cell diagonal.  The walk's fp32 rules (clipping, start voxel,
    boundary parameters, ties x then y then z) are in include/pvb.h.  The result depends on neither the ray order nor
    the thread order.  Returns uint8 [nx, ny, nz] on points' device."""
    rays = _rays(points, origins, max_range)
    lattice = _depth_lattice(resolution, range_per_dim, free_margin)
    src = rays.points.device
    return nat.deliver(_ray_state(rays, lattice, nat.compute_device(src)), src)


# ---------------------------------------------------------------- occupancy maps
LOG_ODDS_UNIT = 1024         # log-odds are stored as int16 in units of 1 / LOG_ODDS_UNIT
LOG_ODDS_UNOBSERVED = -32768


class OccupancyParams(NamedTuple):
    """OccupancyMap's update parameters in units of 1 / LOG_ODDS_UNIT."""
    hit: int
    miss: int
    clamp_lo: int
    clamp_hi: int
    threshold: int


def _occupancy_params(hit, miss, clamp, threshold):
    """Each parameter quantized once as round(x * 1024) (Python's round: nearest, ties to even), then checked:
    -32767 <= clamp_lo <= miss < 0 < hit <= clamp_hi <= 32767 and miss < threshold <= hit."""
    if len(clamp) != 2:
        raise ValueError(f"clamp must be (lo, hi), got {clamp!r}")
    raw = dict(hit=hit, miss=miss, clamp_lo=clamp[0], clamp_hi=clamp[1], threshold=threshold)
    for name, x in raw.items():
        if not math.isfinite(float(x)):
            raise ValueError(f"{name} must be finite, got {x}")
    p = OccupancyParams(**{name: round(float(x) * LOG_ODDS_UNIT) for name, x in raw.items()})
    if not (-32767 <= p.clamp_lo <= p.miss < 0 < p.hit <= p.clamp_hi <= 32767 and p.miss < p.threshold <= p.hit):
        raise ValueError(f"in units of 1/{LOG_ODDS_UNIT} the parameters must satisfy -32767 <= clamp_lo <= miss < 0 "
                         f"< hit <= clamp_hi <= 32767 and miss < threshold <= hit, got {p}")
    return p


class OccupancyMap:
    """A log-odds occupancy grid that fuses depth frames over time on the GPU (pvb_depth_integrate).

    The lattice is depth_occupancy's: the range snapped by get_divisible_range_by_resolution, voxel i centred at
    lo + i r, 2..1024 voxels per axis.  Each voxel holds a log-odds L, stored as an int16 in units of 1/1024, or
    "never observed".  Every parameter is quantized once as round(x * 1024), and after that they must satisfy
    -32767 <= clamp_lo <= miss < 0 < hit <= clamp_hi <= 32767 and miss < threshold <= hit (ValueError otherwise), so
    that a single observation decides a fresh voxel.  The defaults approximate OctoMap's (p_hit 0.7, p_miss 0.4,
    clamping at 0.12 / 0.97, threshold 0.5).

    integrate() adds one observation of the views of one call.  In int32 arithmetic, a voxel never observed starting
    from 0, each voxel receives at most one update per call:
      hit   a valid pixel's point of any view falls into it:  L = min(L + hit, clamp_hi);
      free  otherwise, when some view says free (depth_occupancy's rule, free_margin included):  L = max(L + miss,
            clamp_lo);
      otherwise L is unchanged.
    The result depends on neither the view order nor the thread order; frames taken at different times go in separate
    calls.  Because the evidence is bounded by the clamps, old evidence can be overturned: a voxel holding L turns free
    after ceil((L - threshold + 1) / -miss) free observations in a row, 9 from the upper clamp with the defaults, so an
    object that has moved leaves no ghost where later frames see free space.  After one call on a fresh map, state()
    equals depth_occupancy of the same views.  integrate does not synchronise with the host when the depth images are
    on the GPU.  integrate_points() adds one observation of point clouds with their sensor origins by the same update,
    ray_occupancy's rules deciding hit and free, and after one call on a fresh map state() equals ray_occupancy.

    :param free_margin: depth_occupancy's and ray_occupancy's, for every call; defaults to sqrt(3) r / 2
    :param device: device state() and log_odds() return on, and sdf()'s default device (the grid lives on the GPU)"""

    def __init__(self, resolution, range_per_dim, hit=0.85, miss=-0.4, clamp=(-2.0, 3.5), threshold=0.0,
                 free_margin=None, device="cpu"):
        self.params = _occupancy_params(hit, miss, clamp, threshold)
        self.resolution, self.range_per_dim, self.free_margin = _depth_lattice(resolution, range_per_dim, free_margin)
        self.device = device
        self._cdev = nat.compute_device(device)
        self._hits = VoxelGrid(self.resolution, self.range_per_dim, dtype=torch.bool, device=self._cdev)
        self._hits.voxels._geom()            # reads the lattice from the device once, so integrate never synchronises
        self.shape = tuple(self._hits.get_voxel_values().shape)
        self._log_odds = torch.full(self.shape, LOG_ODDS_UNOBSERVED, dtype=torch.int16, device=self._cdev)
        self._lo = (ctypes.c_float * 3)(*[float(min(r)) for r in self._hits.range_per_dim])
        self._dims = (ctypes.c_int32 * 3)(*self.shape)
        self._update = (ctypes.c_int32 * 4)(*self.params[:4])

    def integrate(self, depth, K, cam_to_world, max_depth=math.inf):
        """Add one observation of depth images [V, H, W] (V up to 64) to the map; the arguments are
        depth_to_points'.  Write 0 on pixels that should say nothing (the robot's own body, say)."""
        views = _depth_views(depth, K, cam_to_world, max_depth)
        d = views.depth.to(self._cdev).contiguous()
        V, H, W = d.shape
        intr = (ctypes.c_float * (4 * V))(*views.intrinsics.reshape(-1).tolist())
        c2w = (ctypes.c_float * (12 * V))(*views.cam_to_world[:, :3].to(torch.float32).reshape(-1).tolist())
        w2c = (ctypes.c_float * (12 * V))(
            *invert_rigid(views.cam_to_world)[:, :3].to(torch.float32).reshape(-1).tolist())
        L = nat.lib()
        with nat.on_device(self._cdev):
            points = torch.empty(V * H * W, 3, dtype=torch.float32, device=self._cdev)
            nat.check(L.pvb_depth_points(nat.ptr(d), V, H, W, intr, c2w, views.max_depth, nat.ptr(points),
                                         nat.stream_ptr(self._cdev)), "pvb_depth_points")
            self._hits[points] = True           # the NaN point of an invalid pixel falls into no voxel
            nat.check(L.pvb_depth_integrate(nat.ptr(d), V, H, W, intr, w2c, views.max_depth, self.free_margin,
                                            self._lo, self.resolution, self._dims,
                                            nat.ptr(self._hits.get_voxel_values()), nat.ptr(self._log_odds),
                                            self._update, nat.stream_ptr(self._cdev)), "pvb_depth_integrate")

    def integrate_points(self, points, origins, max_range=math.inf):
        """Add one observation of point clouds taken from known sensor origins to the map; the arguments are
        ray_occupancy's, with the map's free_margin.  Per voxel, a valid ray's return falling into it is a hit, and
        otherwise a valid ray's walk passing through it is a free observation (ray_occupancy's rules), each updating L
        as integrate's do; the call is one observation, so depth frames and point clouds can be fused into the same
        map in any interleaving.  With points and origins on the GPU it does not synchronise with the host.  Write NaN
        on points that should say nothing (the robot's own body, say)."""
        rays = _rays(points, origins, max_range)
        marks = self._hits.get_voxel_values().view(torch.uint8)
        out = _ray_carve(rays, self.free_margin, self._lo, self.resolution, self._dims, marks, self._cdev)
        with nat.on_device(self._cdev):
            self._hits[out] = True              # an invalid ray's NaN point falls into no voxel: hits win over free
            nat.check(nat.lib().pvb_occupancy_apply(nat.ptr(marks), nat.ptr(self._log_odds), self._dims,
                                                    self._update, nat.stream_ptr(self._cdev)), "pvb_occupancy_apply")

    def _state(self):
        L = self._log_odds
        return (L >= self.params.threshold).to(torch.uint8).masked_fill_(L == LOG_ODDS_UNOBSERVED, 2)

    def state(self):
        """uint8 [nx, ny, nz] on the map's device: 1 occupied (L >= threshold), 0 free, 2 never observed --
        depth_occupancy's encoding."""
        return nat.deliver(self._state(), self.device)

    def log_odds(self):
        """float32 [nx, ny, nz] on the map's device: the stored value / 1024 (exact), NaN where never observed."""
        L = self._log_odds
        return nat.deliver((L.to(torch.float32) / LOG_ODDS_UNIT).masked_fill_(L == LOG_ODDS_UNOBSERVED, math.nan),
                           self.device)

    def sdf(self, unknown="occupied", interpolation="nearest", device=None):
        """OccupancySDF of state() on the map's lattice: voxels never observed count as occupied
        (unknown="occupied") or free ("free"), OccupancySDF.from_depth's rule.  ValueError unless both states are
        present.  device defaults to the map's."""
        if unknown not in ("occupied", "free"):
            raise ValueError(f"unknown must be 'occupied' or 'free', got {unknown!r}")
        state = self._state()
        grid = VoxelGrid(self.resolution, self.range_per_dim, dtype=torch.bool, device=self._cdev)
        grid.get_voxel_values().copy_(state == 1 if unknown == "free" else state != 0)
        return OccupancySDF(grid, interpolation=interpolation, device=self.device if device is None else device)

    def reset(self):
        """Every voxel back to "never observed"."""
        self._log_odds.fill_(LOG_ODDS_UNOBSERVED)
        self._hits.get_voxel_values().zero_()


def sample_mesh_points(obj_factory: ObjectFactory = None, num_points=100, seed=0, name="",
                       clean_cache=False, dtype=torch.float, min_init_sample_points=200,
                       dbpath='model_points_cache.pkl', device="cpu", cache=None):
    """Area-uniform surface samples and their face normals (reference sdf.py:617-670).

    Same arguments, cache layout ({name: {seed: {num_points: (points, normals, None)}}}, torch.save) and return
    value `(points, normals, cache)` as the reference.  The samples come from a counter-based GPU generator, so the
    actual point set for a given seed differs from Open3D's mt19937 stream (the reference's stream is not
    reproducible outside Open3D either); it is deterministic per (mesh, seed, num_points).
    """
    # cache layout of the reference (sdf.py:620-634, 665): {name: {seed: {num_points: (points, normals, None)}}}, kept in
    # the caller's dict when one is passed, otherwise in the torch.save file `dbpath`
    caller_owns_cache = cache is not None
    if cache is None:
        cache = torch.load(dbpath) if os.path.exists(dbpath) else {}
    per_count = cache.setdefault(name, {}).setdefault(seed, {})
    hit = None if clean_cache else per_count.get(num_points)
    if hit is not None:
        points, normals = (None if t is None else t.to(device=device, dtype=dtype) for t in hit[:2])
        return points, normals, cache

    if obj_factory is None:
        raise RuntimeError(f"Expect model points to be cached for {name} {seed} {num_points} in {dbpath}")
    if obj_factory._mesh is None:
        obj_factory.precompute_sdf()

    cdev = nat.compute_device(device)
    sample_num_points = max(min_init_sample_points, 2 * num_points)       # sdf.py:650
    points = _sample_surface(obj_factory, sample_num_points, seed, cdev)
    # dispersion: keep a random subset of the over-sampled set (sdf.py:658)
    gen = torch.Generator(device=cdev)
    gen.manual_seed(int(seed))
    keep = torch.randperm(sample_num_points, generator=gen, device=cdev)[:num_points]
    points = points[keep]
    res = obj_factory.object_frame_closest_point(points, compute_normal=True)   # sdf.py:660
    normals = res.normal

    per_count[num_points] = points.cpu(), normals.cpu(), None
    if not caller_owns_cache:
        torch.save(cache, dbpath)
    return points.to(device=device, dtype=dtype), normals.to(device=device, dtype=dtype), cache


def _sample_surface(obj_factory, n, seed, device, return_faces=False):
    """n area-uniform fp64 surface points: stratified allocation of the samples to faces by cumulative area
    (face t receives round(cum_area_fraction(t) * n) - (samples so far), the Open3D rule behind sdf.py:654), then
    (1-sqrt(r1)) v0 + sqrt(r1)(1-r2) v1 + sqrt(r1) r2 v2 inside the face."""
    areas = obj_factory._mesh.triangle_areas()
    cum = np.cumsum(areas / areas.sum())
    upto = np.minimum(np.floor(cum * n + 0.5).astype(np.int64), n)
    upto = np.maximum.accumulate(upto)
    upto[-1] = n
    st = obj_factory._device_state(device)
    with torch.cuda.device(device):
        cum_dev = torch.from_numpy(upto).to(device)
        out = torch.empty(n, 3, dtype=torch.float64, device=device)
        face = torch.empty(n, dtype=torch.int32, device=device) if return_faces else None
        nat.check(nat.lib().pvb_mesh_sample(nat.ptr(st["v64"]), nat.ptr(st["faces"]), len(areas), nat.ptr(cum_dev),
                                            n, int(seed) & 0xFFFFFFFFFFFFFFFF, nat.ptr(out), nat.ptr(face),
                                            nat.stream_ptr(device)), "pvb_mesh_sample")
    return (out, face) if return_faces else out
