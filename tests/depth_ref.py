"""fp64 reference of the depth-image semantics (depth_to_points, depth_occupancy, OccupancySDF.from_depth), and the
host build of their device routines (tests/hostsim/hostsim_depth.cpp).

Definition (include/pvb.h): a pixel is valid when its depth d is finite, d > 0 and d <= max_depth.
1. Back-projection: pixel (row i, column j) gives p_cam = ((j - cx) d / fx, (i - cy) d / fy, d), world = cam_to_world
   p_cam.
2. Carving, per voxel centre c = lo + i r and view: with (x, y, z) = world_to_cam c, the view says nothing when
   z <= 0, when the pixel (floor(fy y / z + cy + 0.5), floor(fx x / z + cx + 0.5)) lies outside the image or is
   invalid; otherwise free when z < d - margin.
3. Fusion: occupied (1) when a valid pixel's point falls into the voxel (index round((p - lo) / r)), otherwise free
   (0) when any view says free, otherwise unknown (2).

The reference computes everything in fp64 and flags each voxel whose result could go either way in fp32: a view that
projects it within 1e-3 px of a rounding boundary of u or v, or with |z - (d - margin)| < 1e-5 d, and a voxel a point
lands in within 1e-3 cells of a cell boundary (both neighbours are flagged)."""
import ctypes
import math

import numpy as np

PX_TOL = 1e-3
DEPTH_TOL = 1e-5
CELL_TOL = 1e-3


def _f64(a):
    return np.asarray(a.detach().cpu() if hasattr(a, "detach") else a, dtype=np.float64)


def views(K, cam_to_world, V):
    """(K fp64 [V, 3, 3], cam_to_world fp64 [V, 4, 4], world_to_cam fp64 [V, 4, 4]) with K broadcast over V."""
    K = np.broadcast_to(_f64(K), (V, 3, 3))
    c2w = _f64(cam_to_world).reshape(V, 4, 4)
    w2c = np.zeros_like(c2w)
    R, t = c2w[:, :3, :3], c2w[:, :3, 3]
    w2c[:, :3, :3] = R.transpose(0, 2, 1)
    w2c[:, :3, 3] = -np.einsum("vji,vj->vi", R, t)
    w2c[:, 3, 3] = 1
    return K, c2w, w2c


def lattice(resolution, range_per_dim):
    """(lo fp64 [3], dims [3]) of the OccupancySDF lattice: the range snapped by get_divisible_range_by_resolution."""
    from pytorch_volumetric_b200.voxel import get_coordinates_and_points_in_grid, get_divisible_range_by_resolution
    snapped = get_divisible_range_by_resolution(resolution, range_per_dim)
    coords, _ = get_coordinates_and_points_in_grid(resolution, snapped, get_points=False)
    return np.array([min(r) for r in snapped], np.float64), tuple(len(c) for c in coords)


def valid(depth, max_depth=math.inf):
    d = np.asarray(depth, np.float32)
    return np.isfinite(d) & (d > 0) & (d <= np.float32(max_depth))


def points(depth, K, cam_to_world, max_depth=math.inf):
    """(points fp64 [V, H, W, 3], valid [V, H, W]); NaN where invalid."""
    d = np.asarray(depth, np.float32)
    V, H, W = d.shape
    K, c2w, _ = views(K, cam_to_world, V)
    ok = valid(d, max_depth)
    dd = np.where(ok, d, np.nan).astype(np.float64)
    i, j = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    fx, fy, cx, cy = (K[:, 0, 0, None, None], K[:, 1, 1, None, None], K[:, 0, 2, None, None], K[:, 1, 2, None, None])
    cam = np.stack([(j - cx) * dd / fx, (i - cy) * dd / fy, dd], -1)
    world = np.einsum("vkl,vhwl->vhwk", c2w[:, :3, :3], cam) + c2w[:, None, None, :3, 3]
    return world, ok


def carve(depth, K, cam_to_world, resolution, range_per_dim, max_depth=math.inf, margin=None):
    """(state uint8 [nx, ny, nz] with 0 free / 2 unknown, ambiguous bool [nx, ny, nz]) of rule 2."""
    d = np.asarray(depth, np.float32)
    V, H, W = d.shape
    K, _, w2c = views(K, cam_to_world, V)
    margin = math.sqrt(3.0) * resolution / 2 if margin is None else margin
    lo, dims = lattice(resolution, range_per_dim)
    idx = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in dims], indexing="ij"), -1).reshape(-1, 3)
    c = lo + idx * resolution
    free = np.zeros(len(c), bool)
    amb = np.zeros(len(c), bool)
    ok = valid(d, max_depth)
    for v in range(V):
        p = c @ w2c[v, :3, :3].T + w2c[v, :3, 3]
        z = p[:, 2]
        front = z > 0
        zs = np.where(front, z, 1.0)
        u = K[v, 0, 0] * p[:, 0] / zs + K[v, 0, 2] + 0.5
        w = K[v, 1, 1] * p[:, 1] / zs + K[v, 1, 2] + 0.5
        near_edge = front & (np.abs(u) < 2 * W + 2) & (np.abs(w) < 2 * H + 2) & (
            (np.abs(u - np.rint(u)) < PX_TOL) | (np.abs(w - np.rint(w)) < PX_TOL))
        col, row = np.floor(u), np.floor(w)
        inside = front & (col >= 0) & (col < W) & (row >= 0) & (row < H)
        ci, ri = np.where(inside, col, 0).astype(np.int64), np.where(inside, row, 0).astype(np.int64)
        dv = d[v, ri, ci].astype(np.float64)
        seen = inside & ok[v, ri, ci]
        thr = dv - margin
        says = seen & (z < thr)
        free |= says
        amb |= near_edge | (seen & (np.abs(z - thr) < DEPTH_TOL * dv))
    state = np.where(free, 0, 2).astype(np.uint8)
    return state.reshape(dims), amb.reshape(dims)


def fuse(state, ambiguous, pts, ok, resolution, range_per_dim):
    """Rule 3 on top of carve(): (state with 1 where a valid point falls, ambiguous) -- pts fp64 [..., 3]."""
    lo, dims = lattice(resolution, range_per_dim)
    state, ambiguous = state.copy(), ambiguous.copy()
    p = np.asarray(pts, np.float64)[np.asarray(ok)].reshape(-1, 3)
    f = (p - lo) / resolution + 0.5
    idx = np.floor(f).astype(np.int64)
    frac = f - idx
    shape = np.array(dims)
    inb = ((idx >= 0) & (idx < shape)).all(1)
    state[tuple(idx[inb].T)] = 1
    for k in range(3):
        for side, step in ((frac[:, k] < CELL_TOL, -1), (frac[:, k] > 1 - CELL_TOL, 1)):
            for base in (idx, idx + np.eye(3, dtype=np.int64)[k] * step):
                sel = side & ((base >= 0) & (base < shape)).all(1)
                ambiguous[tuple(base[sel].T)] = True
    return state, ambiguous


# ---------------------------------------------------------------- the host build
def rows(K, cam_to_world, V):
    """The entry points' HOST arrays, as sdf.py builds them: (intrinsics fp32 [V, 4], cam_to_world rows fp32 [V, 12],
    world_to_cam rows fp32 [V, 12]) -- world_to_cam inverted in fp64, then rounded."""
    import torch
    from pytorch_volumetric_b200.transforms import invert_rigid
    K, c2w, _ = views(K, cam_to_world, V)
    intr = np.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], 1).astype(np.float32)
    m = torch.from_numpy(c2w)
    return (np.ascontiguousarray(intr), np.ascontiguousarray(m[:, :3].float().reshape(V, 12).numpy()),
            np.ascontiguousarray(invert_rigid(m)[:, :3].float().reshape(V, 12).numpy()))


def host_points(depth, K, cam_to_world, max_depth=math.inf):
    """float32 [V, H, W, 3] of the host build of depth_points_kernel."""
    import hostsim_lib as hs
    d = np.ascontiguousarray(depth, np.float32)
    V, H, W = d.shape
    intr, c2w, _ = rows(K, cam_to_world, V)
    out = np.empty((V, H, W, 3), np.float32)
    hs.lib().simdepth_points(hs._p(d), V, H, W, hs._p(intr), hs._p(c2w), ctypes.c_float(max_depth), hs._p(out))
    return out


def host_carve(depth, K, cam_to_world, resolution, range_per_dim, max_depth=math.inf, margin=None):
    """uint8 [nx, ny, nz] (0 / 2) of the host build of depth_carve_kernel."""
    import hostsim_lib as hs
    d = np.ascontiguousarray(depth, np.float32)
    V, H, W = d.shape
    intr, _, w2c = rows(K, cam_to_world, V)
    margin = math.sqrt(3.0) * resolution / 2 if margin is None else margin
    lo, dims = lattice(resolution, range_per_dim)
    lo32 = lo.astype(np.float32)
    out = np.empty(dims, np.uint8)
    hs.lib().simdepth_carve(hs._p(d), V, H, W, hs._p(intr), hs._p(w2c), ctypes.c_float(max_depth),
                            ctypes.c_float(margin), hs._p(lo32), ctypes.c_float(resolution),
                            (ctypes.c_int * 3)(*dims), hs._p(out))
    return out
