"""fp64 reference of the ray carve (ray_occupancy, pvb_ray_carve), and the host build of its device routines
(tests/hostsim/hostsim_rays.cpp).

Definition (include/pvb.h): a ray from origin o to return p, both fp32, is valid when its coordinates are finite and
0 < |p - o| <= max_range.  Its free segment is o + t (p - o), 0 <= t <= t_end = (l - m) / l (nothing when l <= m).  In
lattice coordinates a = (x - lo) / r + 0.5 voxel i covers [i, i + 1).  The reference takes, in fp64, the voxels whose
half-open cube meets the free segment with positive length: the segment is cut at every lattice plane it crosses, and
each piece of positive length lies in one voxel (the one holding its midpoint).

The fp32 walk may differ from it only where the segment passes close to a face or an edge of a voxel, or where a
voxel's piece begins or ends close to the segment's ends: classify() decides whether a voxel of the symmetric
difference is of that kind, with the distance eps counted in cells."""
import ctypes
import math

import numpy as np

EPS = 1e-4


def lattice(resolution, range_per_dim):
    """(lo fp64 [3], dims [3]) of depth_occupancy's lattice."""
    import depth_ref
    return depth_ref.lattice(resolution, range_per_dim)


def segment(o, p, max_range, margin, lo, r):
    """fp64 (valid, a [3], u [3], t_end) of one ray of fp32 o and p: a = (o - lo32) / r + 0.5, u = (p - o) / r, with lo
    rounded to fp32 as the entry point receives it; t_end is None when nothing is carved."""
    o, p = np.float64(np.float32(o)), np.float64(np.float32(p))
    lo32 = np.float64(np.float32(lo))
    if not (np.isfinite(o).all() and np.isfinite(p).all()):
        return False, None, None, None
    d = p - o
    ln = float(np.sqrt((d * d).sum()))
    if not (0 < ln <= max_range and math.isfinite(ln)):
        return False, None, None, None
    a = (o - lo32) / r + 0.5
    u = d / r
    return True, a, u, ((ln - margin) / ln if ln > margin else None)


def _clip(a, u, t_end, dims):
    t_lo, t_hi = 0.0, t_end
    for k in range(3):
        if u[k] == 0:
            if not 0 <= a[k] < dims[k]:
                return None
        else:
            t0, t1 = -a[k] / u[k], (dims[k] - a[k]) / u[k]
            t_lo, t_hi = max(t_lo, min(t0, t1)), min(t_hi, max(t0, t1))
    return (t_lo, t_hi) if t_lo < t_hi else None


def voxels(a, u, t_end, dims):
    """int64 [K, 3]: the voxels of the free segment in order along it."""
    if t_end is None:
        return np.zeros((0, 3), np.int64)
    c = _clip(a, u, t_end, dims)
    if c is None:
        return np.zeros((0, 3), np.int64)
    t_lo, t_hi = c
    ts = [np.array([t_lo, t_hi])]
    for k in range(3):
        if u[k] != 0:
            x0, x1 = sorted((a[k] + t_lo * u[k], a[k] + t_hi * u[k]))
            planes = np.arange(math.floor(x0), math.floor(x1) + 1, dtype=np.float64)
            ts.append((planes - a[k]) / u[k])
    t = np.unique(np.concatenate(ts))
    t = t[(t >= t_lo) & (t <= t_hi)]
    mid = 0.5 * (t[:-1] + t[1:])[t[1:] > t[:-1]]
    idx = np.floor(a[None] + mid[:, None] * u[None]).astype(np.int64)
    idx = np.clip(idx, 0, np.asarray(dims) - 1)
    keep = np.ones(len(idx), bool)
    keep[1:] = (idx[1:] != idx[:-1]).any(1)
    return idx[keep]


def _interval(a, u, v, grow):
    """The t interval on which a + t u lies in the closed cube of voxel v grown by `grow` cells per side."""
    t_lo, t_hi = -math.inf, math.inf
    for k in range(3):
        lo_k, hi_k = v[k] - grow, v[k] + 1 + grow
        if u[k] == 0:
            if not lo_k <= a[k] <= hi_k:
                return math.inf, -math.inf
        else:
            t0, t1 = (lo_k - a[k]) / u[k], (hi_k - a[k]) / u[k]
            t_lo, t_hi = max(t_lo, min(t0, t1)), min(t_hi, max(t0, t1))
    return t_lo, t_hi


def classify(v, a, u, t_end, in_walk, eps=EPS):
    """Whether voxel v of the symmetric difference is explained by a near tie: the fp64 segment passes within eps
    cells of one of v's faces or edges, or v's piece begins or ends within eps cells of the segment's ends.  in_walk:
    v is in the fp32 walk (and not in the reference), else the other way round."""
    dt = eps / max(float(np.linalg.norm(u)), 1e-300)           # eps cells along the ray, in t
    if in_walk:
        # the segment, its ends extended by eps, comes within eps of v's cube
        t0, t1 = _interval(a, u, v, eps)
        return max(t0, -dt) <= min(t1, t_end + dt)
    # the segment's piece in v, shrunk by eps on every face and at the segment's ends, is empty
    t0, t1 = _interval(a, u, v, -eps)
    return not max(t0, dt) < min(t1, t_end - dt)


def compare(walk, ref, a, u, t_end):
    """(differences, unclassified) between one ray's fp32 walk and its reference voxels."""
    w = {tuple(x) for x in np.asarray(walk).tolist()}
    f = {tuple(x) for x in np.asarray(ref).tolist()}
    bad = [v for v in w - f if not classify(v, a, u, t_end, True)]
    bad += [v for v in f - w if not classify(v, a, u, t_end, False)]
    return len(w ^ f), bad


def path_lengths(points, origins, per_origin, max_range, margin, lo, r, dims):
    """int64 [n_rays]: the number of voxels of every ray's free segment, vectorised (1 + the lattice planes crossed
    inside the grid), for counting visits in the benchmark; 0 for an invalid ray or an empty segment."""
    p = np.asarray(points, np.float32).reshape(-1, 3).astype(np.float64)
    o = np.repeat(np.asarray(origins, np.float32).reshape(-1, 3), per_origin, axis=0).astype(np.float64)
    lo32 = np.asarray(lo, np.float32).astype(np.float64)
    n = np.asarray(dims, np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        d = p - o
        ln = np.sqrt((d * d).sum(1))
        valid = np.isfinite(p).all(1) & np.isfinite(o).all(1) & (ln > 0) & (ln <= max_range) & np.isfinite(ln) & (
            ln > margin)
        t_end = np.where(valid, (ln - margin) / np.where(valid, ln, 1.0), 0.0)
        a = (o - lo32) / r + 0.5
        u = d / r
        t0, t1 = -a / u, (n - a) / u
        inside = (a >= 0) & (a < n)
        enter = np.where(u == 0, np.where(inside, -np.inf, np.inf), np.minimum(t0, t1))
        leave = np.where(u == 0, np.where(inside, np.inf, -np.inf), np.maximum(t0, t1))
        t_lo = np.maximum(0.0, enter.max(1))
        t_hi = np.minimum(t_end, leave.min(1))
        ok = valid & (t_lo < t_hi)
        x0 = np.floor(a + t_lo[:, None] * u)
        x1 = np.floor(a + t_hi[:, None] * u)
        x0 = np.clip(x0, 0, n - 1)
        x1 = np.clip(x1, 0, n - 1)
        count = 1 + np.abs(x1 - x0).sum(1)
    return np.where(ok, count, 0).astype(np.int64)


# ---------------------------------------------------------------- the host build
def _args(points, origins, per_origin, resolution, range_per_dim, margin):
    pts = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
    org = np.ascontiguousarray(np.asarray(origins, np.float32).reshape(-1, 3))
    assert len(pts) == len(org) * per_origin
    lo, dims = lattice(resolution, range_per_dim)
    margin = math.sqrt(3.0) * resolution / 2 if margin is None else margin
    return pts, org, lo.astype(np.float32), dims, margin


def host_carve(points, origins, per_origin, resolution, range_per_dim, max_range=math.inf, margin=None, marks=None):
    """(marks uint8 [nx, ny, nz], out_points float32 [n_rays, 3]) of the host build of ray_carve_kernel."""
    import hostsim_lib as hs
    pts, org, lo32, dims, margin = _args(points, origins, per_origin, resolution, range_per_dim, margin)
    marks = np.zeros(dims, np.uint8) if marks is None else np.array(marks, np.uint8, order="C")
    out = np.empty_like(pts)
    hs.lib().simray_carve(hs._p(pts), ctypes.c_longlong(len(pts)), ctypes.c_longlong(per_origin), hs._p(org),
                          ctypes.c_float(max_range), ctypes.c_float(margin), hs._p(lo32), ctypes.c_float(resolution),
                          (ctypes.c_int * 3)(*dims), hs._p(marks), hs._p(out))
    return marks, out


def host_walks(points, origins, per_origin, resolution, range_per_dim, max_range=math.inf, margin=None):
    """([int32 [count, 3] per ray] in visiting order, valid bool [n_rays]) of the host build of ray_walk."""
    import hostsim_lib as hs
    pts, org, lo32, dims, margin = _args(points, origins, per_origin, resolution, range_per_dim, margin)
    cap = sum(dims)
    idx = np.zeros((len(pts), cap, 3), np.int32)
    count = np.zeros(len(pts), np.int32)
    valid = np.zeros(len(pts), np.uint8)
    hs.lib().simray_walks(hs._p(pts), ctypes.c_longlong(len(pts)), ctypes.c_longlong(per_origin), hs._p(org),
                          ctypes.c_float(max_range), ctypes.c_float(margin), hs._p(lo32), ctypes.c_float(resolution),
                          (ctypes.c_int * 3)(*dims), hs._p(idx), hs._p(count), hs._p(valid))
    return [idx[t, :count[t]] for t in range(len(pts))], valid.astype(bool)


def host_apply(marks, L, q):
    """(marks, L) after the host build of occupancy_apply_kernel, from copies."""
    import hostsim_lib as hs
    marks = np.array(marks, np.uint8, order="C")
    L = np.array(L, np.int16, order="C")
    hs.lib().simray_apply(hs._p(marks), hs._p(L), ctypes.c_longlong(L.size), (ctypes.c_int * 4)(*q[:4]))
    return marks, L
