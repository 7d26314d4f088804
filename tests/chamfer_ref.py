"""fp64 restatement of batch_chamfer_dist (reference chamfer.py:62-94) and of the pose-set metrics built on it,
pairwise_distance_chamfer (chamfer.py:20-59) and PlausibleDiversity (chamfer.py:130-195), for the CPU and GPU tiers.

Object-frame points are computed in fp64 from the fp32 transforms and points the kernel reads.  The unsigned distance
of each route is evaluated without kernel code:
  mesh_spec(v, f)                 brute-force point-triangle distance (robot_ref.closest_on_triangles) on fp32 vertices
  grid_spec(cached)               nearest voxel + bounding-box rule (composed_ref.grid_eval); with
                                  OutOfBoundsStrategy.LOOKUP_GT_SDF the brute-force mesh distance outside the range
  primitive_spec(desc)            SphereSDF / BoxSDF / CylinderSDF (primitive_ref)
  trilinear_spec(cached)          trilinear CachedSDF (oracle.port.trilinear_lookup_port)
The chamfer value is the fp64 mean over the points of (scale * d)^2.  Test infrastructure only."""
import numpy as np
import torch

import helpers
import primitive_ref as pr
from composed_ref import grid_eval
from robot_ref import closest_on_triangles

U32 = 2.0 ** -24          # fp32 unit roundoff


# ------------------------------------------------------------------ specs
def mesh_spec(v, f):
    """The kernel reads fp32 vertices."""
    v32 = np.asarray(v, dtype=np.float32).astype(np.float64)
    return {"kind": "mesh", "tri": v32[np.asarray(f)]}


def grid_spec(cached, gt_mesh=None):
    """Nearest-voxel CachedSDF; gt_mesh=(v, f) for OutOfBoundsStrategy.LOOKUP_GT_SDF."""
    s = helpers.grid_spec(cached)
    if gt_mesh is not None:
        s["gt"] = mesh_spec(*gt_mesh)
    return s


def primitive_spec(desc):
    return {"kind": "primitive", "desc": desc}


def trilinear_spec(cached):
    return {"kind": "trilinear", "val": cached.voxels.raw_data.detach().cpu().reshape(tuple(cached.voxels.shape)),
            "ranges": cached.ranges, "bb": cached.bb.detach().cpu().numpy().astype(np.float64)}


# ------------------------------------------------------------------ distances
def mesh_distance(tri, q):
    """Unsigned distance of q [n, 3] to the triangles tri [F, 3, 3], fp64 brute force."""
    q = np.asarray(q, dtype=np.float64).reshape(-1, 3)
    out = np.empty(len(q))
    step = max(1, 1_000_000 // len(tri))
    for s in range(0, len(q), step):
        out[s:s + step] = closest_on_triangles(q[s:s + step], tri)[1].min(axis=1)
    return out


def distance(spec, q):
    """Unsigned distance [n] of each route at object-frame points q [n, 3] (fp64)."""
    q = np.asarray(q, dtype=np.float64).reshape(-1, 3)
    kind = spec["kind"]
    if kind == "mesh":
        return mesh_distance(spec["tri"], q)
    if kind == "primitive":
        return np.abs(pr.primitive_ref(spec["desc"], q)[0])
    if kind == "trilinear":
        from oracle import port
        v, _g, _inb = port.trilinear_lookup_port(spec["val"], spec["ranges"], spec["bb"], torch.from_numpy(q))
        return np.abs(v.numpy())
    assert kind == "grid", kind
    v = np.abs(grid_eval(spec, q)[0])
    if "gt" in spec:
        out = ~np.all((q >= spec["lo"]) & (q <= spec["hi"]), axis=1)
        if out.any():
            v[out] = mesh_distance(spec["gt"]["tri"], q[out])
    return v


def grid_alternatives(spec, q):
    """Every unsigned distance the nearest-voxel rule can give at q (3,) when a coordinate within helpers.FLIP_BAND
    cells of a cell boundary, or within 1e-6 of the range edge, falls on either side (voxel-boundary flips of the
    fp32 transform)."""
    lo, hi, val = spec["lo"], spec["hi"], spec["val"]
    n = np.array(val.shape)
    res = (hi - lo) / (n - 1)
    edge = 1e-6
    out = []
    if np.all((q >= lo - edge) & (q <= hi + edge)):
        u = (q - lo) / res
        opts = []
        for a in range(3):
            o = {int(np.clip(np.rint(u[a]), 0, n[a] - 1))}
            if abs(u[a] - np.floor(u[a]) - 0.5) < helpers.FLIP_BAND:
                o.update({int(np.clip(np.floor(u[a]), 0, n[a] - 1)), int(np.clip(np.floor(u[a]) + 1, 0, n[a] - 1))})
            opts.append(sorted(o))
        out += [abs(val[i, j, k]) for i in opts[0] for j in opts[1] for k in opts[2]]
    if np.any((q < lo + edge) | (q > hi - edge)):
        out.append(float(mesh_distance(spec["gt"]["tri"], q[None])[0]) if "gt" in spec
                   else float(helpers._aabb_rule(spec["bb"], q)[0]))
    return out


# ------------------------------------------------------------------ chamfer
def object_points(w2o, pts):
    """(B, N, 3) fp64 object-frame points of the fp32-rounded transforms (B, 4, 4) and points (N, 3)."""
    W = np.asarray(w2o, dtype=np.float32).astype(np.float64)
    p = np.asarray(pts, dtype=np.float32).astype(np.float64)
    return np.einsum("bij,nj->bni", W[:, :3, :3], p) + W[:, None, :3, 3]


def transform_error(w2o, pts):
    """(B, N) bound on |q_fp32 - q_fp64| of the kernel's FMA chain q_i = R_i0 p_0 + R_i1 p_1 + R_i2 p_2 + t_i:
    3u (sum_j |R_ij p_j| + |t_i|) per component."""
    W = np.asarray(w2o, dtype=np.float32).astype(np.float64)
    p = np.abs(np.asarray(pts, dtype=np.float32).astype(np.float64))
    e = 3 * U32 * (np.einsum("bij,nj->bni", np.abs(W[:, :3, :3]), p) + np.abs(W[:, None, :3, 3]))
    return np.linalg.norm(e, axis=-1)


def per_pair(spec, w2o, pts):
    """(B, N) unsigned fp64 distances."""
    q = object_points(w2o, pts)
    return distance(spec, q.reshape(-1, 3)).reshape(q.shape[:2])


def chamfer(spec, w2o, pts, scale=1000.0):
    """(B,) fp64 mean over the points of (scale * d)^2."""
    return ((scale * per_pair(spec, w2o, pts)) ** 2).mean(axis=1)


def square_bound(d, dd, scale):
    """Bound on |(scale d')^2 - (scale d)^2| for |d' - d| <= dd."""
    return scale ** 2 * (2 * np.abs(d) * dd + dd ** 2)


def composite_error(left, right, pts):
    """(L*R, N) bound on the object-frame error that an fp32 einsum of the composites left[i] @ right[j] adds over
    the fp64 composites: 4u (|L| |R|) per entry (four products summed), applied to |p| and the translation."""
    L = np.abs(np.asarray(left, dtype=np.float64))
    R = np.abs(np.asarray(right, dtype=np.float64))
    E = (4 * U32 * np.einsum("bij,pjk->bpik", L, R)).reshape(-1, 4, 4)
    p = np.abs(np.asarray(pts, dtype=np.float64))
    return np.linalg.norm(np.einsum("bij,nj->bni", E[:, :3, :3], p) + E[:, None, :3, 3], axis=-1)


def sum_bound(n, n_blk):
    """Relative bound on the kernel's fp32 sum of n non-negative terms over n_blk blocks of 256 threads: each thread
    adds up to k terms with fmaf, then 5 warp-shuffle and 8 warp-sum additions; plus the rounding of scale * d (2u on
    its square), the fp64 finish and the fp32 result."""
    k = -(-n // (n_blk * 256))
    return (k + 5 + 8 + 2 + 1) * U32


# ------------------------------------------------------------------ exact box cloud
def box_mesh(half):
    """12-triangle axis-aligned box [-half, half]^3, outward faces."""
    v = np.array([[x, y, z] for x in (-half, half) for y in (-half, half) for z in (-half, half)], dtype=np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                  [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    return v, f


def exact_box_cloud(n, half, heights, rng, margin=0.05):
    """n object-frame points straight above the face interiors of box_mesh(half), at the dyadic `heights`, with
    in-face coordinates on a 2^-12 grid at least `margin` inside the face.  Returns (points [n, 3], heights [n])."""
    axis = rng.integers(0, 3, n)
    sign = np.where(rng.integers(0, 2, n) == 0, -1.0, 1.0)
    h = np.asarray(heights, dtype=np.float64)[rng.integers(0, len(heights), n)]
    lim = int((half - margin) * 4096)
    q = rng.integers(-lim, lim + 1, (n, 3)).astype(np.float64) / 4096
    q[np.arange(n), axis] = sign * (half + h)
    return q, h


def signed_permutations(k, rng):
    """k random 3x3 signed permutation matrices (symmetries of a box centred at the origin)."""
    out = np.zeros((k, 3, 3))
    for i in range(k):
        out[i, np.arange(3), rng.permutation(3)] = np.where(rng.integers(0, 2, 3) == 0, -1.0, 1.0)
    return out


# ------------------------------------------------------------------ pose-set metrics
def rigid_inverse(m):
    m = np.asarray(m, dtype=np.float64)
    out = np.zeros_like(m)
    R = np.swapaxes(m[:, :3, :3], 1, 2)
    out[:, :3, :3] = R
    out[:, :3, 3] = -np.einsum("bij,bj->bi", R, m[:, :3, 3])
    out[:, 3, 3] = 1.0
    return out


def pairwise_composites(A_link_to_world, B_world_to_link=None):
    """The reference's einsum("bij,pjk->bpik", T_inv, T) over (len(T_inv), len(T)), flat in that order, fp64."""
    T = np.asarray(A_link_to_world, dtype=np.float64)
    T_inv = rigid_inverse(T) if B_world_to_link is None else np.asarray(B_world_to_link, dtype=np.float64)
    return np.einsum("bij,pjk->bpik", T_inv, T).reshape(-1, 4, 4)


def pairwise_distance_chamfer(spec, pts, A_link_to_world, B_world_to_link=None, scale=1000.0):
    """errors.view(len(A), len(B)) of the flat T_inv-major data (chamfer.py:49-58), fp64."""
    n_a = len(A_link_to_world)
    n_b = n_a if B_world_to_link is None else len(B_world_to_link)
    flat = chamfer(spec, pairwise_composites(A_link_to_world, B_world_to_link), pts, scale)
    return flat.reshape(n_a, n_b)


def plausible_diversity_from_errors(errors):
    """(plausibility, coverage, argmin per estimate, argmin per plausible): min over each dimension, sum / B and
    sum / P (chamfer.py:185-195)."""
    B, P = errors.shape
    return errors.min(axis=1).sum() / B, errors.min(axis=0).sum() / P, errors.argmin(axis=1), errors.argmin(axis=0)


def plausible_diversity(spec, pts, T_est_inv, T_p, bidirectional=False, scale=1000.0):
    """PlausibleDiversity.__call__ (chamfer.py:150-173): errors[b, p] = chamfer(T_est_inv[b] @ T_p[p]); with
    bidirectional, the swapped sets' plausibility and coverage trade places and both are averaged."""
    def errors(left, right):
        comp = np.einsum("bij,pjk->bpik", np.asarray(left, np.float64), np.asarray(right, np.float64))
        return chamfer(spec, comp.reshape(-1, 4, 4), pts, scale).reshape(comp.shape[:2])
    pl, cov, best_est, best_pl = plausible_diversity_from_errors(errors(T_est_inv, T_p))
    if bidirectional:
        pl2, cov2, _, _ = plausible_diversity_from_errors(errors(T_p, T_est_inv))
        pl, cov = (pl + cov2) / 2, (cov + pl2) / 2
    return pl, cov, best_est, best_pl
