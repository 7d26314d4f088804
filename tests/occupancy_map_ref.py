"""numpy int32 reference of the occupancy-map update (OccupancyMap, pvb_depth_integrate), and the host build of its
device routines (tests/hostsim/hostsim_occupancy_map.cpp).

Definition (include/pvb.h): log-odds are int16 in units of 1/1024, -32768 meaning "never observed".  One call observes
each voxel at most once, as depth_occupancy's state of the same views says: 1 (a hit), 0 (free) or 2 (nothing).  With
L = 0 for a voxel never observed, a hit gives min(L + hit, clamp_hi), a free observation max(L + miss, clamp_lo), and
nothing leaves the stored value as it is.  state() is 2 where never observed, 1 where L >= threshold, 0 elsewhere."""
import ctypes
import math

import numpy as np

UNOBSERVED = -32768
DEFAULTS = dict(hit=0.85, miss=-0.4, clamp=(-2.0, 3.5), threshold=0.0)


def quantize(hit, miss, clamp, threshold):
    """(hit, miss, clamp_lo, clamp_hi, threshold) in 1/1024 units: round(x * 1024), nearest with ties to even."""
    return tuple(int(np.rint(np.float64(x) * 1024)) for x in (hit, miss, clamp[0], clamp[1], threshold))


def update(L, obs, q):
    """int16 [...]: one call's update of the stored values L under observations obs (1 hit, 0 free, 2 nothing)."""
    hit, miss, lo, hi = q[:4]
    L = np.asarray(L, np.int16)
    obs = np.asarray(obs, np.uint8)
    base = np.where(L == UNOBSERVED, 0, L.astype(np.int32))
    out = np.where(obs == 1, np.minimum(base + hit, hi), np.where(obs == 0, np.maximum(base + miss, lo), L))
    return out.astype(np.int16)


def replay(states, q, shape=None):
    """int16: the stored values after the calls whose per-call observations are `states` (depth_occupancy grids)."""
    states = list(states)
    L = np.full(np.shape(states[0]) if shape is None else shape, UNOBSERVED, np.int16)
    for s in states:
        L = update(L, s, q)
    return L


def state(L, q):
    L = np.asarray(L)
    return np.where(L == UNOBSERVED, 2, np.where(L >= q[4], 1, 0)).astype(np.uint8)


def log_odds(L):
    L = np.asarray(L)
    return np.where(L == UNOBSERVED, np.nan, L.astype(np.float32) / np.float32(1024)).astype(np.float32)


# ---------------------------------------------------------------- the host build
def host_update(L, obs, q):
    """int16 [...]: occupancy_update of the host build on every (L, obs) pair."""
    import hostsim_lib as hs
    L = np.ascontiguousarray(L, np.int16)
    obs = np.ascontiguousarray(np.broadcast_to(obs, L.shape), np.uint8)
    out = np.empty_like(L)
    hs.lib().simocc_update(hs._p(L), hs._p(obs), ctypes.c_longlong(L.size), (ctypes.c_int * 4)(*q[:4]), hs._p(out))
    return out


def host_integrate(L, hits, depth, K, cam_to_world, resolution, range_per_dim, q, max_depth=math.inf, margin=None):
    """(L int16, hits uint8) after the host build of depth_integrate_kernel's per-voxel body, from copies of the
    stored values L and the hit grid."""
    import depth_ref
    import hostsim_lib as hs
    d = np.ascontiguousarray(depth, np.float32)
    V, H, W = d.shape
    intr, _, w2c = depth_ref.rows(K, cam_to_world, V)
    margin = math.sqrt(3.0) * resolution / 2 if margin is None else margin
    lo, dims = depth_ref.lattice(resolution, range_per_dim)
    lo32 = lo.astype(np.float32)
    L = np.array(L, np.int16, order="C")
    hits = np.array(hits, np.uint8, order="C")
    assert L.shape == hits.shape == tuple(dims)
    hs.lib().simocc_integrate(hs._p(d), V, H, W, hs._p(intr), hs._p(w2c), ctypes.c_float(max_depth),
                              ctypes.c_float(margin), hs._p(lo32), ctypes.c_float(resolution),
                              (ctypes.c_int * 3)(*dims), hs._p(hits), hs._p(L), (ctypes.c_int * 4)(*q[:4]))
    return L, hits
