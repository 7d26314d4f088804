"""GPU: ray-cast point clouds (pvb_ray_carve, pvb_occupancy_apply, ray_occupancy, OccupancySDF.from_rays,
OccupancyMap.integrate_points).

1. pvb_ray_carve's marks and out_points equal the host build (tests/hostsim/hostsim_rays.cpp) bit for bit: the CPU
   tier's ray sets on their grids, and LiDAR scans and depth frames fed as rays on the 0.02 m and 0.01 m tabletop
   grids, 256^3 and 1024 x 64 x 64.
2. On depth frames fed as rays (camera centres as origins), ray_occupancy's occupied voxels are depth_occupancy's.
3. A fresh map: one integrate_points gives state() = ray_occupancy and sdf() = OccupancySDF.from_rays, bit for bit,
   with the default parameters and test_gpu_occupancy_map.OTHER.
4. Sequences of integrate_points calls interleaved with integrate depth calls equal occupancy_map_ref.replay over the
   per-call ray_occupancy and depth_occupancy states, both clamps reached, the scratch all zero after every call.
5. Determinism: permuted rays, and one scan split into V scans with repeated origins, give the same bits.
6. A box in LiDAR scans for 6 calls, then removed: its saturated voxels that later scans traverse turn free after
   exactly 9 calls; those no scan traverses stay occupied.
7. integrate_points does not synchronise from the second call on."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

import occupancy_map_ref as omr
import ray_ref
import workloads
from test_gpu_depth_occupancy import _cube
from test_gpu_occupancy_map import OTHER
from test_ray_occupancy_cpu import CASES, GRIDS

pytestmark = pytest.mark.gpu

RANGE = workloads.TABLETOP_RANGE
LO = (-1.1, -0.6, -0.35)
BIG_GRIDS = {"0.02 m": (0.02, RANGE), "0.01 m": (0.01, RANGE), "256^3": (0.0075, _cube((256,) * 3, 0.0075, LO)),
             "1024x64x64": (0.00176, _cube((1024, 64, 64), 0.00176, (-1.1, -0.55, -0.3)))}


@functools.lru_cache(maxsize=None)
def _lidar(n, beams=64, columns=1024):
    return workloads.tabletop_lidar(n, beams, columns)


@functools.lru_cache(maxsize=None)
def _depth_rays(n):
    """(points fp32 [n, H * W, 3] with NaN for invalid pixels, origins fp32 [n, 3], (depth, K, poses))."""
    import pytorch_volumetric_b200 as pv
    depth, K, poses = workloads.tabletop_views(n)
    pts, _ = pv.depth_to_points(torch.from_numpy(depth).cuda(), K, poses)
    return (pts.reshape(n, -1, 3).cpu().numpy(), np.ascontiguousarray(poses[:, :3, 3], np.float32),
            (depth, K, poses))


def _gpu_carve(P, O, per, res, rng, max_range=math.inf, margin=None):
    from pytorch_volumetric_b200 import _native as nat
    lo, dims = ray_ref.lattice(res, rng)
    margin = math.sqrt(3.0) * res / 2 if margin is None else margin
    p = torch.from_numpy(np.ascontiguousarray(P, np.float32).reshape(-1, 3)).cuda()
    o = torch.from_numpy(np.ascontiguousarray(O, np.float32).reshape(-1, 3)).cuda()
    marks = torch.zeros(dims, dtype=torch.uint8, device="cuda")
    out = torch.empty_like(p)
    nat.check(nat.lib().pvb_ray_carve(nat.ptr(p), p.shape[0], per, nat.ptr(o), max_range, margin,
                                      (ctypes.c_float * 3)(*lo), res, (ctypes.c_int32 * 3)(*dims), nat.ptr(marks),
                                      nat.ptr(out), None), "pvb_ray_carve")
    return marks.cpu().numpy(), out.cpu().numpy()


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


# ---------------------------------------------------------------- 1. bit for bit against the host build
def test_carve_equals_the_host_build_on_the_cpu_tier_rays():
    for grid, name, pts, org, max_range, margin in CASES:
        res, rng = GRIDS[grid]
        N = pts.shape[-2]
        want = ray_ref.host_carve(pts.reshape(-1, 3), org.reshape(-1, 3), N, res, rng, max_range, margin)
        got = _gpu_carve(pts, org, N, res, rng, max_range, margin)
        assert np.array_equal(got[0], want[0]), (grid, name)
        assert _same_bits(got[1], want[1]), (grid, name)


@pytest.mark.parametrize("grid", list(BIG_GRIDS))
def test_carve_equals_the_host_build_on_lidar_and_depth_rays(grid):
    res, rng = BIG_GRIDS[grid]
    pl, ol = _lidar(2)
    pd, od, _ = _depth_rays(4)
    for P, O in ((pl, ol), (pd, od)):
        N = P.shape[1]
        want = ray_ref.host_carve(P.reshape(-1, 3), O, N, res, rng)
        got = _gpu_carve(P, O, N, res, rng)
        assert (want[0] == 2).sum() > 1000
        assert np.array_equal(got[0], want[0])
        assert _same_bits(got[1], want[1])
    # max_range drops the far returns
    want = ray_ref.host_carve(pl.reshape(-1, 3), ol, pl.shape[1], res, rng, max_range=1.5)
    got = _gpu_carve(pl, ol, pl.shape[1], res, rng, max_range=1.5)
    assert np.array_equal(got[0], want[0]) and _same_bits(got[1], want[1])
    assert np.isnan(got[1]).any(1).sum() > np.isnan(pl).any(2).sum()


# ---------------------------------------------------------------- 2. depth frames as rays
@pytest.mark.parametrize("grid", ["0.02 m", "0.01 m"])
def test_depth_frames_as_rays_have_depth_occupancys_occupied_voxels(grid):
    import pytorch_volumetric_b200 as pv
    res, rng = BIG_GRIDS[grid]
    P, O, (depth, K, poses) = _depth_rays(4)
    got = pv.ray_occupancy(torch.from_numpy(P).cuda(), torch.from_numpy(O).cuda(), res, rng)
    want = pv.depth_occupancy(torch.from_numpy(depth).cuda(), K, poses, res, rng)
    assert got.is_cuda and got.dtype == torch.uint8
    assert torch.equal(got == 1, want == 1)
    assert (got == 0).sum() > 1000 and (got == 2).sum() > 1000


# ---------------------------------------------------------------- 3. one call on a fresh map
@pytest.mark.parametrize("params", [{}, OTHER], ids=["default", "other"])
@pytest.mark.parametrize("grid", list(BIG_GRIDS))
def test_fresh_map_reproduces_ray_occupancy_and_from_rays(grid, params):
    import pytorch_volumetric_b200 as pv
    res, rng = BIG_GRIDS[grid]
    pl, ol = _lidar(4)
    P, O = torch.from_numpy(pl).cuda(), torch.from_numpy(ol).cuda()
    m = pv.OccupancyMap(res, rng, device="cuda", **params)
    m.integrate_points(P, O)
    want = pv.ray_occupancy(P, O, res, rng)
    assert torch.equal(m.state(), want)
    assert (want == 0).any() and (want == 1).any() and (want == 2).any()
    assert not m._hits.get_voxel_values().view(torch.uint8).any()
    q = omr.quantize(**(omr.DEFAULTS | params))
    lo_ = m.log_odds()
    assert torch.equal(torch.isnan(lo_), want == 2)
    assert (lo_[want == 1] == q[0] / 1024).all() and (lo_[want == 0] == q[1] / 1024).all()
    if grid not in ("0.02 m", "1024x64x64") or params:
        return
    for unknown in ("occupied", "free"):
        for interp in ("nearest", "trilinear"):
            a = m.sdf(unknown=unknown, interpolation=interp)
            b = pv.OccupancySDF.from_rays(P, O, res, rng, unknown=unknown, interpolation=interp, device="cuda")
            assert torch.equal(a.occupancy, b.occupancy)
            assert torch.equal(a._table.view(torch.int32), b._table.view(torch.int32)), (unknown, interp)
    # unknown="free" is from_points of the valid returns
    valid = torch.isfinite(P).all(-1).reshape(-1)
    c = pv.OccupancySDF.from_points(P.reshape(-1, 3)[valid], res, rng, device="cuda")
    b = pv.OccupancySDF.from_rays(P, O, res, rng, unknown="free", device="cuda")
    assert torch.equal(b.occupancy, c.occupancy) and torch.equal(b._table.view(torch.int32),
                                                                 c._table.view(torch.int32))


# ---------------------------------------------------------------- 4. sequences, interleaved with depth frames
@pytest.mark.parametrize("params", [{}, OTHER], ids=["default", "other"])
def test_interleaved_sequences_equal_the_reference_replay(params):
    import pytorch_volumetric_b200 as pv
    r = 0.02
    q = omr.quantize(**(omr.DEFAULTS | params))
    m = pv.OccupancyMap(r, RANGE, device="cuda", **params)
    pl, ol = _lidar(6)
    noisy, on = workloads.tabletop_lidar(3, 32, 512, noise=0.01, seed=9)
    P, O, (depth, K, poses) = _depth_rays(4)
    calls = [("rays", pl[:2], ol[:2], math.inf), ("depth", depth[:2], poses[:2], math.inf),
             ("rays", pl[2:5], ol[2:5], 2.5), ("rays", noisy, on, math.inf), ("rays", P, O, math.inf),
             ("depth", depth[2:], poses[2:], 3.0)]
    calls += [("rays", pl[k:k + 1], ol[k:k + 1], math.inf) for k in range(6)] * 2
    calls += [("depth", depth, poses, math.inf)] * 6
    states = []
    for kind, a, b, mr in calls:
        if kind == "rays":
            a, b = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
            m.integrate_points(a, b, max_range=mr)
            states.append(pv.ray_occupancy(a, b, r, RANGE, max_range=mr).cpu().numpy())
        else:
            d = torch.from_numpy(a).cuda()
            m.integrate(d, K, b, max_depth=mr)
            states.append(pv.depth_occupancy(d, K, b, r, RANGE, max_depth=mr).cpu().numpy())
        assert not m._hits.get_voxel_values().view(torch.uint8).any()
    want = omr.replay(states, q)
    got = m.log_odds().cpu().numpy()
    assert np.array_equal(np.isnan(got), want == omr.UNOBSERVED)
    assert np.array_equal(got.view(np.uint32), omr.log_odds(want).view(np.uint32))
    assert np.array_equal(m.state().cpu().numpy(), omr.state(want, q))
    assert (want == q[3]).sum() > 1000 and (want == q[2]).sum() > 1000 and (want == omr.UNOBSERVED).any()


# ---------------------------------------------------------------- 5. determinism
def test_permuted_and_split_scans_give_the_same_bits():
    import pytorch_volumetric_b200 as pv
    r = 0.01
    pl, ol = _lidar(1, 128, 2048)
    P, O = torch.from_numpy(pl[0]).cuda(), torch.from_numpy(ol[0]).cuda()
    base = pv.ray_occupancy(P, O, r, RANGE)
    perm = torch.randperm(P.shape[0], generator=torch.Generator().manual_seed(3)).cuda()
    assert torch.equal(pv.ray_occupancy(P[perm], O, r, RANGE), base)
    V = 16
    split = pv.ray_occupancy(P.reshape(V, -1, 3), O.expand(V, 3).contiguous(), r, RANGE)
    assert torch.equal(split, base)
    maps = [pv.OccupancyMap(r, RANGE, device="cuda") for _ in range(3)]
    for _ in range(2):
        maps[0].integrate_points(P, O)
        maps[1].integrate_points(P[perm], O)
        maps[2].integrate_points(P.reshape(V, -1, 3), O.expand(V, 3).contiguous())
    assert torch.equal(maps[0]._log_odds, maps[1]._log_odds) and torch.equal(maps[0]._log_odds, maps[2]._log_odds)


# ---------------------------------------------------------------- 6. a box that leaves
MOVED_BOX = (-0.1, -0.1, -0.2, 0.2, 0.2, 0.3)


def test_a_box_that_leaves_turns_free_after_nine_scans():
    import pytorch_volumetric_b200 as pv
    r = 0.02
    q = omr.quantize(**omr.DEFAULTS)
    with_box = workloads.tabletop_lidar(4, 64, 1024, boxes=workloads.TABLETOP_ROOM + (MOVED_BOX,))
    without = workloads.tabletop_lidar(4, 64, 1024)
    W = [torch.from_numpy(a).cuda() for a in with_box]
    N = [torch.from_numpy(a).cuda() for a in without]
    m = pv.OccupancyMap(r, RANGE, device="cuda")
    for _ in range(6):
        m.integrate_points(*W)
    L = m.log_odds().cpu().numpy() * 1024
    after = pv.ray_occupancy(*N, r, RANGE).cpu().numpy()
    lo, dims = ray_ref.lattice(r, RANGE)
    c = lo + np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing="ij"), -1) * r
    blo, bhi = np.array(MOVED_BOX[:3]), np.array(MOVED_BOX[:3]) + np.array(MOVED_BOX[3:])
    in_box = ((c > blo - r) & (c < bhi + r)).all(-1)
    ghost = in_box & (L == q[3])
    carved = ghost & (after == 0)
    kept = ghost & (after != 0)
    assert carved.sum() > 50 and kept.sum() > 0, (int(carved.sum()), int(kept.sum()))
    for k in range(1, 13):
        m.integrate_points(*N)
        state = m.state().cpu().numpy()
        assert (state[carved] == (1 if k < 9 else 0)).all(), k
        assert (state[kept] == 1).all(), k


# ---------------------------------------------------------------- 7. no synchronisation
def test_integrate_points_does_not_synchronise():
    import pytorch_volumetric_b200 as pv
    pl, ol = _lidar(2)
    P, O = torch.from_numpy(pl).cuda(), torch.from_numpy(ol).cuda()
    m = pv.OccupancyMap(0.02, RANGE, device="cuda")
    m.integrate_points(P, O)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            m.integrate_points(P, O, max_range=5.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s0 = pv.ray_occupancy(P, O, 0.02, RANGE).cpu().numpy()
    s1 = pv.ray_occupancy(P, O, 0.02, RANGE, max_range=5.0).cpu().numpy()
    assert np.array_equal(m._log_odds.cpu().numpy(), omr.replay([s0] + [s1] * 3, omr.quantize(**omr.DEFAULTS)))
