"""CPU tier of the depth-image scenes (pvb_depth_points, pvb_depth_carve, depth_to_points, depth_occupancy,
OccupancySDF.from_depth).

1. The host build of the device routines (tests/hostsim/hostsim_depth.cpp) against the fp64 reference of
   tests/depth_ref.py on rendered box scenes: every carve disagreement is a voxel the reference flags as ambiguous.
2. Back-projection against numpy within 1e-6 of the point's scale.
3. Views that see nothing (behind the camera, outside the frustum, every pixel invalid), V = 1 and V = 64.
4. The Python ValueErrors and the C entry points' refusals, without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import depth_ref
import workloads
from hostsim_lib import PVB_ERR_INVALID

RANGE = workloads.TABLETOP_RANGE


def _views(n, seed=0, H=120, W=160, f=200.0):
    return workloads.tabletop_views(n, H=H, W=W, f=f, seed=seed)


def _check_carve(depth, K, poses, r, rng=RANGE, max_depth=math.inf, margin=None):
    got = depth_ref.host_carve(depth, K, poses, r, rng, max_depth, margin)
    want, amb = depth_ref.carve(depth, K, poses, r, rng, max_depth, margin)
    bad = (got != want) & ~amb
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5])
    return got, want, amb


# ---------------------------------------------------------------- 1. carve against the fp64 reference
@pytest.mark.parametrize("n,r", [(1, 0.04), (4, 0.03), (4, 0.02), (8, 0.05)])
def test_carve_matches_the_fp64_reference(n, r):
    depth, K, poses = _views(n, seed=n)
    got, want, amb = _check_carve(depth, K, poses, r)
    assert (got == 0).any() and (got == 2).any()
    assert amb.mean() < 0.2
    # every view that says free, says so on a voxel in front of the surface: no voxel inside a box is carved
    lo, dims = depth_ref.lattice(r, RANGE)
    c = lo + np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing="ij"), -1) * r
    for b in workloads.TABLETOP_BOXES:
        blo, bhi = np.array(b[:3]), np.array(b[:3]) + np.array(b[3:])
        deep = ((c > blo + r) & (c < bhi - r)).all(-1)
        assert (got[deep] == 2).all()


def test_carve_with_a_margin_and_max_depth():
    depth, K, poses = _views(4, seed=9)
    for max_depth, margin in [(2.5, 0.0), (math.inf, 0.1), (3.0, 0.01)]:
        got, _, _ = _check_carve(depth, K, poses, 0.04, max_depth=max_depth, margin=margin)
        assert (got == 0).any()
    near, _, _ = _check_carve(depth, K, poses, 0.04, max_depth=2.0)
    far, _, _ = _check_carve(depth, K, poses, 0.04)
    assert ((near == 0) <= (far == 0)).all() and (near == 0).sum() < (far == 0).sum()


def test_carve_with_noisy_depth_and_masked_pixels():
    K, poses = workloads.camera_ring(3, (-0.25, 0.0, 0.2), 2.2, 1.3, 200.0, 120, 160, seed=4)
    depth = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses, 120, 160, noise=0.01, seed=4)
    g = np.random.default_rng(4)
    depth[g.random(depth.shape) < 0.1] = 0.0                             # masked out
    depth[g.random(depth.shape) < 0.02] = np.nan
    depth[g.random(depth.shape) < 0.02] = np.inf
    depth[g.random(depth.shape) < 0.02] = -1.0
    _check_carve(depth, K, poses, 0.03)


def test_fusion_is_the_or_of_the_views_in_any_order():
    depth, K, poses = _views(5, seed=2)
    every = depth_ref.host_carve(depth, K, poses, 0.05, RANGE)
    perm = [3, 0, 4, 2, 1]
    assert np.array_equal(depth_ref.host_carve(depth[perm], K, poses[perm], 0.05, RANGE), every)
    ones = [depth_ref.host_carve(depth[v:v + 1], K, poses[v:v + 1], 0.05, RANGE) for v in range(5)]
    assert np.array_equal(every == 0, np.logical_or.reduce([o == 0 for o in ones]))


# ---------------------------------------------------------------- 2. back-projection
@pytest.mark.parametrize("max_depth", [math.inf, 3.0])
def test_back_projection_against_numpy(max_depth):
    depth, K, poses = _views(3, seed=1)
    depth[0, :5] = np.nan
    depth[1, :, :3] = -2.0
    depth[2, 7] = np.inf
    got = depth_ref.host_points(depth, K, poses, max_depth)
    want, ok = depth_ref.points(depth, K, poses, max_depth)
    assert ok.any() and (~ok).any()
    assert np.isnan(got[~ok]).all() and np.isfinite(got[ok]).all()
    # relative to the point's scale: |p_cam| + |t| (a world point near the origin is a difference of such terms)
    V, H, W = depth.shape
    i, j = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    cam = np.stack([(j - K[0, 2]) * depth / K[0, 0], (i - K[1, 2]) * depth / K[1, 1], depth], -1)
    scale = np.linalg.norm(cam, axis=-1) + np.linalg.norm(poses[:, None, None, :3, 3], axis=-1)
    err = np.linalg.norm(got.astype(np.float64) - want, axis=-1)
    assert (err[ok] <= 1e-6 * scale[ok]).all(), float((err[ok] / scale[ok]).max())


# ---------------------------------------------------------------- 3. views that see nothing; V = 1 and V = 64
def test_views_that_see_nothing():
    r, rng = 0.05, RANGE
    K, _ = workloads.camera_ring(1, (0, 0, 0), 1.0, 0.0, 200.0, 120, 160)
    d = np.full((1, 120, 160), 1.0, np.float32)
    behind = workloads.look_at((3.0, 0.0, 0.2), (10.0, 0.0, 0.2))[None]          # the scene lies behind it
    aside = workloads.look_at((-0.25, 3.0, 0.2), (10.0, 3.0, 0.2))[None]          # beside it, outside the frustum
    for pose, depth in ((behind, d), (aside, d), (workloads.tabletop_views(1, 120, 160, 200.0)[2], 0 * d),
                        (workloads.tabletop_views(1, 120, 160, 200.0)[2], np.full_like(d, np.nan))):
        got, _, _ = _check_carve(depth, K, pose, r, rng)
        assert (got == 2).all()
        pts = depth_ref.host_points(depth, K, pose)
        if not depth_ref.valid(depth).any():
            assert np.isnan(pts).all()


def test_one_view_and_64_views():
    depth, K, poses = _views(64, seed=3, H=24, W=32, f=40.0)
    got, _, _ = _check_carve(depth, K, poses, 0.05)
    one, _, _ = _check_carve(depth[:1], K, poses[:1], 0.05)
    assert (one == 0).sum() < (got == 0).sum()
    assert ((one == 0) <= (got == 0)).all()


# ---------------------------------------------------------------- 4. refusals
def test_python_value_errors_before_device_work():
    import pytorch_volumetric_b200 as pv
    depth, K, poses = _views(2, H=12, W=16, f=20.0)
    d = torch.from_numpy(depth)
    P = torch.from_numpy(poses)
    r = 0.05
    skew = K.copy(); skew[0, 1] = 0.1
    bottom = K.copy(); bottom[2, 0] = 0.1
    last = K.copy(); last[2, 2] = 2.0
    lower = K.copy(); lower[1, 0] = 0.1
    neg_f = K.copy(); neg_f[0, 0] = -200.0
    nan_c = K.copy(); nan_c[0, 2] = np.nan
    scaled = P.clone(); scaled[0, :3, :3] *= 2
    bad_row = P.clone(); bad_row[1, 3, 0] = 1.0
    nan_t = P.clone(); nan_t[0, 0, 3] = np.nan
    mirror = P.clone(); mirror[0, :3, 0] *= -1
    bad = [
        dict(depth=d.double()), dict(depth=d[0]), dict(depth=torch.zeros(65, 4, 4)), dict(depth=torch.zeros(1, 0, 4)),
        dict(depth=torch.zeros(1, 4, 32769)), dict(K=skew), dict(K=bottom), dict(K=last), dict(K=lower),
        dict(K=neg_f), dict(K=nan_c), dict(K=np.stack([K] * 3)), dict(K=K[:2]), dict(cam_to_world=P[:1]),
        dict(cam_to_world=P[:, :3]), dict(cam_to_world=scaled), dict(cam_to_world=bad_row), dict(cam_to_world=nan_t),
        dict(cam_to_world=mirror), dict(max_depth=0.0), dict(max_depth=-1.0), dict(max_depth=float("nan")),
    ]
    for kw in bad:
        args = dict(depth=d, K=K, cam_to_world=P) | kw
        with pytest.raises(ValueError):
            pv.depth_to_points(**args)
        with pytest.raises(ValueError):
            pv.depth_occupancy(resolution=r, range_per_dim=RANGE, **args)
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_depth(resolution=r, range_per_dim=RANGE, **args)
    lattice_bad = [dict(resolution=0.0), dict(resolution=float("nan")), dict(resolution=-0.05),
                   dict(resolution=0.001), dict(range_per_dim=[(0, 1), (0, 1), (0, 0)]),
                   dict(range_per_dim=[(0, 1), (0, 1)]), dict(free_margin=-0.01), dict(free_margin=float("inf")),
                   dict(free_margin=float("nan"))]
    for kw in lattice_bad:
        args = dict(depth=d, K=K, cam_to_world=P, resolution=r, range_per_dim=RANGE) | kw
        with pytest.raises(ValueError):
            pv.depth_occupancy(**args)
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_depth(**args)
    for kw in (dict(unknown="seen"), dict(unknown=None), dict(interpolation="cubic")):
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_depth(d, K, P, r, RANGE, **kw)


def test_abi_refuses_invalid_inputs(built_lib):
    L = built_lib
    fake = ctypes.c_void_p(1 << 12)            # never dereferenced: every call below fails its argument checks
    V = 2
    intr = (ctypes.c_float * (4 * V))(*([500.0, 500.0, 319.5, 239.5] * V))
    rows = (ctypes.c_float * (12 * V))(*([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0] * V))
    lo = (ctypes.c_float * 3)(0, 0, 0)
    dims = (ctypes.c_int32 * 3)(10, 20, 30)

    def intr_with(k, value):
        a = (ctypes.c_float * (4 * V))(*intr)
        a[k] = value
        return a

    def rows_with(k, value):
        a = (ctypes.c_float * (12 * V))(*rows)
        a[k] = value
        return a

    shared = [dict(V=0), dict(V=65), dict(V=-1), dict(H=0), dict(W=0), dict(H=32769), dict(W=32769),
              dict(depth=None), dict(intr=None), dict(rows=None), dict(out=None),
              dict(intr=intr_with(0, 0.0)), dict(intr=intr_with(5, -1.0)), dict(intr=intr_with(4, math.nan)),
              dict(intr=intr_with(1, math.inf)), dict(intr=intr_with(2, math.nan)), dict(intr=intr_with(7, math.inf)),
              dict(rows=rows_with(3, math.nan)), dict(rows=rows_with(20, math.inf)),
              dict(max_depth=0.0), dict(max_depth=-1.0), dict(max_depth=math.nan)]

    def points(depth=fake, V=V, H=480, W=640, intr=intr, rows=rows, max_depth=math.inf, out=fake):
        return L.pvb_depth_points(depth, V, H, W, intr, rows, max_depth, out, None)

    def carve(depth=fake, V=V, H=480, W=640, intr=intr, rows=rows, max_depth=math.inf, margin=0.01, lo=lo, r=0.01,
              dims=dims, out=fake):
        return L.pvb_depth_carve(depth, V, H, W, intr, rows, max_depth, margin, lo, r, dims, out, None)

    for kw in shared:
        assert points(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_depth_points"), kw
    carve_only = [dict(dims=None), dict(dims=(ctypes.c_int32 * 3)(1, 20, 30)),
                  dict(dims=(ctypes.c_int32 * 3)(10, 1025, 30)), dict(r=0.0), dict(r=-0.01), dict(r=math.nan),
                  dict(r=math.inf), dict(margin=-0.01), dict(margin=math.nan), dict(margin=math.inf), dict(lo=None),
                  dict(lo=(ctypes.c_float * 3)(0, math.nan, 0))]
    for kw in shared + carve_only:
        assert carve(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_depth_carve"), kw
    assert b"1..64" in (carve(V=65), L.pvb_last_error())[1]
    assert b"2..1024" in (carve(dims=(ctypes.c_int32 * 3)(1, 20, 30)), L.pvb_last_error())[1]
    assert b"focal" in (points(intr=intr_with(0, 0.0)), L.pvb_last_error())[1]
    assert b"max_depth" in (carve(max_depth=math.nan), L.pvb_last_error())[1]
    assert b"free_margin" in (carve(margin=-1.0), L.pvb_last_error())[1]
