"""CPU tier of the occupancy maps (OccupancyMap, pvb_depth_integrate).

1. occupancy_update of the host build (tests/hostsim/hostsim_occupancy_map.cpp) equals the numpy reference of
   tests/occupancy_map_ref.py on every int16 value and every observation, for parameter sets that reach both int16
   extremes and have hit = clamp_hi.
2. The host build of depth_integrate_kernel's per-voxel body equals depth_ref.host_carve plus the reference update on
   small tabletop grids, over sequences of calls, and clears the hit grid.
3. Parameter quantization and every ValueError, before any device work; the C entry point's refusals."""
import ctypes
import math

import numpy as np
import pytest

import depth_ref
import occupancy_map_ref as ref
import workloads
from hostsim_lib import PVB_ERR_INVALID

RANGE = workloads.TABLETOP_RANGE
PARAMS = [ref.quantize(**ref.DEFAULTS), (870, -410, -2048, 870, 1), (32767, -32767, -32767, 32767, 0),
          (1, -1, -32767, 32767, 1), (32767, -1, -1, 32767, 32767), (1, -32767, -32767, 1, -32766),
          (5000, -3000, -3000, 6000, 2500)]


# ---------------------------------------------------------------- 1. the update, exhaustively
@pytest.mark.parametrize("q", PARAMS)
def test_update_equals_the_reference_on_every_int16(q):
    L = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    for obs in (0, 1, 2):
        got = ref.host_update(L, obs, q)
        want = ref.update(L, np.full(L.shape, obs, np.uint8), q)
        assert np.array_equal(got, want), (obs, np.argwhere(got != want)[:5])
    hit, miss, lo, hi = q[:4]
    # a fresh voxel: one hit gives hit, one free observation miss; nothing leaves it unobserved
    assert ref.host_update(np.int16([ref.UNOBSERVED] * 3), np.uint8([1, 0, 2]), q).tolist() == [hit, miss,
                                                                                                  ref.UNOBSERVED]
    # observed values stay inside the clamps
    obs_L = L[(L >= lo) & (L <= hi)]
    for obs in (0, 1):
        out = ref.host_update(obs_L, obs, q)
        assert out.min() >= lo and out.max() <= hi


def test_update_reference_by_hand():
    q = ref.quantize(**ref.DEFAULTS)
    assert q == (870, -410, -2048, 3584, 0)
    L = np.int16([ref.UNOBSERVED, 0, 3000, 3584, -1900, -2048])
    assert ref.update(L, np.uint8([1] * 6), q).tolist() == [870, 870, 3584, 3584, -1030, -1178]
    assert ref.update(L, np.uint8([0] * 6), q).tolist() == [-410, -410, 2590, 3174, -2048, -2048]
    assert ref.update(L, np.uint8([2] * 6), q).tolist() == L.tolist()
    # from the upper clamp, the 9th free observation in a row crosses the default threshold: 3584 - 410 m < 0
    s = [np.uint8([0])] * 9
    assert ref.state(ref.replay([np.uint8([1])] * 5 + s[:8], q), q).tolist() == [1]
    assert ref.state(ref.replay([np.uint8([1])] * 5 + s, q), q).tolist() == [0]


# ---------------------------------------------------------------- 2. the per-voxel body
def _frames():
    """Tabletop frames at 120 x 160 from different rings, view counts, noise and masks."""
    out = []
    for k, (n, noise, masked) in enumerate([(1, 0.0, False), (3, 0.0, False), (2, 0.01, False), (4, 0.0, True),
                                            (1, 0.005, True), (5, 0.0, False)]):
        K, poses = workloads.camera_ring(n, (-0.25, 0.0, 0.2), 2.2, 1.3, 200.0, 120, 160, seed=10 + k)
        depth = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses, 120, 160, noise=noise, seed=k)
        if masked:
            depth[:, 40:90, 50:110] = 0.0
            depth[np.random.default_rng(k).random(depth.shape) < 0.05] = np.nan
        out.append((depth, K, poses))
    return out


@pytest.mark.parametrize("r,q", [(0.04, PARAMS[0]), (0.03, PARAMS[0]), (0.05, PARAMS[1]), (0.05, PARAMS[6])])
def test_integrate_body_equals_carve_plus_the_reference(r, q):
    lo, dims = depth_ref.lattice(r, RANGE)
    L = np.full(dims, ref.UNOBSERVED, np.int16)
    want = L.copy()
    g = np.random.default_rng(int(r * 1000))
    frames = _frames() * 2
    for k, (depth, K, poses) in enumerate(frames):
        carve = depth_ref.host_carve(depth, K, poses, r, RANGE)
        if k % 3 == 2:      # hits anywhere, carved voxels included: a hit wins
            hits = g.random(dims) < 0.05
        else:               # the voxels the fp64 points fall into
            pts, ok = depth_ref.points(depth, K, poses)
            hits = depth_ref.fuse(np.full(dims, 2, np.uint8), np.zeros(dims, bool), pts, ok, r, RANGE)[0] == 1
        L, cleared = ref.host_integrate(L, hits.astype(np.uint8), depth, K, poses, r, RANGE, q)
        assert not cleared.any()
        obs = np.where(hits, 1, carve)
        want = ref.update(want, obs, q)
        assert np.array_equal(L, want), (k, int((L != want).sum()))
    hit, miss, lo_c, hi_c = q[:4]
    assert (L == ref.UNOBSERVED).any() and (L == hi_c).any() and (L == lo_c).any()


def test_integrate_body_with_margin_and_max_depth():
    q = PARAMS[0]
    depth, K, poses = _frames()[1]
    lo, dims = depth_ref.lattice(0.04, RANGE)
    L0 = np.full(dims, ref.UNOBSERVED, np.int16)
    for max_depth, margin in ((2.5, 0.0), (math.inf, 0.1)):
        L, _ = ref.host_integrate(L0, np.zeros(dims, np.uint8), depth, K, poses, 0.04, RANGE, q, max_depth, margin)
        carve = depth_ref.host_carve(depth, K, poses, 0.04, RANGE, max_depth, margin)
        assert np.array_equal(L, ref.update(L0, carve, q)) and (carve == 0).any()


# ---------------------------------------------------------------- 3. parameters and refusals
def test_parameter_quantization():
    from pytorch_volumetric_b200.sdf import _occupancy_params
    assert tuple(_occupancy_params(0.85, -0.4, (-2.0, 3.5), 0.0)) == (870, -410, -2048, 3584, 0)
    # round(x * 1024): nearest, ties to even, like the reference's np.rint
    for hit, miss, clamp, thr in [(0.85, -0.4, (-2.0, 3.5), 0.0), (3 / 2048, -3 / 2048, (-5 / 2048, 5 / 2048), 0.0),
                                  (31.99, -31.99, (-31.999, 31.999), -31.0), (2.0, -0.25, (-1.0, 4.0), 1.0),
                                  (0.3333, -0.1111, (-0.7777, 0.9999), 0.0001)]:
        assert tuple(_occupancy_params(hit, miss, clamp, thr)) == ref.quantize(hit, miss, clamp, thr)
    # ties: 0.5 -> 0 would fail (hit must be positive); 1.5 -> 2, 2.5 -> 2, -2.5 -> -2
    assert tuple(_occupancy_params(2.5 / 1024, -2.5 / 1024, (-2.5 / 1024, 2.5 / 1024), 1.5 / 1024)) == (2, -2, -2, 2, 2)
    with pytest.raises(ValueError):
        _occupancy_params(0.5 / 1024, -0.4, (-2.0, 3.5), 0.0)


def test_parameter_value_errors_before_device_work():
    import pytorch_volumetric_b200 as pv
    bad = [dict(hit=0.0), dict(hit=-0.1), dict(miss=0.0), dict(miss=0.1), dict(hit=1 / 4096),      # rounds to 0
           dict(miss=-1 / 4096), dict(clamp=(-0.3, 3.5)), dict(clamp=(-2.0, 0.8)), dict(clamp=(-32.0, 3.5)),
           dict(clamp=(-2.0, 32.0)), dict(clamp=(-2.0,)), dict(clamp=(-2.0, 3.5, 4.0)), dict(threshold=-0.4),
           dict(threshold=0.86), dict(threshold=-1.0), dict(hit=math.nan), dict(miss=-math.inf),
           dict(clamp=(-2.0, math.inf)), dict(threshold=math.nan), dict(hit=1e300)]
    for kw in bad:
        with pytest.raises(ValueError):
            pv.OccupancyMap(0.05, RANGE, **kw)
    for kw in (dict(resolution=0.0), dict(resolution=math.nan), dict(resolution=0.001),
               dict(range_per_dim=[(0, 1), (0, 1), (0, 0)]), dict(free_margin=-0.01), dict(free_margin=math.inf)):
        with pytest.raises(ValueError):
            pv.OccupancyMap(**(dict(resolution=0.05, range_per_dim=RANGE) | kw))
    # the extremes that pass: hit = clamp_hi, clamps at +-32767, threshold = hit
    from pytorch_volumetric_b200.sdf import _occupancy_params
    assert tuple(_occupancy_params(31.999, -31.999, (-31.999, 31.999), 31.999)) == (32767, -32767, -32767, 32767,
                                                                                    32767)


def test_abi_refuses_invalid_inputs(built_lib):
    L = built_lib
    fake = ctypes.c_void_p(1 << 12)            # never dereferenced: every call below fails its argument checks
    V = 2
    intr = (ctypes.c_float * (4 * V))(*([500.0, 500.0, 319.5, 239.5] * V))
    rows = (ctypes.c_float * (12 * V))(*([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0] * V))
    lo = (ctypes.c_float * 3)(0, 0, 0)
    dims = (ctypes.c_int32 * 3)(10, 20, 30)
    good = (ctypes.c_int32 * 4)(870, -410, -2048, 3584)

    def call(depth=fake, V=V, H=480, W=640, intr=intr, rows=rows, max_depth=math.inf, margin=0.01, lo=lo, r=0.01,
             dims=dims, hits=fake, log_odds=fake, params=good):
        return L.pvb_depth_integrate(depth, V, H, W, intr, rows, max_depth, margin, lo, r, dims, hits, log_odds,
                                     params, None)

    def params(*p):
        return (ctypes.c_int32 * 4)(*p)

    intr0 = (ctypes.c_float * (4 * V))(*intr)
    intr0[0] = 0.0
    rows_nan = (ctypes.c_float * (12 * V))(*rows)
    rows_nan[3] = math.nan
    bad = [dict(V=0), dict(V=65), dict(H=0), dict(W=32769), dict(depth=None), dict(intr=None), dict(rows=None),
           dict(intr=intr0), dict(rows=rows_nan), dict(max_depth=0.0), dict(max_depth=math.nan), dict(dims=None),
           dict(dims=(ctypes.c_int32 * 3)(1, 20, 30)), dict(dims=(ctypes.c_int32 * 3)(10, 1025, 30)), dict(r=0.0),
           dict(r=math.inf), dict(margin=-0.01), dict(margin=math.nan), dict(lo=None),
           dict(lo=(ctypes.c_float * 3)(0, math.inf, 0)), dict(hits=None), dict(log_odds=None), dict(params=None),
           dict(params=params(0, -410, -2048, 3584)), dict(params=params(870, 0, -2048, 3584)),
           dict(params=params(870, -410, -409, 3584)), dict(params=params(870, -410, -2048, 869)),
           dict(params=params(870, -410, -32768, 3584)), dict(params=params(870, -410, -2048, 32768)),
           dict(params=params(-870, 410, 2048, -3584))]
    for kw in bad:
        assert call(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_depth_integrate"), kw
    assert b"clamp_lo <= miss" in (call(params=params(870, -410, -409, 3584)), L.pvb_last_error())[1]
    assert b"2..1024" in (call(dims=(ctypes.c_int32 * 3)(1, 20, 30)), L.pvb_last_error())[1]
    assert b"null" in (call(hits=None), L.pvb_last_error())[1]
