"""GPU: occupancy maps (OccupancyMap, pvb_depth_integrate).

1. A fresh map reproduces the one-call API: after one integrate, state() equals depth_occupancy of the same views bit
   for bit, and sdf()'s table equals OccupancySDF.from_depth's, on test_gpu_depth_occupancy's grids (a 1024-long axis
   included), for the default and a non-default parameter set.
2. Sequences of calls with different rings, view counts, noise and masked pixels: log_odds() and state() equal the
   reference replay (tests/occupancy_map_ref.py) over the per-call depth_occupancy states exactly, both clamps reached.
3. A box that leaves the scene: its voxels that later frames carve turn free at exactly the predicted frame count;
   those no later frame carves stay occupied.
4. Determinism: reversed views give the same bits, two maps fed the same calls agree, and the hit scratch is cleared.
5. integrate does not synchronise from the second call on.
6. 128 ring views in 8 calls of 16 equal the replay, and the map's sdf() as the cached arm's scene gives the same
   results on the fused and composition routes, as tests/test_gpu_scene.py requires."""
import functools

import numpy as np
import pytest
import torch

import occupancy_map_ref as ref
import workloads
from test_gpu_depth_occupancy import CASES, _cube

pytestmark = pytest.mark.gpu

RANGE = workloads.TABLETOP_RANGE
TARGET = (-0.25, 0.0, 0.2)
OTHER = dict(hit=2.0, miss=-0.25, clamp=(-1.0, 4.0), threshold=1.0)


@functools.lru_cache(maxsize=None)
def _views(n):
    return workloads.tabletop_views(n)


def _q(kw):
    return ref.quantize(**(ref.DEFAULTS | kw))


def _replay_check(m, calls, r, rng, q):
    """Feed `calls` [(depth, K, poses, max_depth)] to m; compare with the replay of the per-call depth_occupancy."""
    import pytorch_volumetric_b200 as pv
    states = []
    for depth, K, poses, max_depth in calls:
        d = torch.from_numpy(depth).cuda()
        m.integrate(d, K, poses, max_depth=max_depth)
        states.append(pv.depth_occupancy(d, K, poses, r, rng, max_depth=max_depth).cpu().numpy())
    want = ref.replay(states, q)
    got = m.log_odds().cpu().numpy()
    assert np.array_equal(np.isnan(got), want == ref.UNOBSERVED)
    assert np.array_equal(got.view(np.uint32), ref.log_odds(want).view(np.uint32))
    assert np.array_equal(m.state().cpu().numpy(), ref.state(want, q))
    return want, states


# ---------------------------------------------------------------- 1. one call on a fresh map
@pytest.mark.parametrize("params", [{}, OTHER], ids=["default", "other"])
@pytest.mark.parametrize("V,shape,r,lo", CASES)
def test_fresh_map_reproduces_the_one_call_api(V, shape, r, lo, params):
    import pytorch_volumetric_b200 as pv
    depth, K, poses = _views(V)
    rng = _cube(shape, r, lo)
    d = torch.from_numpy(depth).cuda()
    m = pv.OccupancyMap(r, rng, device="cuda", **params)
    assert m.shape == shape
    m.integrate(d, K, poses)
    state = m.state()
    assert state.is_cuda and state.dtype == torch.uint8
    want = pv.depth_occupancy(d, K, poses, r, rng)
    assert torch.equal(state, want)
    assert (want == 0).any() and (want == 1).any() and (want == 2).any()
    q = _q(params)
    lo_ = m.log_odds()
    assert torch.equal(torch.isnan(lo_), want == 2)
    assert (lo_[want == 1] == q[0] / 1024).all() and (lo_[want == 0] == q[1] / 1024).all()
    if shape == (64, 64, 64) or params:
        return      # the tables: once per grid, default parameters
    for unknown in ("occupied", "free"):
        for interp in ("nearest", "trilinear"):
            a = m.sdf(unknown=unknown, interpolation=interp)
            b = pv.OccupancySDF.from_depth(d, K, poses, r, rng, unknown=unknown, interpolation=interp, device="cuda")
            assert torch.equal(a.occupancy, b.occupancy)
            assert torch.equal(a._table.view(torch.int32), b._table.view(torch.int32)), (unknown, interp)
            assert np.array_equal(a.surface_bounding_box().numpy(), b.surface_bounding_box().numpy())


def test_results_on_the_maps_device_and_errors():
    import pytorch_volumetric_b200 as pv
    depth, K, poses = _views(1)
    m = pv.OccupancyMap(0.05, RANGE)
    assert m.state().device.type == "cpu" and (m.state() == 2).all() and torch.isnan(m.log_odds()).all()
    with pytest.raises(ValueError):
        m.sdf()                                      # one state only
    m.integrate(torch.from_numpy(depth), K, poses)   # host depth
    s = m.sdf(device="cuda")
    assert s.device == "cuda"
    with pytest.raises(ValueError):
        m.sdf(unknown="seen")
    with pytest.raises(ValueError):
        m.sdf(interpolation="cubic")
    with pytest.raises(ValueError):
        m.integrate(torch.from_numpy(depth).double(), K, poses)
    m.reset()
    assert (m.state() == 2).all()


# ---------------------------------------------------------------- 2. sequences
def _sequence():
    """16 calls: rings with different seeds and view counts, a noisy frame, a frame with masked and invalid pixels, a
    max_depth, and the same four views repeated (into the upper clamp where they hit, the lower where they carve)."""
    calls = []
    for k, n in enumerate([1, 3, 2, 5, 1, 4, 2, 8]):
        K, poses = workloads.camera_ring(n, TARGET, 2.2, 1.3, 800.0, seed=20 + k)
        calls.append((workloads.render_depth(workloads.TABLETOP_BOXES, K, poses), K, poses, float("inf")))
    K, poses = workloads.camera_ring(3, TARGET, 2.0, 1.5, 700.0, seed=40)
    calls.append((workloads.render_depth(workloads.TABLETOP_BOXES, K, poses, noise=0.01, seed=3), K, poses,
                  float("inf")))
    K, poses = workloads.camera_ring(2, TARGET, 2.4, 1.0, 800.0, seed=41)
    masked = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses)
    masked[:, 150:330, 200:450] = 0.0
    masked[:, ::7, ::5] = np.nan
    calls.append((masked, K, poses, 3.0))
    depth, K, poses = _views(4)
    calls += [(depth, K, poses, float("inf"))] * 6
    return calls


@pytest.mark.parametrize("params", [{}, OTHER], ids=["default", "other"])
def test_sequences_equal_the_reference_replay(params):
    import pytorch_volumetric_b200 as pv
    r = 0.02
    q = _q(params)
    m = pv.OccupancyMap(r, RANGE, device="cuda", **params)
    want, states = _replay_check(m, _sequence(), r, RANGE, q)
    assert (want == q[3]).sum() > 1000 and (want == q[2]).sum() > 1000 and (want == ref.UNOBSERVED).any()
    # voxels that changed their mind: hit in one call, free in another
    s = np.stack(states)
    assert ((s == 1).any(0) & (s == 0).any(0)).sum() > 100


# ---------------------------------------------------------------- 3. a box that leaves
MOVED_BOX = (-0.1, -0.1, -0.2, 0.2, 0.2, 0.3)


def test_a_box_that_leaves_turns_free_at_the_predicted_frame():
    import pytorch_volumetric_b200 as pv
    r = 0.02
    q = _q({})
    K, poses = workloads.camera_ring(4, TARGET, 2.2, 1.3, 800.0, seed=7)
    with_box = torch.from_numpy(workloads.render_depth(workloads.TABLETOP_BOXES + (MOVED_BOX,), K, poses)).cuda()
    without = torch.from_numpy(workloads.render_depth(workloads.TABLETOP_BOXES, K, poses)).cuda()
    m = pv.OccupancyMap(r, RANGE, device="cuda")
    n_with = 6
    for _ in range(n_with):
        m.integrate(with_box, K, poses)
    L = m.log_odds().cpu().numpy() * 1024
    after = pv.depth_occupancy(without, K, poses, r, RANGE).cpu().numpy()
    lo, dims = np.array([min(a) for a in pv.VoxelGrid(r, RANGE).range_per_dim]), m.shape
    c = lo + np.stack(np.meshgrid(*[np.arange(k) for k in dims], indexing="ij"), -1) * r
    blo, bhi = np.array(MOVED_BOX[:3]), np.array(MOVED_BOX[:3]) + np.array(MOVED_BOX[3:])
    in_box = ((c > blo - r) & (c < bhi + r)).all(-1)
    ghost = in_box & (L == q[3])                      # saturated by the box
    carved = ghost & (after == 0)
    kept = ghost & (after != 0)
    assert carved.sum() > 100 and kept.sum() > 0, (int(carved.sum()), int(kept.sum()))
    # 3584 - 410 m < 0 first at m = 9
    m_free = -(-(q[3] - q[4] + 1) // -q[1])
    assert m_free == 9
    for k in range(1, 13):
        m.integrate(without, K, poses)
        state = m.state().cpu().numpy()
        assert (state[carved] == (1 if k < m_free else 0)).all(), k
        assert (state[kept] == 1).all(), k


# ---------------------------------------------------------------- 4. determinism
def test_view_order_repeat_and_the_cleared_hit_scratch():
    import pytorch_volumetric_b200 as pv
    r = 0.02
    depth, K, poses = _views(16)
    d = torch.from_numpy(depth).cuda()
    a, b, c = (pv.OccupancyMap(r, RANGE, device="cuda") for _ in range(3))
    calls = [(d[:8], poses[:8]), (d[8:], poses[8:]), (d[3:11], poses[3:11])]
    for dd, pp in calls:
        a.integrate(dd, K, pp)
        b.integrate(dd, K, pp)
        c.integrate(dd.flip(0), K, pp[::-1].copy())
    La, Lb, Lc = (x._log_odds.clone() for x in (a, b, c))
    assert torch.equal(La, Lb) and torch.equal(La, Lc)
    # a call that observes nothing: every pixel invalid.  A voxel hit in the last call gets no second hit.
    a.integrate(torch.zeros_like(d[:2]), K, poses[:2])
    assert torch.equal(a._log_odds, La)
    assert not a._hits.get_voxel_values().any()


# ---------------------------------------------------------------- 5. no synchronisation
def test_integrate_does_not_synchronise():
    import pytorch_volumetric_b200 as pv
    depth, K, poses = _views(4)
    d = torch.from_numpy(depth).cuda()
    m = pv.OccupancyMap(0.02, RANGE, device="cuda")
    m.integrate(d, K, poses)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            m.integrate(d, K, poses)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = ref.replay([pv.depth_occupancy(d, K, poses, 0.02, RANGE).cpu().numpy()] * 4, _q({}))
    assert np.array_equal(m._log_odds.cpu().numpy(), want)


# ---------------------------------------------------------------- 6. beyond 64 views, as a scene
def test_128_views_in_8_calls_as_a_scene(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    from test_gpu_scene import _check, _per_point, robot_of
    K, poses = workloads.camera_ring(128, TARGET, 2.2, 1.3, 400.0, H=240, W=320, seed=5)
    depth = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses, H=240, W=320)
    rng, r = [[-1.6, 1.2], [-1.2, 1.2], [-0.5, 1.6]], 0.02
    m = pv.OccupancyMap(r, rng, device="cuda")
    calls = [(depth[16 * k:16 * (k + 1)], K, poses[16 * k:16 * (k + 1)], float("inf")) for k in range(8)]
    _replay_check(m, calls, r, rng, _q({}))
    robot, q = robot_of(tmp_path, "nearest")
    robot.set_joint_configuration(q)
    lp = robot.link_surface_points(num_points=256, seed=1)
    S = lp.shape[0]
    seen = False
    for interp in ("nearest", "trilinear"):
        scene = m.sdf(interpolation=interp, device="cuda")
        robot.set_joint_configuration(q)
        _, _, _, g = _per_point(robot.sdf, scene, lp, [True] * S)
        keep = torch.isfinite(g).flatten(1).all(1)       # see test_gpu_depth_occupancy: the range's shell
        assert int(keep.sum()) >= 0.75 * len(q), int(keep.sum())
        robot.set_joint_configuration(q[keep])
        for mg in (0.02, 0.1):
            _, cost = _check(monkeypatch, robot, scene, lp, None, mg, ("map", interp, mg))
            seen |= bool((cost[0] > 0).any())
    assert seen
