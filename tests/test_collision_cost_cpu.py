"""CPU tier for collision-cost queries (ComposedSDF.collision_cost / RobotSDF.collision_cost /
pvb_composed_query_collision_cost): for every configuration and every segment of points, the hinge cost
sum_p max(0, m - d)^2 and its twist gradient per sub-SDF, and for a robot its joint gradient.

1. The device arithmetic, compiled for the host by tests/hostsim/hostsim_collision_cost.cpp in the order
   robot_collision_cost_kernel and collision_cost_finish_kernel run it, on the nearest, trilinear, mixed, drill,
   primitive and primitive+grid golden sets, under several chunk sizes, accumulator counts, tile widths (lanes) and unit
   orders:
   - every pair the sequence evaluates has the per-pair query's value, gradient and sub-SDF, bit for bit, and no pair
     whose value is below the margin is skipped (instrumented: every pair reports whether it was evaluated);
   - cost and every twist component are within 1e-5 * sum|term| of the fp64 sum of the per-pair query's outputs;
   - at a fixed seg_len the results do not depend on the unit order, the tile width or the configuration slab.
2. The joint-gradient algebra, without a GPU: on the `mixed` chain of test_gpu_robot_fp64.py (oblique unnormalised
   axes, a continuous and a prismatic joint, fixed joints, visual offsets) with primitive links, RobotSDF.joint_twists,
   joint_moves_link and joint_gradient applied to the fp64 twist gradient of robot_ref.RefRobot equal central finite
   differences of the fp64 cost in q, over the points whose argmin link and shape rule stay put over the step.
3. The C ABI refusals and the Python shape and margin rules, without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from hostsim_lib import PVB_ERR_INVALID, _p
from pytorch_volumetric_b200 import _native as nat
from robot_ref import build_robot, joint_values


def _fused(descs, xforms, n_cfg, points, n_seg, margin, cfg_begin=0, cfg_count=None, chunk=0, n_acc=8, lanes=32,
           unit_order=0, shuffle_seed=0, first=-1):
    """robot_collision_cost_kernel + collision_cost_finish_kernel on the host: (cost [R], twist [R, S, 6], and per
    pair of the slab: visited, value, gradient, sub-SDF, plus the number of lookups)."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    seg_len = len(p) // n_seg
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    R, NP = cfg_count * n_seg, cfg_count * len(p)
    cost, twist = np.empty(R, np.float32), np.empty((R, S, 6), np.float32)
    visited, pv, pg, pw = np.empty(NP, np.uint8), np.empty(NP, np.float32), np.empty((NP, 3), np.float32), \
        np.empty(NP, np.int32)
    evals = ctypes.c_longlong(0)
    hs.lib().simcc_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                         ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(seg_len),
                         ctypes.c_float(margin), ctypes.c_int(chunk), ctypes.c_int(n_acc), ctypes.c_int(lanes),
                         ctypes.c_int(unit_order), ctypes.c_int(shuffle_seed), ctypes.c_int(first), _p(cost),
                         _p(twist), _p(visited), _p(pv), _p(pg), _p(pw), ctypes.byref(evals))
    return cost, twist, visited.astype(bool), pv, pg, pw, evals.value


def _fp64_cost(v, g, w, pts, m, S):
    """The fp64 composition: cost [..., n_seg], twist [..., n_seg, S, 6] and the sums of |term| of both, from
    per-pair values v [..., n_seg, L], gradients g [..., n_seg, L, 3], sub-SDFs w and points pts [n_seg, L, 3]."""
    v, g = np.asarray(v, np.float64), np.asarray(g, np.float64)
    pts = np.asarray(pts, np.float64)
    h = np.maximum(m - v, 0.0)
    terms = np.concatenate([g, np.cross(np.broadcast_to(pts, g.shape), g)], axis=-1) * (2.0 * h)[..., None]
    onehot = (w[..., None] == np.arange(S)).astype(np.float64)                  # [..., L, S]
    twist = np.einsum("...ls,...lk->...sk", onehot, terms)
    abs_tw = np.einsum("...ls,...lk->...sk", onehot, np.abs(terms))
    return (h * h).sum(-1), twist, (h * h).sum(-1), abs_tw


def _check_within(cost, twist, ref, what):
    rc, rt, ac, at = ref
    assert (np.abs(cost - rc) <= 1e-5 * ac + 1e-30).all(), (what, "cost", float(np.abs(cost - rc).max()))
    assert (np.abs(twist - rt) <= 1e-5 * at + 1e-30).all(), (what, "twist", float(np.abs(twist - rt).max()))


def _margins(v):
    """Two margins that leave some pairs inside and most outside, and one below 0 when some value is negative."""
    ms = [np.quantile(v, 0.05), np.quantile(v, 0.3)] + ([np.quantile(v[v < 0], 0.5)] if (v < 0).sum() > 10 else [])
    return [float(np.float32(m)) for m in ms]                   # the fp32 margin the kernel computes with


# ---------------------------------------------------------------- 1. the kernels' sequence
def test_chunk_rule_depends_on_seg_len_alone():
    L = hs.lib()
    for n in (1, 7, 511, 512, 513, 1000, 4096, 131072, 131073, 10 ** 5, 10 ** 6, (1 << 31) - 1):
        c, k = L.simcc_chunk(n), L.simcc_chunks(n)
        assert 1 <= c <= n and k == -(-n // c) and k <= 256, n
        assert c == n or c % 512 == 0, n
    assert L.simcc_chunks(0) == 0


@pytest.mark.parametrize("A", [7, 40])
def test_fused_cost_equals_the_fp64_composition(built_lib, A):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else hs.trajectory(zc["tmat"], S, A0, A, seed=A)
    for n_seg in (1, 4):
        q = np.asarray(zc["q"], dtype=np.float32)[: (len(zc["q"]) // n_seg) * n_seg]
        L = len(q) // n_seg
        pts = q.reshape(n_seg, L, 3)
        for name, descs in sets:
            v, g, w = hs.composed(descs, tm, A, q, ext=True)
            v, g, w = v.reshape(A, n_seg, L), g.reshape(A, n_seg, L, 3), w.reshape(A, n_seg, L)
            for m in _margins(v):
                what = (name, A, n_seg, m)
                cost, twist, vis, pv, pg, pw, evals = _fused(descs, tm, A, q, n_seg, m)
                vis, pv, pg, pw = vis.reshape(A, n_seg, L), pv.reshape(A, n_seg, L), pg.reshape(A, n_seg, L, 3), \
                    pw.reshape(A, n_seg, L)
                inside = v < m
                assert inside.any() and (~inside).any(), what
                # no pair below the margin is skipped, and every evaluated pair below it is the per-pair query's
                assert vis[inside].all(), what
                assert np.array_equal(pv[inside], v[inside]) and np.array_equal(pw[inside], w[inside]), what
                assert np.array_equal(pg[inside], g[inside]), what
                # an evaluated pair at or above the margin may be inexact, but is never below it
                assert not ((pw >= 0) & ~inside & (pv < m)).any(), what
                ref = _fp64_cost(v, g, w, pts, m, S)
                _check_within(cost.reshape(A, n_seg), twist.reshape(A, n_seg, S, 6), ref, what)
                # pruning is static: far fewer lookups than pairs x links
                assert evals < A * len(q) * S, what
                # unit orders, tile widths and the first visit change nothing at a fixed seg_len
                for kw in (dict(unit_order=1), dict(unit_order=2, shuffle_seed=3), dict(lanes=8), dict(lanes=1),
                           dict(first=S - 1, unit_order=1)):
                    c2, t2 = _fused(descs, tm, A, q, n_seg, m, **kw)[:2]
                    assert np.array_equal(c2, cost) and np.array_equal(t2, twist), (what, kw)
                # other chunk sizes and accumulator counts: other summation orders, within the same bound
                for kw in (dict(chunk=7), dict(chunk=64, n_acc=1), dict(chunk=L, n_acc=3)):
                    c2, t2 = _fused(descs, tm, A, q, n_seg, m, **kw)[:2]
                    _check_within(c2.reshape(A, n_seg), t2.reshape(A, n_seg, S, 6), ref, (what, kw))


def test_slabs_reproduce_the_rows_of_the_full_call(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    A = 70
    tm = hs.trajectory(zc["tmat"], S, A0, A, seed=11)
    q = np.asarray(zc["q"], dtype=np.float32)[:3000]
    for name, descs in sets:
        v = hs.composed(descs, tm, A, q, ext=True)[0]
        m = float(np.float32(np.quantile(v, 0.2)))
        cost, twist = _fused(descs, tm, A, q, 3, m)[:2]
        for begin, count in ((0, 1), (5, 32), (31, 2), (33, 37), (69, 1), (1, 69)):
            c2, t2 = _fused(descs, tm, A, q, 3, m, cfg_begin=begin, cfg_count=count)[:2]
            rows = slice(begin * 3, (begin + count) * 3)
            assert np.array_equal(c2, cost[rows]) and np.array_equal(t2, twist[rows]), (name, begin, count)


def test_far_clouds_cost_exactly_zero(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A = int(zc["S"]), int(zc["A"])
    q = np.asarray(zc["q"], dtype=np.float32)[:500] + np.float32(50.0)
    for name, descs in sets:
        cost, twist, vis, pv, pg, pw, evals = _fused(descs, zc["tmat"], A, q, 1, 0.05)
        assert not cost.any() and not twist.any(), name
        assert not vis.any() and evals == 0, name                 # every point skipped by its bounds


def test_unit_orders_and_duplicates_give_identical_rows(built_lib):
    """Duplicated configurations get identical rows whatever lane and tile they land in."""
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    base = hs.trajectory(zc["tmat"], S, A0, 5, seed=2).reshape(S, 5, 4, 4)
    tm = np.concatenate([base] * 9, axis=1)                       # 45 configurations: 5 repeated 9 times
    A = tm.shape[1]
    tm = tm.reshape(S * A, 4, 4)
    q = np.asarray(zc["q"], dtype=np.float32)[:1200]
    for name, descs in sets:
        v = hs.composed(descs, tm, A, q, ext=True)[0]
        m = float(np.float32(np.quantile(v, 0.25)))
        cost, twist = _fused(descs, tm, A, q, 2, m, unit_order=2, shuffle_seed=5)[:2]
        cost, twist = cost.reshape(A, 2), twist.reshape(A, 2, S, 6)
        for a in range(5, A):
            assert np.array_equal(cost[a], cost[a % 5]) and np.array_equal(twist[a], twist[a % 5]), (name, a)


# ---------------------------------------------------------------- 2. the joint gradient of a serial chain
def _mixed(tmp_path):
    robot, ref, text = build_robot("mixed", tmp_path, dtype=torch.float64, device="cpu")
    return robot, ref, text


def _ref_cost_terms(ref, q, pts, m):
    """fp64 per-point (value, robot-frame gradient, link, gap to the shape rule, second-best value) at joint values q
    [A, J] for points [P, 3]."""
    per = ref.evaluate(ref.object_to_link(q), pts)
    v, g, w = ref.compose(per)
    vals = np.sort(per["value"], axis=0)
    gap = np.take_along_axis(per["gap"], w[None], 0)[0]
    return v, g, w, gap, vals[1]


def test_joint_gradient_equals_finite_differences(tmp_path):
    robot, ref, text = _mixed(tmp_path)
    J, S = len(robot.joint_names), len(robot.sdf_to_link_name)
    assert J == ref.n_joints and S == len(ref.links)
    qs = joint_values(ref, text, 4, seed=7).astype(np.float64)
    robot.set_joint_configuration(torch.from_numpy(qs))
    twists = robot.joint_twists().numpy()                           # [A, J, 6]
    moves = robot.joint_moves_link()
    assert twists.shape == (4, J, 6) and tuple(moves.shape) == (J, S)
    # the move mask of a serial chain: a joint moves every link at or after its frame
    frame_of_link = [l.frame for l in ref.links]
    frame_of_joint = [f for f, t in enumerate(ref.types) if t != "fixed"]
    assert moves.tolist() == [[fj <= fs for fs in frame_of_link] for fj in frame_of_joint]
    rng = np.random.default_rng(3)
    pts = rng.uniform(-0.45, 0.45, (6000, 3)) + np.array([0.0, 0.0, 0.45])
    # the reference rounds joint values to fp32: a step of 2^-16 keeps q +- h exact for |q| < 64
    m, h = 0.06, 2.0 ** -16
    checked = 0
    for a in range(len(qs)):
        v, g, w, gap, second = _ref_cost_terms(ref, qs[a:a + 1], pts, m)
        v, g, w, gap, second = v[0], g[0], w[0], gap[0], second[0]
        hinge = np.maximum(m - v, 0.0)
        terms = np.concatenate([g, np.cross(pts, g)], axis=1) * (2.0 * hinge)[:, None]
        twist = np.stack([terms[w == s].sum(0) for s in range(S)])           # [S, 6]
        grad = robot.joint_gradient(torch.from_numpy(twist[None, None]), torch.from_numpy(twists[a:a + 1]),
                                    moves).numpy()[0, 0]
        # central differences of the cost over the points whose link and shape rule stay put over the step
        stable = (gap > 1e-3) & (second - v > 1e-3) & (v < m + 1e-2)
        for j in range(J):
            qp, qm = qs[a:a + 1].copy(), qs[a:a + 1].copy()
            qp[0, j] += h
            qm[0, j] -= h
            vp, _, wp, _, _ = (x[0] for x in _ref_cost_terms(ref, qp, pts, m))
            vm, _, wm, _, _ = (x[0] for x in _ref_cost_terms(ref, qm, pts, m))
            keep = stable & (wp == w) & (wm == w)
            fd = ((np.maximum(m - vp, 0) ** 2 - np.maximum(m - vm, 0) ** 2)[keep]).sum() / (2 * h)
            # the analytic gradient restricted to the same points
            tw_k = np.stack([terms[keep & (w == s)].sum(0) for s in range(S)])
            an = robot.joint_gradient(torch.from_numpy(tw_k[None, None]), torch.from_numpy(twists[a:a + 1]),
                                      moves).numpy()[0, 0, j]
            scale = np.abs(terms[keep]).sum() * (1.0 + np.abs(twists[a, j]).max()) + 1e-12
            assert abs(fd - an) <= 1e-5 * scale, (a, j, fd, an, scale)
            checked += int(keep.sum())
        assert np.isfinite(grad).all() and grad.shape == (J,)
    assert checked > 1000


def test_joint_twists_follow_the_configuration(tmp_path):
    robot, ref, text = _mixed(tmp_path)
    q1 = torch.zeros(3, len(robot.joint_names), dtype=torch.float64)
    robot.set_joint_configuration(q1)
    t1 = robot.joint_twists()
    assert robot.joint_twists() is t1                               # cached with the configuration
    robot.set_joint_configuration(q1 + 0.3)
    t2 = robot.joint_twists()
    assert t2 is not t1 and not torch.equal(t1, t2)
    # prismatic joints rotate nothing; revolute twists are unit rotations with v = -w x t
    kinds = [t for t in ref.types if t != "fixed"]
    for j, k in enumerate(kinds):
        if k == "prismatic":
            assert torch.equal(t2[:, j, 3:], torch.zeros_like(t2[:, j, 3:]))
            assert torch.allclose(t2[:, j, :3].norm(dim=-1), torch.ones(3, dtype=torch.float64))
        else:
            assert torch.allclose(t2[:, j, 3:].norm(dim=-1), torch.ones(3, dtype=torch.float64))
            assert torch.allclose((t2[:, j, :3] * t2[:, j, 3:]).sum(-1), torch.zeros(3, dtype=torch.float64),
                                  atol=1e-12)


# ---------------------------------------------------------------- 3. C ABI refusals and Python rules (no device)
def test_abi_refuses_invalid_collision_cost_queries(built_lib):
    near, tri, keep = hs.table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_seg=10, seg_len=100, margin=0.05,
             ws=fake, ws_bytes=1 << 40, cost=fake, twist=fake):
        return L.pvb_composed_query_collision_cost(descs, n_sdf, xf, n_cfg, begin, count, pts, n_seg, seg_len, margin,
                                                   ws, ws_bytes, cost, twist, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    mesh = near.copy()
    mesh.kind = nat.PVB_KIND_MESH
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(cost=None), dict(twist=None), dict(ws=None),
             dict(ws_bytes=0), dict(ws=ctypes.c_void_p((1 << 12) + 2)), dict(n_sdf=0), dict(n_cfg=0), dict(begin=-1),
             dict(count=-1), dict(count=0), dict(begin=2, count=3), dict(n_seg=-1), dict(seg_len=-1),
             dict(seg_len=1 << 31, n_seg=1), dict(n_seg=1 << 62, seg_len=4), dict(margin=float("nan")),
             dict(margin=float("inf")), dict(margin=-float("inf")),
             dict(descs=nat.desc_array([near] * 9), n_sdf=9), dict(descs=nat.desc_array([near, gt])),
             dict(descs=nat.desc_array([near, mesh])), dict(seg_len=0, cost=None)]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_collision_cost"), (kw, msg)
    assert b"finite" in (call(margin=float("nan")), L.pvb_last_error())[1]
    assert b"workspace" in (call(ws_bytes=8), L.pvb_last_error())[1]
    assert b"compose" in (call(descs=nat.desc_array([near] * 9), n_sdf=9), L.pvb_last_error())[1]
    assert b"configurations" in (call(count=0), L.pvb_last_error())[1]
    # nothing to do: no segments, or no configurations and no points
    assert call(n_seg=0, pts=None, ws=None, ws_bytes=0, cost=None, twist=None) == 0
    assert call(seg_len=0, count=0, pts=None, ws=None, ws_bytes=0, cost=None, twist=None) == 0
    # the workspace size: one fp32 row of 1 + 6 n_sdf per (configuration, segment, chunk)
    W = L.pvb_collision_cost_workspace
    assert W(2, 4, 10, 100) == 4 * 4 * 10 * 1 * 13
    assert W(8, 200, 1, 10 ** 5) == 4 * 200 * 1 * hs.lib().simcc_chunks(10 ** 5) * 49
    assert W(3, 5, 7, 0) == 0 and W(0, 1, 1, 1) == -1 and W(1, -1, 1, 1) == -1 and W(8, 1 << 30, 1 << 40, 1 << 30) == -1


def test_collision_cost_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(3,))
    for shape in ((5, 2), (3,), (4, 5, 4), (), (0,)):
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.collision_cost(torch.zeros(shape), 0.1)
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.query_collision_cost(torch.zeros(shape), 0.1)
    for margin in (float("nan"), float("inf"), -math.inf, "x", None, torch.tensor([0.1, 0.2])):
        with pytest.raises(ValueError, match="margin"):
            comp.collision_cost(torch.zeros(10, 3), margin)
        with pytest.raises(ValueError, match="margin"):
            comp.query_collision_cost(torch.zeros(10, 3), margin)
    for begin, count in ((1, 0), (-1, 2), (2, 2)):
        with pytest.raises(ValueError, match="configuration slab"):
            comp.query_collision_cost(torch.zeros(10, 3), 0.1, cfg_begin=begin, cfg_count=count)
