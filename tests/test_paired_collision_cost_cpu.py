"""CPU tier for paired collision-cost queries (ComposedSDF.paired_collision_cost / RobotSDF.paired_collision_cost /
pvb_composed_query_paired_collision_cost): every configuration's hinge cost over its OWN cloud and its twist gradient.

1. The device arithmetic, compiled for the host by tests/hostsim/hostsim_paired_collision_cost.cpp in the order
   robot_paired_collision_cost_kernel and collision_cost_finish_kernel run it, on the nearest, trilinear, mixed, drill,
   primitive and primitive+grid golden sets, at segment lengths on both sides of a warp step and of a chunk:
   - row (a, b) equals the shared-cloud sequence (tests/hostsim/hostsim_collision_cost.cpp) of configuration a alone
     over points[a], bit for bit in cost and twist, under every unit order, a forced first link and forced chunks;
   - every pair the sequence evaluates has the per-pair query's value, gradient and sub-SDF, bit for bit, and no pair
     whose value is below the margin is skipped;
   - cost and every twist component are within 1e-5 * sum|term| of the fp64 sum of the per-pair query's outputs;
   - clouds far from every link cost exactly 0 without a single lookup.
2. The C ABI refusals and the Python shape and margin rules, without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from hostsim_lib import PVB_ERR_INVALID, _p
from pytorch_volumetric_b200 import _native as nat


def _pcc_fused(descs, xforms, n_cfg, own, margin, cfg_begin=0, chunk=0, unit_order=0, shuffle_seed=0, first=-1):
    """robot_paired_collision_cost_kernel + collision_cost_finish_kernel on the host (simpcc_fused, built into
    hs.lib() with every tests/hostsim/*.cpp); own [cfg_count, n_seg, L, 3].  Returns (cost [R], twist [R, S, 6], and
    per pair of the slab: visited, value, gradient, sub-SDF, plus the number of lookups), R = cfg_count * n_seg."""
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    R, NP = cfg_count * n_seg, cfg_count * n_seg * L
    cost, twist = np.empty(R, np.float32), np.empty((R, S, 6), np.float32)
    visited, pv, pg, pw = np.empty(NP, np.uint8), np.empty(NP, np.float32), np.empty((NP, 3), np.float32), \
        np.empty(NP, np.int32)
    evals = ctypes.c_longlong(0)
    hs.lib().simpcc_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                          ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                          ctypes.c_float(margin), ctypes.c_int(chunk), ctypes.c_int(unit_order),
                          ctypes.c_int(shuffle_seed), ctypes.c_int(first), _p(cost), _p(twist), _p(visited), _p(pv),
                          _p(pg), _p(pw), ctypes.byref(evals))
    return cost, twist, visited.astype(bool), pv, pg, pw, evals.value


def _single(descs, xforms, n_cfg, a, points, n_seg, margin, chunk=0):
    """The shared-cloud sequence (simcc_fused) of configuration a alone over points [n_seg * L, 3]: (cost [n_seg],
    twist [n_seg, S, 6]).  One lane per tile: the tile width does not change a row (test_collision_cost_cpu.py)."""
    p = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    S, seg_len = len(descs), len(p) // n_seg
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    NP = len(p)
    cost, twist = np.empty(n_seg, np.float32), np.empty((n_seg, S, 6), np.float32)
    visited, pv, pg, pw = np.empty(NP, np.uint8), np.empty(NP, np.float32), np.empty((NP, 3), np.float32), \
        np.empty(NP, np.int32)
    evals = ctypes.c_longlong(0)
    hs.lib().simcc_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(a), ctypes.c_int(1), _p(p),
                         ctypes.c_longlong(n_seg), ctypes.c_int(seg_len), ctypes.c_float(margin), ctypes.c_int(chunk),
                         ctypes.c_int(8), ctypes.c_int(1), ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(-1),
                         _p(cost), _p(twist), _p(visited), _p(pv), _p(pg), _p(pw), ctypes.byref(evals))
    return cost, twist


def _fp64_cost(v, g, w, pts, m, S):
    """The fp64 composition from per-pair values v [A, n_seg, L], gradients g, sub-SDFs w and each configuration's
    own points pts [A, n_seg, L, 3]: cost, twist [A, n_seg, S, 6] and the sums of |term| of both."""
    v, g, pts = np.asarray(v, np.float64), np.asarray(g, np.float64), np.asarray(pts, np.float64)
    h = np.maximum(m - v, 0.0)
    terms = np.concatenate([g, np.cross(pts, g)], axis=-1) * (2.0 * h)[..., None]
    onehot = (w[..., None] == np.arange(S)).astype(np.float64)
    twist = np.einsum("...ls,...lk->...sk", onehot, terms)
    abs_tw = np.einsum("...ls,...lk->...sk", onehot, np.abs(terms))
    return (h * h).sum(-1), twist, (h * h).sum(-1), abs_tw


def _check_within(cost, twist, ref, what):
    rc, rt, ac, at = ref
    assert (np.abs(cost - rc) <= 1e-5 * ac + 1e-30).all(), (what, "cost", float(np.abs(cost - rc).max()))
    assert (np.abs(twist - rt) <= 1e-5 * at + 1e-30).all(), (what, "twist", float(np.abs(twist - rt).max()))


# segment lengths on both sides of one warp step (32) and of one chunk (512), and a segment of three chunks
SEGMENTS = [(1, 1), (3, 31), (2, 33), (2, 511), (1, 513), (2, 1500)]


@pytest.mark.parametrize("n_seg,L", SEGMENTS)
def test_paired_rows_equal_the_single_configuration_rows(built_lib, n_seg, L):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    A = 5
    tm = hs.trajectory(zc["tmat"], S, A0, A, seed=L)
    own = hs.own_points(zc["q"], A, seed=n_seg * L)[:, :n_seg * L].reshape(A, n_seg, L, 3)
    for name, descs in sets:
        v, g, w = hs.sim_paired(descs, tm, A, own.reshape(A, n_seg * L, 3))
        v, g, w = v.reshape(A, n_seg, L), g.reshape(A, n_seg, L, 3), w.reshape(A, n_seg, L)
        margins = [float(np.float32(np.quantile(v, q))) for q in (0.05, 0.3)]
        if (v < 0).sum() > 10:
            margins.append(float(np.float32(np.quantile(v[v < 0], 0.5))))
        for m in margins:
            what = (name, n_seg, L, m)
            cost, twist, vis, pv, pg, pw, evals = _pcc_fused(descs, tm, A, own, m)
            vis, pv, pg, pw = vis.reshape(A, n_seg, L), pv.reshape(A, n_seg, L), pg.reshape(A, n_seg, L, 3), \
                pw.reshape(A, n_seg, L)
            inside = v < m
            # no pair below the margin is skipped, and every evaluated pair below it is the per-pair query's
            assert vis[inside].all(), what
            assert np.array_equal(pv[inside], v[inside]) and np.array_equal(pw[inside], w[inside]), what
            assert np.array_equal(pg[inside], g[inside]), what
            assert not ((pw >= 0) & ~inside & (pv < m)).any(), what
            _check_within(cost.reshape(A, n_seg), twist.reshape(A, n_seg, S, 6), _fp64_cost(v, g, w, own, m, S),
                          what)
            # row a is configuration a alone over its own points, bit for bit
            for a in range(A):
                c1, t1 = _single(descs, tm, A, a, own[a], n_seg, m)
                rows = slice(a * n_seg, (a + 1) * n_seg)
                assert np.array_equal(cost[rows], c1) and np.array_equal(twist[rows], t1), (what, a)
            # unit orders and the first visit change nothing
            for kw in (dict(unit_order=1), dict(unit_order=2, shuffle_seed=3), dict(first=S - 1, unit_order=2)):
                c2, t2 = _pcc_fused(descs, tm, A, own, m, **kw)[:2]
                assert np.array_equal(c2, cost) and np.array_equal(t2, twist), (what, kw)
            # a forced chunk: still the single-configuration rows of that chunk
            if L > 7:
                c3, t3 = _pcc_fused(descs, tm, A, own, m, chunk=7, unit_order=2)[:2]
                for a in range(A):
                    c1, t1 = _single(descs, tm, A, a, own[a], n_seg, m, chunk=7)
                    rows = slice(a * n_seg, (a + 1) * n_seg)
                    assert np.array_equal(c3[rows], c1) and np.array_equal(t3[rows], t1), (what, "chunk", a)


def test_slabs_reproduce_the_rows_of_the_full_call(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    A = 40
    tm = hs.trajectory(zc["tmat"], S, A0, A, seed=11)
    own = hs.own_points(zc["q"], A, seed=4)[:, :600].reshape(A, 2, 300, 3)
    for name, descs in sets:
        v = hs.sim_paired(descs, tm, A, own.reshape(A, 600, 3))[0]
        m = float(np.float32(np.quantile(v, 0.2)))
        cost, twist = _pcc_fused(descs, tm, A, own, m)[:2]
        for begin, count in ((0, 1), (5, 32), (31, 2), (33, 7), (39, 1), (1, 39)):
            c2, t2 = _pcc_fused(descs, tm, A, own[begin:begin + count], m, cfg_begin=begin)[:2]
            rows = slice(begin * 2, (begin + count) * 2)
            assert np.array_equal(c2, cost[rows]) and np.array_equal(t2, twist[rows]), (name, begin, count)


def test_far_clouds_cost_exactly_zero(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A = int(zc["S"]), int(zc["A"])
    own = hs.own_points(zc["q"], A, seed=9)[:, :500].reshape(A, 1, 500, 3) + np.float32(50.0)
    for name, descs in sets:
        cost, twist, vis, pv, pg, pw, evals = _pcc_fused(descs, zc["tmat"], A, own, 0.05)
        assert not cost.any() and not twist.any(), name
        assert not vis.any() and evals == 0, name                 # every step skipped by its bounds


# ---------------------------------------------------------------- 2. C ABI refusals and Python rules (no device)
def test_abi_refuses_invalid_paired_collision_cost_queries(built_lib):
    near, tri, keep = hs.table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_seg=10, seg_len=100, margin=0.05,
             ws=fake, ws_bytes=1 << 40, cost=fake, twist=fake):
        return L.pvb_composed_query_paired_collision_cost(descs, n_sdf, xf, n_cfg, begin, count, pts, n_seg, seg_len,
                                                          margin, ws, ws_bytes, cost, twist, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    mesh = near.copy()
    mesh.kind = nat.PVB_KIND_MESH
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(cost=None), dict(twist=None), dict(ws=None),
             dict(ws_bytes=0), dict(ws_bytes=8), dict(ws=ctypes.c_void_p((1 << 12) + 2)), dict(n_sdf=0),
             dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0), dict(begin=2, count=3), dict(n_seg=-1),
             dict(seg_len=-1), dict(seg_len=1 << 31, n_seg=1), dict(n_seg=1 << 60, seg_len=4),
             dict(margin=float("nan")), dict(margin=float("inf")), dict(margin=-float("inf")),
             dict(descs=nat.desc_array([near] * 9), n_sdf=9), dict(descs=nat.desc_array([near, gt])),
             dict(descs=nat.desc_array([near, mesh])), dict(seg_len=0, cost=None)]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_paired_collision_cost"), (kw, msg)
    assert b"finite" in (call(margin=float("nan")), L.pvb_last_error())[1]
    assert b"workspace" in (call(ws_bytes=8), L.pvb_last_error())[1]
    assert b"compose" in (call(descs=nat.desc_array([near] * 9), n_sdf=9), L.pvb_last_error())[1]
    assert b"compose" in (call(descs=nat.desc_array([near, mesh])), L.pvb_last_error())[1]
    # cfg_count * n_seg * seg_len = 2^64: each factor pair alone fits in int64
    assert b"2^63" in (call(n_seg=1 << 60, seg_len=4), L.pvb_last_error())[1]
    # nothing to do: no segments, or no configurations and no points
    assert call(n_seg=0, pts=None, ws=None, ws_bytes=0, cost=None, twist=None) == 0
    assert call(seg_len=0, count=0, pts=None, ws=None, ws_bytes=0, cost=None, twist=None) == 0


def test_paired_collision_cost_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(3,))
    # the slab form: [..., N, 3] splitting into cfg_count blocks
    for shape in ((5, 2), (3,), (3, 5, 4), (), (0,)):
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.query_paired_collision_cost(torch.zeros(shape), 0.1)
    for shape, count in (((4, 10, 3), None), ((2, 10, 3), None), ((5, 10, 3), 2), ((6, 3), None), ((1, 10, 3), 0)):
        with pytest.raises(ValueError, match="do not split"):
            comp.query_paired_collision_cost(torch.zeros(shape), 0.1, cfg_count=count)
    for begin, count in ((1, 3), (-1, 2), (2, 2), (0, -1)):
        with pytest.raises(ValueError, match="configuration slab"):
            comp.query_paired_collision_cost(torch.zeros(3, 10, 3), 0.1, cfg_begin=begin, cfg_count=count)
    # the batched form: the configuration batch leading
    for shape in ((4, 10, 3), (2, 5, 10, 3), (10, 3, 3)):
        with pytest.raises(ValueError, match="configuration batch A = \\(3,\\) leading"):
            comp.paired_collision_cost(torch.zeros(shape), 0.1)
    for shape in ((3, 3), (3,), (3, 10, 4)):
        with pytest.raises(ValueError, match=r"\[\*A, \.\.\., N, 3\]"):
            comp.paired_collision_cost(torch.zeros(shape), 0.1)
    for margin in (float("nan"), float("inf"), -math.inf, "x", None, torch.tensor([0.1, 0.2])):
        with pytest.raises(ValueError, match="margin"):
            comp.paired_collision_cost(torch.zeros(3, 10, 3), margin)
        with pytest.raises(ValueError, match="margin"):
            comp.query_paired_collision_cost(torch.zeros(3, 10, 3), margin)
    # without a configuration batch it is collision_cost, with its rules
    single = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(2, 1, 1)))
    with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
        single.paired_collision_cost(torch.zeros(5, 2), 0.1)
