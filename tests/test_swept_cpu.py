"""CPU tier for swept composed queries (ComposedSDF.swept / RobotSDF.swept / pvb_composed_query_swept): at every point,
the minimum over the configurations.

1. The device arithmetic (rs_swept_pair, swept_before and swept_fold of pvb_device.cuh, compiled for the host by
   tests/hostsim/hostsim_swept.cpp in the order robot_swept_kernel runs them, and composed_point folded as
   composed_swept_kernel does): the result equals the lexicographic (value, configuration, sub-SDF) reduction of the
   per-configuration results bit for bit -- values, gradients, configuration and sub-SDF -- on the golden composition
   with nearest, trilinear, mixed and primitive sets, with pruning on or off, any first visit and any lane order.
2. Ties on purpose: duplicated configurations and duplicated sub-SDFs report the first of each.
3. The C ABI refusals and the Python shape rules, without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from pytorch_volumetric_b200 import _native as nat
from test_paired_cpu import _sets, _table_descs
from test_trilinear_composed_cpu import _sim_composed, _unpruned

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_swept.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_swept.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_swept.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
                   os.path.join(root, "pytorch_volumetric_b200", "csrc", "pvb_device.cuh"),
                   os.path.join(root, "include", "pvb.h")]
        if not os.path.exists(_SIM_LIB) or any(os.path.getmtime(f) > os.path.getmtime(_SIM_LIB) for f in sources):
            os.makedirs(os.path.dirname(_SIM_LIB), exist_ok=True)
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                            "-I", _SIM_DIR, sources[0], "-o", _SIM_LIB], check=True)
        _sim = ctypes.CDLL(_SIM_LIB)
    return _sim


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _outs(n):
    return np.empty(n, np.float32), np.empty((n, 3), np.float32), np.empty(n, np.int32), np.empty(n, np.int32)


def _sim_fused(descs, xforms, n_cfg, points, cfg_begin=0, cfg_count=None, first=-1, lanes_reversed=0):
    """(val, grad, cfg, which, lookups) of robot_swept_kernel's sequence over the slab."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    out = _outs(len(p))
    evals = ctypes.c_longlong(0)
    _simlib().simswept_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                             ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(len(p)), ctypes.c_int(first),
                             ctypes.c_int(lanes_reversed), *[_p(a) for a in out], ctypes.byref(evals))
    return out + (evals.value,)


def _sim_generic(descs, xforms, n_cfg, points, cfg_begin=0, cfg_count=None):
    """(val, grad, cfg, which) of composed_swept_kernel's per-thread work."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(hs.bit_reversed_order(S), dtype=np.uint8)
    margin_max = max([0.0] + [float(d.prune_margin) for d in descs])
    out = _outs(len(p))
    _simlib().simswept_generic(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                               ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(len(p)), ctypes.c_float(margin_max),
                               *[_p(a) for a in out])
    return out


def _reference(descs, xforms, n_cfg, points, cfg_begin=0, cfg_count=None):
    """The lexicographic (value, configuration, sub-SDF) reduction of the per-configuration results."""
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    P = len(points)
    v, g, w = _sim_composed(descs, xforms, n_cfg, points)
    v = v.reshape(n_cfg, P)[cfg_begin:cfg_begin + cfg_count]
    g = g.reshape(n_cfg, P, 3)[cfg_begin:cfg_begin + cfg_count]
    w = w.reshape(n_cfg, P)[cfg_begin:cfg_begin + cfg_count]
    c = np.argmax(v == v.min(axis=0), axis=0)                 # first configuration attaining the minimum
    i = np.arange(P)
    return v[c, i], g[c, i], (c + cfg_begin).astype(np.int32), w[c, i]


def _trajectory(tmat, S, A0, A, seed):
    """[S * A, 4, 4]: A configurations, configuration a the golden configuration a % A0 moved by a small rigid motion
    of the object frame (a robot-like sweep: the same motion for every sub-SDF of a configuration)."""
    g = np.random.default_rng(seed)
    m = np.asarray(tmat, dtype=np.float64).reshape(S, A0, 4, 4)
    out = np.empty((S, A, 4, 4))
    for a in range(A):
        w = g.normal(0.0, 0.15, 3)
        th = np.linalg.norm(w)
        k = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / max(th, 1e-12)
        T = np.eye(4)
        T[:3, :3] = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        T[:3, 3] = g.normal(0.0, 0.01, 3)
        out[:, a] = m[:, a % A0] @ T
    return out.reshape(S * A, 4, 4).astype(np.float32)


def _primitive_set():
    import pytorch_volumetric_b200 as pv
    return [pv.BoxSDF([0.05, 0.03, 0.04]).native_desc("cpu"), pv.CylinderSDF(0.015, 0.06).native_desc("cpu"),
            pv.SphereSDF(0.02).native_desc("cpu"), pv.BoxSDF([0.02, 0.02, 0.08]).native_desc("cpu")]


def _all_sets():
    zc, sets, keep = _sets()
    _, tri_probe, keep2 = _table_descs("probe")
    prim = _primitive_set()
    return zc, sets + [("primitive", prim), ("primitive+grid", [prim[0], sets[0][1][0], prim[1], tri_probe])], \
        (keep, keep2)


def _assert_same(got, ref, what):
    for a, b, name in zip(got, ref, ("val", "grad", "cfg", "which")):
        assert np.array_equal(a, b), (what, name, int(np.sum(a != b)))


@pytest.mark.parametrize("A", [3, 40])
def test_fused_swept_equals_the_reduction(built_lib, A):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else _trajectory(zc["tmat"], S, A0, A, seed=A)
    q = np.asarray(zc["q"], dtype=np.float32)
    for name, descs in sets:
        ref = _reference(descs, tm, A, q)
        got = _sim_fused(descs, tm, A, q)
        _assert_same(got[:4], ref, name)
        assert len(set(got[2].tolist())) > 1, name                  # the minimum moves between configurations
        # pruning off (no PVB_GRID_PRUNE_OK: every bound is -inf), then every first visit and the other lane order
        unpruned = _sim_fused(_unpruned(descs), tm, A, q)
        _assert_same(unpruned[:4], ref, (name, "unpruned"))
        assert got[4] < unpruned[4], name                          # pruning skips lookups
        for first in range(S):
            _assert_same(_sim_fused(descs, tm, A, q, first=first, lanes_reversed=first & 1)[:4], ref, (name, first))
        # slabs: the absolute configuration index, remainder tiles of every size
        for begin, count in ((1, A - 1), (A // 2, 1), (0, min(A, 7)), (A - 2, 2)):
            ref_s = _reference(descs, tm, A, q, cfg_begin=begin, cfg_count=count)
            _assert_same(_sim_fused(descs, tm, A, q, cfg_begin=begin, cfg_count=count)[:4], ref_s, (name, begin, count))


def test_fused_swept_prunes_across_tiles(built_lib):
    """With 40 configurations (a 32-configuration tile, then 8), the second tile's lanes prune against the point's
    best from the first: fewer lookups than the two tiles run as separate slabs."""
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = _trajectory(zc["tmat"], S, A0, 40, seed=5)
    q = np.asarray(zc["q"], dtype=np.float32)
    descs = sets[0][1]
    swept = _sim_fused(descs, tm, 40, q)[4]
    # the same tiles with no best from an earlier tile to prune against
    apart = _sim_fused(descs, tm, 40, q, cfg_count=32)[4] + _sim_fused(descs, tm, 40, q, cfg_begin=32)[4]
    assert swept < apart, (swept, apart)


def test_generic_swept_equals_the_reduction(built_lib):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = _trajectory(zc["tmat"], S, A0, 20, seed=3)
    q = np.asarray(zc["q"], dtype=np.float32)
    for name, descs in sets:
        _assert_same(_sim_generic(descs, tm, 20, q), _reference(descs, tm, 20, q), name)
        _assert_same(_sim_generic(descs, tm, 20, q, cfg_begin=5, cfg_count=9),
                     _reference(descs, tm, 20, q, cfg_begin=5, cfg_count=9), (name, "slab"))


def test_ties_report_the_first_configuration_and_sub_sdf(built_lib):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    base = _trajectory(zc["tmat"], S, A0, 6, seed=7).reshape(S, 6, 4, 4)
    # configurations 6..11 repeat 0..5, and 12..44 all repeat configuration 2: every minimum is attained at least twice
    tm = np.concatenate([base, base, np.repeat(base[:, 2:3], 33, axis=1)], axis=1)
    A = tm.shape[1]
    q = np.asarray(zc["q"], dtype=np.float32)
    for name, descs in sets:
        ref = _reference(descs, tm.reshape(S * A, 4, 4), A, q)
        assert (ref[2] < 6).all()
        for fn in (lambda: _sim_fused(descs, tm.reshape(S * A, 4, 4), A, q)[:4],
                   lambda: _sim_generic(descs, tm.reshape(S * A, 4, 4), A, q)):
            got = fn()
            _assert_same(got, ref, name)
            assert (got[2] < 6).all(), name
    # a sub-SDF listed twice under the same transforms: the first of the two wins its ties
    descs = sets[0][1]
    dup = [descs[0], descs[1], descs[0], descs[2], descs[3]]
    tm5 = np.concatenate([base[0:1], base[1:2], base[0:1], base[2:3], base[3:4]], axis=0)
    ref = _reference(dup, tm5.reshape(5 * 6, 4, 4), 6, q)
    assert (ref[3] != 2).all() and (ref[3] == 0).any()
    _assert_same(_sim_fused(dup, tm5.reshape(5 * 6, 4, 4), 6, q)[:4], ref, "dup")
    _assert_same(_sim_generic(dup, tm5.reshape(5 * 6, 4, 4), 6, q), ref, "dup generic")


# ---------------------------------------------------------------- C ABI refusals (no kernel launch involved)
def test_abi_refuses_invalid_swept_queries(built_lib):
    near, tri, keep = _table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_pts=100, val=fake, grad=fake):
        return L.pvb_composed_query_swept(descs, n_sdf, 0, xf, n_cfg, begin, count, pts, n_pts, nat.PVB_MESH_DEFAULT,
                                          val, grad, None, None, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    bad_kind = near.copy()
    bad_kind.kind = 7
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(val=None), dict(grad=None), dict(n_sdf=0),
             dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0), dict(begin=2, count=3), dict(n_pts=-1),
             dict(descs=nat.desc_array([near] * 129), n_sdf=129), dict(descs=nat.desc_array([near, gt])),
             dict(descs=nat.desc_array([near, bad_kind]))]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_swept"), (kw, msg)
    assert b"empty configuration slab" in (call(count=0), L.pvb_last_error())[1]
    assert b"128" in (call(descs=nat.desc_array([near] * 129), n_sdf=129), L.pvb_last_error())[1]
    assert b"bounding-box" in (call(descs=nat.desc_array([near, gt])), L.pvb_last_error())[1]
    assert b"unknown kind" in (call(descs=nat.desc_array([near, bad_kind])), L.pvb_last_error())[1]
    # no points: nothing to do, whatever the slab, without pointers to points or outputs
    assert call(n_pts=0, pts=None, val=None, grad=None) == 0
    assert call(n_pts=0, count=0, pts=None, val=None, grad=None) == 0


# ---------------------------------------------------------------- shape rules, before any device work
def test_swept_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(3,))
    for shape in ((5, 2), (0,), (4, 5, 4), ()):
        with pytest.raises(ValueError, match=r"\[\.\.\., 3\]"):
            comp.swept(torch.zeros(shape))
        with pytest.raises(ValueError, match=r"\[\.\.\., 3\]"):
            comp.query_swept(torch.zeros(shape))
    with pytest.raises(ValueError, match="empty configuration slab"):
        comp.query_swept(torch.zeros(10, 3), cfg_begin=1, cfg_count=0)
