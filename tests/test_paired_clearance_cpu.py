"""CPU tier for paired clearance queries (ComposedSDF.paired_clearance / RobotSDF.paired_clearance /
pvb_composed_query_paired_clearance): every configuration against its own cloud, for every segment the
per-configuration result at the first point attaining the minimum.

1. The device arithmetic, compiled for the host by tests/hostsim/hostsim_paired_clearance.cpp in the order the kernels
   run it: robot_paired_clearance_kernel's sequence (a warp per unit, the running value shared over the warp after
   every step) and the same sequence under every unit order, chunk size, seeding, first visit and step order, with a
   whole block per unit and without the sharing as further schedules, then paired_clearance_finish_kernel -- equal to
   the reduction of the per-configuration results on each configuration's own points bit for bit (values, gradients,
   point and sub-SDF) on the golden composition with nearest, trilinear, mixed, primitive and primitive+grid sets, with
   duplicated points, configurations and sub-SDFs.
2. Pruning: the sequence evaluates fewer links than pairs x links on a scene-like cloud.
3. The general route (composed_paired_clearance_kernel and its finish) gives the fused route's keys and results.
4. The C ABI refusals and the Python shape rules, without a GPU."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from pytorch_volumetric_b200 import _native as nat
from test_paired_cpu import _own_points, _table_descs
from test_swept_cpu import _all_sets, _trajectory
from test_trilinear_composed_cpu import _sim_composed, _unpruned

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_paired_clearance.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_paired_clearance.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when
    stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_paired_clearance.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
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


def _margin_max(descs):
    return max([0.0] + [float(d.prune_margin) for d in descs])


def _fused_keys(descs, xforms, n_cfg, own, cfg_begin=0, chunk=None, lanes=32, share=1, unit_order=0, shuffle_seed=0,
                seeded=1, first=-1, steps_reversed=0):
    """(keys [cfg_count * n_seg], lookups) of robot_paired_clearance_kernel's sequence; own [cfg_count, n_seg, L, 3]."""
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    keys = np.empty(cfg_count * n_seg, np.uint64)
    evals = ctypes.c_longlong(0)
    _simlib().simpcl_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                           ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                           ctypes.c_int(chunk or L), ctypes.c_int(lanes), ctypes.c_int(share),
                           ctypes.c_int(unit_order), ctypes.c_int(shuffle_seed), ctypes.c_int(seeded),
                           ctypes.c_int(first), ctypes.c_int(steps_reversed), _p(keys), ctypes.byref(evals))
    return keys, evals.value


def _generic_keys(descs, xforms, n_cfg, own, cfg_begin=0):
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(hs.bit_reversed_order(S), dtype=np.uint8)
    keys = np.empty(cfg_count * n_seg, np.uint64)
    _simlib().simpcl_generic(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                             ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                             ctypes.c_float(_margin_max(descs)), _p(keys))
    return keys


def _finish(descs, xforms, n_cfg, own, keys, cfg_begin=0, mesh=0):
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(hs.bit_reversed_order(S), dtype=np.uint8)
    R = len(keys)
    out = np.empty(R, np.float32), np.empty((R, 3), np.float32), np.empty(R, np.int32), np.empty(R, np.int32)
    _simlib().simpcl_finish(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                            ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                            ctypes.c_int(mesh), ctypes.c_float(_margin_max(descs)), _p(np.ascontiguousarray(keys)),
                            *[_p(a) for a in out])
    return out


def _reference(descs, xforms, n_cfg, own, cfg_begin=0):
    """Configuration by configuration: composed_point on its own points alone, then for every segment the first point
    attaining the minimum value (numpy: -0 == +0, as in torch)."""
    cfg_count, n_seg, L = own.shape[:3]
    S = len(descs)
    tm = np.asarray(xforms, dtype=np.float32).reshape(S, n_cfg, 4, 4)
    out = [[] for _ in range(4)]
    for c in range(cfg_count):
        v, g, w = _sim_composed(descs, tm[:, cfg_begin + c], 1, own[c].reshape(-1, 3))
        v, g, w = v.reshape(n_seg, L), g.reshape(n_seg, L, 3), w.reshape(n_seg, L)
        i = np.argmax(v == v.min(axis=-1, keepdims=True), axis=-1)[..., None]
        for k, t in enumerate((np.take_along_axis(v, i, -1).reshape(-1),
                               np.take_along_axis(g, i[..., None], -2).reshape(-1, 3),
                               i.reshape(-1).astype(np.int32), np.take_along_axis(w, i, -1).reshape(-1))):
            out[k].append(t)
    return tuple(np.concatenate(o) for o in out)


def _assert_same(got, ref, what):
    for a, b, name in zip(got, ref, ("val", "grad", "point", "which")):
        assert np.array_equal(a, b), (what, name, int(np.sum(a != b)))


def _clouds(zc, A, n_seg, L, seed):
    """[A, n_seg, L, 3]: every configuration its own shuffled, shifted copy of the golden points."""
    return _own_points(zc["q"], A, seed)[:, :n_seg * L].reshape(A, n_seg, L, 3)


# ---------------------------------------------------------------- 1. the fused sequence
@pytest.mark.parametrize("A", [3, 40])
def test_fused_paired_clearance_equals_the_reduction(built_lib, A):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else _trajectory(zc["tmat"], S, A0, A, seed=A)
    for n_seg, L in ((3, 300), (1, 700)):
        own = _clouds(zc, A, n_seg, L, seed=A + n_seg)
        for name, descs in sets:
            ref = _reference(descs, tm, A, own)
            keys, evals = _fused_keys(descs, tm, A, own)
            _assert_same(_finish(descs, tm, A, own, keys), ref, (name, n_seg))
            assert len(set(ref[2].tolist())) > 1, name                # the argmin point differs between pairs
            # pruning off (no PVB_GRID_PRUNE_OK: every bound is -inf)
            unpruned_keys, unpruned = _fused_keys(_unpruned(descs), tm, A, own)
            assert np.array_equal(unpruned_keys, keys), (name, "unpruned")
            assert evals < unpruned, name
            # chunk sizes, unit widths, sharing, unit orders, seeding and step orders: the same keys
            for chunk in (7, 32, 64, L):
                for lanes in (32, 256):
                    for order, seed in ((0, 0), (1, 0), (2, chunk + lanes)):
                        got = _fused_keys(descs, tm, A, own, chunk=chunk, lanes=lanes, share=(order + 1) & 1,
                                          unit_order=order, shuffle_seed=seed, seeded=(chunk + order) & 1,
                                          steps_reversed=order & 1)[0]
                        assert np.array_equal(got, keys), (name, n_seg, chunk, lanes, order)
            for first in range(S):
                got = _fused_keys(descs, tm, A, own, chunk=64, first=first, steps_reversed=first & 1)[0]
                assert np.array_equal(got, keys), (name, n_seg, first)
            # slabs: the absolute configuration picks the transforms
            for begin, count in ((1, A - 1), (A // 2, 1), (A - 2, 2)):
                sub = own[begin:begin + count]
                ks = _fused_keys(descs, tm, A, sub, cfg_begin=begin, chunk=64)[0]
                _assert_same(_finish(descs, tm, A, sub, ks, cfg_begin=begin), _reference(descs, tm, A, sub, begin),
                             (name, begin, count))


def test_ties_report_the_first_point(built_lib):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    base = _trajectory(zc["tmat"], S, A0, 6, seed=7).reshape(S, 6, 4, 4)
    # configurations 6..11 repeat 0..5 with the same clouds, and 12..44 repeat configuration 2 and its cloud
    tm = np.concatenate([base, base, np.repeat(base[:, 2:3], 33, axis=1)], axis=1)
    A = tm.shape[1]
    tm = tm.reshape(S * A, 4, 4)
    c6 = _clouds(zc, 6, 4, 75, seed=11)
    c6 = np.concatenate([c6, c6], axis=2)                        # every segment's points twice in a row
    own = np.concatenate([c6, c6, np.repeat(c6[2:3], 33, axis=0)], axis=0)
    for name, descs in sets:
        ref = _reference(descs, tm, A, own)
        assert (ref[2] < 75).all()
        for keys in (_fused_keys(descs, tm, A, own)[0],
                     _fused_keys(descs, tm, A, own, chunk=7, unit_order=1, share=0)[0],
                     _fused_keys(descs, tm, A, own, chunk=32, lanes=256, unit_order=2, shuffle_seed=3,
                                 steps_reversed=1)[0],
                     _generic_keys(descs, tm, A, own)):
            _assert_same(_finish(descs, tm, A, own, keys), ref, name)
        v = ref[0].reshape(A, 4)
        assert np.array_equal(v[0:6], v[6:12]) and (v[12:] == v[2]).all()
    # a sub-SDF listed twice under the same transforms: the first of the two wins its ties
    descs = sets[0][1]
    dup = [descs[0], descs[1], descs[0], descs[2], descs[3]]
    tm5 = np.concatenate([base[0:1], base[1:2], base[0:1], base[2:3], base[3:4]], axis=0).reshape(5 * 6, 4, 4)
    ref = _reference(dup, tm5, 6, c6)
    assert (ref[3] != 2).all() and (ref[3] == 0).any()
    _assert_same(_finish(dup, tm5, 6, c6, _fused_keys(dup, tm5, 6, c6, chunk=32)[0]), ref, "dup")
    _assert_same(_finish(dup, tm5, 6, c6, _generic_keys(dup, tm5, 6, c6), mesh=1), ref, "dup generic")


# ---------------------------------------------------------------- 2. pruning
def test_pruning_on_a_scene_cloud(built_lib):
    """A cloud of a few flat patches around the object, shifted per configuration (an environment per configuration):
    the bounds skip most links, seeding skips more, and so does the warp's shared running value."""
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    A, N = 24, 2048
    tm = _trajectory(zc["tmat"], S, A0, A, seed=13)
    q = np.asarray(zc["q"], dtype=np.float64)
    lo, hi = q.min(0), q.max(0)
    g = np.random.default_rng(14)
    own = np.empty((A, 1, N, 3), np.float32)
    for a in range(A):
        patches = []
        for k in range(4):
            axis = k % 3
            pts = g.uniform(lo, hi, (N // 4, 3))
            pts[:, axis] = (lo if k < 2 else hi)[axis] + g.normal(0.0, 0.002)
            patches.append(pts)
        own[a, 0] = np.concatenate(patches) + g.normal(0.0, 0.01, 3)
    for name, descs in sets:
        keys, evals = _fused_keys(descs, tm, A, own, chunk=256)
        _assert_same(_finish(descs, tm, A, own, keys), _reference(descs, tm, A, own), name)
        assert evals < A * N * S, (name, evals)
        unseeded = _fused_keys(descs, tm, A, own, chunk=256, seeded=0)[1]
        unshared = _fused_keys(descs, tm, A, own, chunk=256, share=0)[1]
        assert evals <= unseeded and evals <= unshared, (name, evals, unseeded, unshared)
    descs = sets[0][1]
    assert _fused_keys(descs, tm, A, own, chunk=256)[1] < _fused_keys(descs, tm, A, own, chunk=256, share=0)[1]


# ---------------------------------------------------------------- 3. the general route
def test_generic_paired_clearance_equals_the_fused_route(built_lib):
    zc, sets, keep = _all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = _trajectory(zc["tmat"], S, A0, 20, seed=3)
    own = _clouds(zc, 20, 6, 100, seed=4)
    for name, descs in sets:
        keys = _generic_keys(descs, tm, 20, own)
        fused = _fused_keys(descs, tm, 20, own, chunk=32)[0]
        assert np.array_equal(keys, fused), name
        fin = _finish(descs, tm, 20, own, keys, mesh=1)
        assert all(np.array_equal(a, b) for a, b in zip(fin, _finish(descs, tm, 20, own, fused))), name
        _assert_same(fin, _reference(descs, tm, 20, own), name)
        sub = own[5:14]
        ks = _generic_keys(descs, tm, 20, sub, cfg_begin=5)
        _assert_same(_finish(descs, tm, 20, sub, ks, cfg_begin=5, mesh=1), _reference(descs, tm, 20, sub, 5),
                     (name, "slab"))


# ---------------------------------------------------------------- 4. C ABI refusals (no kernel launch involved)
def test_abi_refuses_invalid_paired_clearance_queries(built_lib):
    near, tri, keep = _table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_seg=10, seg_len=100, keys=fake,
             val=fake, grad=fake):
        return L.pvb_composed_query_paired_clearance(descs, n_sdf, 0, xf, n_cfg, begin, count, pts, n_seg, seg_len,
                                                     nat.PVB_MESH_DEFAULT, keys, val, grad, None, None, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    bad_kind = near.copy()
    bad_kind.kind = 7
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(val=None), dict(grad=None), dict(keys=None),
             dict(n_sdf=0), dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0), dict(begin=2, count=3),
             dict(n_seg=-1), dict(seg_len=-1), dict(seg_len=0), dict(seg_len=1 << 31, n_seg=1),
             dict(n_seg=1 << 62, seg_len=4), dict(n_seg=1 << 40, seg_len=1 << 21),
             dict(n_seg=(1 << 61) // 100, seg_len=100, n_cfg=8, count=8),
             dict(descs=nat.desc_array([near] * 129), n_sdf=129),
             dict(descs=nat.desc_array([near, gt])), dict(descs=nat.desc_array([near, bad_kind]))]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_paired_clearance"), (kw, msg)
    assert b"empty configuration slab" in (call(count=0), L.pvb_last_error())[1]
    assert b"empty segment" in (call(seg_len=0), L.pvb_last_error())[1]
    assert b"keys" in (call(keys=None), L.pvb_last_error())[1]
    assert b"2^63" in (call(n_seg=(1 << 61) // 100, seg_len=100, n_cfg=8, count=8), L.pvb_last_error())[1]
    assert b"128" in (call(descs=nat.desc_array([near] * 129), n_sdf=129), L.pvb_last_error())[1]
    assert b"bounding-box" in (call(descs=nat.desc_array([near, gt])), L.pvb_last_error())[1]
    # no segments: nothing to do, whatever the slab, without pointers to points, keys or outputs
    assert call(n_seg=0, pts=None, keys=None, val=None, grad=None) == 0
    assert call(n_seg=0, count=0, pts=None, keys=None, val=None, grad=None) == 0
    assert call(n_seg=0, seg_len=0, pts=None, keys=None, val=None, grad=None) == 0
    assert call(seg_len=0, count=0, pts=None, keys=None, val=None, grad=None) == 0


# ---------------------------------------------------------------- shape rules, before any device work
def test_paired_clearance_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(3,))
    # not [..., N, 3], or no N after the configuration batch
    for shape in ((3, 5, 2), (3, 3), (3,), (), (3, 4, 5, 4)):
        with pytest.raises(ValueError, match=r"N, 3\]"):
            comp.paired_clearance(torch.zeros(shape))
    for shape in ((5, 2), (3,), ()):
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.query_paired_clearance(torch.zeros(shape))
    # the leading dimensions are not A
    for shape in ((4, 10, 3), (2, 10, 3), (1, 3, 10, 3), (6, 10, 3)):
        with pytest.raises(ValueError, match="leading"):
            comp.paired_clearance(torch.zeros(shape))
    with pytest.raises(ValueError, match="do not split"):
        comp.query_paired_clearance(torch.zeros(4, 10, 3))
    with pytest.raises(ValueError, match="do not split"):
        comp.query_paired_clearance(torch.zeros(10, 3), cfg_begin=1, cfg_count=0)
    # empty segments
    for shape in ((3, 0, 3), (3, 2, 0, 3)):
        with pytest.raises(ValueError, match="empty segment"):
            comp.paired_clearance(torch.zeros(shape))
        with pytest.raises(ValueError, match="empty segment"):
            comp.query_paired_clearance(torch.zeros(shape))
    # RobotSDF delegates
    from pytorch_volumetric_b200.model_to_sdf import RobotSDF
    robot = RobotSDF.__new__(RobotSDF)
    robot.sdf = comp
    with pytest.raises(ValueError, match="leading"):
        robot.paired_clearance(torch.zeros(4, 10, 3))
    # the sharded wrapper keeps refusing the combination: query_paired_clearance(cfg_begin=...) is its building block
    from pytorch_volumetric_b200 import distributed as pd
    with pytest.raises(ValueError, match="cannot be combined"):
        pd.sharded_robot_query(type("R", (), {"sdf": comp})(), torch.zeros(3, 10, 3), paired=True, clearance=True)
