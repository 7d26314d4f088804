"""CPU tier for clearance queries (ComposedSDF.clearance / RobotSDF.clearance / pvb_composed_query_clearance): for every
configuration and every segment of points, the per-configuration result at the first point attaining the minimum.

1. The key encoding (clearance_key / clearance_key_value of pvb_device.cuh): the unsigned order of keys is the
   (value, point) order -- +-0, +-inf, subnormals, NaN payloads of both signs, index tie-breaks -- checked exhaustively
   over all 2^32 patterns as well.
2. The device arithmetic, compiled for the host by tests/hostsim/hostsim_clearance.cpp in the order the kernels run
   it: robot_clearance_kernel's sequence with every chunk size, unit order, seeding, first visit and lane order,
   composed_clearance_kernel's per-pair work, and clearance_finish_kernel -- all equal to the reduction of the
   per-configuration results bit for bit (values, gradients, point and sub-SDF) on the golden composition with
   nearest, trilinear, mixed, primitive and primitive+grid sets, with duplicated points, configurations and sub-SDFs.
3. robot_serial_kernel's visit gives composed_point's bits for trilinear, box and cylinder links as well (the finish
   step re-evaluates the winner with composed_point).
4. The C ABI refusals and the Python shape rules, without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from hostsim_lib import PVB_ERR_INVALID, _p
from pytorch_volumetric_b200 import _native as nat


def _keys(v, idx):
    v = np.ascontiguousarray(v, dtype=np.float32)
    idx = np.ascontiguousarray(idx, dtype=np.uint32)
    out, dec = np.empty(len(v), np.uint64), np.empty(len(v), np.float32)
    hs.lib().simclear_keys(_p(v), _p(idx), ctypes.c_longlong(len(v)), _p(out), _p(dec))
    return out, dec


def _fused_keys(descs, xforms, n_cfg, points, n_seg, cfg_begin=0, cfg_count=None, chunk=None, unit_order=0,
                shuffle_seed=0, seeded=1, first=-1, lanes_reversed=0):
    """(keys [cfg_count * n_seg], lookups) of robot_clearance_kernel's sequence."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    seg_len = len(p) // n_seg
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    keys = np.empty(cfg_count * n_seg, np.uint64)
    evals = ctypes.c_longlong(0)
    hs.lib().simclear_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                            ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(seg_len),
                            ctypes.c_int(chunk or seg_len), ctypes.c_int(unit_order), ctypes.c_int(shuffle_seed),
                            ctypes.c_int(seeded), ctypes.c_int(first), ctypes.c_int(lanes_reversed), _p(keys),
                            ctypes.byref(evals))
    return keys, evals.value


def _generic_keys(descs, xforms, n_cfg, points, n_seg, cfg_begin=0, cfg_count=None):
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(hs.bit_reversed_order(S), dtype=np.uint8)
    keys = np.empty(cfg_count * n_seg, np.uint64)
    hs.lib().simclear_generic(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                              ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(len(p) // n_seg),
                              ctypes.c_float(hs.margin_max(descs)), _p(keys))
    return keys


def _finish(descs, xforms, n_cfg, points, n_seg, keys, cfg_begin=0, mesh=0):
    p = np.ascontiguousarray(points, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(hs.bit_reversed_order(S), dtype=np.uint8)
    R = len(keys)
    out = np.empty(R, np.float32), np.empty((R, 3), np.float32), np.empty(R, np.int32), np.empty(R, np.int32)
    hs.lib().simclear_finish(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                             ctypes.c_int(R // n_seg), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(len(p) // n_seg),
                             ctypes.c_int(mesh), ctypes.c_float(hs.margin_max(descs)), _p(np.ascontiguousarray(keys)),
                             *[_p(a) for a in out])
    return out


def _reference(descs, xforms, n_cfg, points, n_seg, cfg_begin=0, cfg_count=None):
    """The reduction of the per-configuration results: for every (configuration, segment), the first point attaining
    the minimum value (numpy: -0 == +0, as in torch)."""
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    P = len(points)
    L = P // n_seg
    v, g, w = hs.composed(descs, xforms, n_cfg, points, ext=True)
    v = v.reshape(n_cfg, n_seg, L)[cfg_begin:cfg_begin + cfg_count]
    g = g.reshape(n_cfg, n_seg, L, 3)[cfg_begin:cfg_begin + cfg_count]
    w = w.reshape(n_cfg, n_seg, L)[cfg_begin:cfg_begin + cfg_count]
    i = np.argmax(v == v.min(axis=-1, keepdims=True), axis=-1)[..., None]
    return (np.take_along_axis(v, i, -1).reshape(-1), np.take_along_axis(g, i[..., None], -2).reshape(-1, 3),
            i.reshape(-1).astype(np.int32), np.take_along_axis(w, i, -1).reshape(-1))


def _assert_same(got, ref, what):
    for a, b, name in zip(got, ref, ("val", "grad", "point", "which")):
        assert np.array_equal(a, b), (what, name, int(np.sum(a != b)))


def _decoded_equals_finish(keys, fin, what):
    """The value in every key is the re-evaluated value of its pair (-0 decodes as +0)."""
    _, dec = _keys(fin[0], np.zeros(len(keys), np.uint32))
    k = np.asarray(keys, dtype=np.uint64)
    fv = (k >> np.uint64(32)).astype(np.uint32)
    kv = np.where(fv >= 0x80000000, fv & 0x7FFFFFFF, ~fv).astype(np.uint32).view(np.float32)
    assert np.array_equal(kv, dec), what


# ---------------------------------------------------------------- 1. the key encoding
def test_key_order_on_special_values():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    sub = np.float32(1e-45)
    neg_nan = np.array([0xFFC00001], np.uint32).view(np.float32)[0]
    pay_nan = np.array([0x7F800001], np.uint32).view(np.float32)[0]
    ordered = [-inf, np.float32(-3.5), np.float32(-1e-38), -sub, np.float32(0.0), sub, np.float32(1e-38),
               np.float32(2.0), inf, nan]
    k, dec = _keys(np.array(ordered, np.float32), np.zeros(len(ordered), np.uint32))
    assert all(int(k[a]) < int(k[a + 1]) for a in range(len(k) - 1))
    assert np.array_equal(dec[:-1], np.array(ordered[:-1], np.float32)) and np.isnan(dec[-1])
    # -0 == +0, and the point index breaks the tie; every NaN is one key above +inf
    k, dec = _keys(np.array([-0.0, 0.0, 0.0, -0.0], np.float32), np.array([3, 3, 1, 7], np.uint32))
    assert k[0] == k[1] and k[2] < k[0] < k[3]
    assert dec.view(np.uint32).tolist() == [0, 0, 0, 0]
    k, dec = _keys(np.array([nan, neg_nan, pay_nan, -nan, inf], np.float32), np.array([5, 5, 5, 2, 9], np.uint32))
    assert k[0] == k[1] == k[2] and k[3] < k[0] and k[4] < k[3] and np.isnan(dec[:4]).all()
    assert int(k[0]) >> 32 == 0xFFFFFFFF
    # the index is the low word; values win over indices
    k, _ = _keys(np.array([1.0, 1.0, np.nextafter(np.float32(1.0), np.float32(2.0))], np.float32),
                 np.array([0x7FFFFFFF, 0, 0], np.uint32))
    assert k[1] < k[0] < k[2] and int(k[0]) & 0xFFFFFFFF == 0x7FFFFFFF


def test_key_order_over_all_patterns():
    bad = np.zeros(3, np.int64)
    hs.lib().simclear_check_all_patterns(_p(bad))
    assert bad.tolist() == [0, 0, 0]


def test_python_keys_match_the_device_keys():
    """ComposedSDF._clearance_keys (the unfused path's order) agrees with clearance_key on special and random values."""
    from pytorch_volumetric_b200.sdf import ComposedSDF
    g = np.random.default_rng(0)
    bits = np.concatenate([g.integers(0, 1 << 32, 20000, dtype=np.uint64).astype(np.uint32),
                           np.array([0, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 1, 0x80000001],
                                    np.uint32)])
    v = bits.view(np.float32)
    dev, _ = _keys(v, np.arange(len(v), dtype=np.uint32))
    py = ComposedSDF._clearance_keys(torch.from_numpy(v.copy())[None, :]).numpy()[0]
    # py is the device key minus 2^63 (as int64): the same order, and the index along the last dimension
    assert np.array_equal(py.view(np.uint64) ^ np.uint64(1 << 63), dev)


# ---------------------------------------------------------------- 2. the kernels' sequences
def _segments(q, n_seg):
    return np.asarray(q, dtype=np.float32)[: (len(q) // n_seg) * n_seg]


@pytest.mark.parametrize("A", [3, 40])
def test_fused_clearance_equals_the_reduction(built_lib, A):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else hs.trajectory(zc["tmat"], S, A0, A, seed=A)
    for n_seg in (6, 1):
        q = _segments(zc["q"], n_seg)
        L = len(q) // n_seg
        for name, descs in sets:
            ref = _reference(descs, tm, A, q, n_seg)
            keys, evals = _fused_keys(descs, tm, A, q, n_seg)
            fin = _finish(descs, tm, A, q, n_seg, keys)
            _assert_same(fin, ref, (name, n_seg))
            _decoded_equals_finish(keys, fin, (name, n_seg))
            assert len(set(ref[2].tolist())) > 1, name                # the argmin point differs between pairs
            # pruning off (no PVB_GRID_PRUNE_OK: every bound is -inf)
            unpruned_keys, unpruned = _fused_keys(hs.unpruned(descs), tm, A, q, n_seg)
            assert np.array_equal(unpruned_keys, keys), (name, "unpruned")
            assert evals < unpruned, name                            # pruning skips lookups
            # chunk sizes, unit orders, seeding, first visits and lane orders: the same keys
            for chunk in (1, 7, 32, L):
                for order, seed in ((0, 0), (1, 0), (2, chunk)):
                    got = _fused_keys(descs, tm, A, q, n_seg, chunk=chunk, unit_order=order, shuffle_seed=seed,
                                      seeded=(chunk + order) & 1, lanes_reversed=order & 1)[0]
                    assert np.array_equal(got, keys), (name, n_seg, chunk, order)
            for first in range(S):
                got = _fused_keys(descs, tm, A, q, n_seg, chunk=32, first=first, lanes_reversed=first & 1)[0]
                assert np.array_equal(got, keys), (name, n_seg, first)
            # slabs: remainder tiles of every size
            for begin, count in ((1, A - 1), (A // 2, 1), (0, min(A, 7)), (A - 2, 2)):
                ref_s = _reference(descs, tm, A, q, n_seg, cfg_begin=begin, cfg_count=count)
                ks = _fused_keys(descs, tm, A, q, n_seg, cfg_begin=begin, cfg_count=count, chunk=64)[0]
                _assert_same(_finish(descs, tm, A, q, n_seg, ks, cfg_begin=begin), ref_s, (name, begin, count))


def test_seeding_prunes_across_blocks(built_lib):
    """Chunks that start from the keys of earlier chunks skip lookups that unseeded chunks make."""
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = hs.trajectory(zc["tmat"], S, A0, 40, seed=5)
    q = _segments(zc["q"], 1)
    descs = sets[0][1]
    seeded = _fused_keys(descs, tm, 40, q, 1, chunk=64, seeded=1)[1]
    unseeded = _fused_keys(descs, tm, 40, q, 1, chunk=64, seeded=0)[1]
    assert seeded < unseeded, (seeded, unseeded)


def test_generic_clearance_equals_the_reduction(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = hs.trajectory(zc["tmat"], S, A0, 20, seed=3)
    q = _segments(zc["q"], 6)
    for name, descs in sets:
        keys = _generic_keys(descs, tm, 20, q, 6)
        fin = _finish(descs, tm, 20, q, 6, keys, mesh=1)
        _assert_same(fin, _reference(descs, tm, 20, q, 6), name)
        _decoded_equals_finish(keys, fin, name)
        assert np.array_equal(keys, _fused_keys(descs, tm, 20, q, 6, chunk=32)[0]), name
        ks = _generic_keys(descs, tm, 20, q, 6, cfg_begin=5, cfg_count=9)
        _assert_same(_finish(descs, tm, 20, q, 6, ks, cfg_begin=5, mesh=1),
                     _reference(descs, tm, 20, q, 6, cfg_begin=5, cfg_count=9), (name, "slab"))


def test_ties_report_the_first_point(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    base = hs.trajectory(zc["tmat"], S, A0, 6, seed=7).reshape(S, 6, 4, 4)
    # configurations 6..11 repeat 0..5, and 12..44 repeat configuration 2
    tm = np.concatenate([base, base, np.repeat(base[:, 2:3], 33, axis=1)], axis=1)
    A = tm.shape[1]
    tm = tm.reshape(S * A, 4, 4)
    # every segment twice in a row, and each segment's points repeated: every minimum is attained at least twice
    q = np.asarray(zc["q"], dtype=np.float32)[:600].reshape(4, 150, 3)
    q = np.concatenate([q, q], axis=1).reshape(-1, 3)
    for name, descs in sets:
        ref = _reference(descs, tm, A, q, 4)
        assert (ref[2] < 150).all()
        for keys in (_fused_keys(descs, tm, A, q, 4)[0], _fused_keys(descs, tm, A, q, 4, chunk=7, unit_order=1)[0],
                     _fused_keys(descs, tm, A, q, 4, chunk=32, unit_order=2, shuffle_seed=3, lanes_reversed=1)[0],
                     _generic_keys(descs, tm, A, q, 4)):
            fin = _finish(descs, tm, A, q, 4, keys)
            _assert_same(fin, ref, name)
        # duplicated configurations give identical rows
        v = ref[0].reshape(A, 4)
        assert np.array_equal(v[0:6], v[6:12]) and (v[12:] == v[2]).all()
    # a sub-SDF listed twice under the same transforms: the first of the two wins its ties
    descs = sets[0][1]
    b6 = base.reshape(S, 6, 4, 4)
    dup = [descs[0], descs[1], descs[0], descs[2], descs[3]]
    tm5 = np.concatenate([b6[0:1], b6[1:2], b6[0:1], b6[2:3], b6[3:4]], axis=0).reshape(5 * 6, 4, 4)
    ref = _reference(dup, tm5, 6, q, 4)
    assert (ref[3] != 2).all() and (ref[3] == 0).any()
    _assert_same(_finish(dup, tm5, 6, q, 4, _fused_keys(dup, tm5, 6, q, 4, chunk=32)[0]), ref, "dup")
    _assert_same(_finish(dup, tm5, 6, q, 4, _generic_keys(dup, tm5, 6, q, 4), mesh=1), ref, "dup generic")


# ---------------------------------------------------------------- 3. the serial visit == composed_point, every link kind
def test_serial_visit_equals_composed_point_for_every_link_kind(built_lib):
    """robot_serial_kernel's visit sequence (nearest, trilinear, box, cylinder and sphere links, every first visit)
    gives composed_point's bits: value, gradient and link.  The finish step relies on it."""
    import pytorch_volumetric_b200 as pv
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = hs.trajectory(zc["tmat"], S, A0, 10, seed=9)
    q = np.asarray(zc["q"], dtype=np.float32)
    box, cyl = pv.BoxSDF([0.03, 0.05, 0.02]).native_desc("cpu"), pv.CylinderSDF(0.02, 0.07).native_desc("cpu")
    extra = [("box+cylinder", [box, cyl, box, cyl])]
    for name, descs in sets + extra:
        ref = hs.composed(descs, tm, 10, q, ext=True)
        for first in [-1] + list(range(S)):
            arr = (nat.SdfDesc * S)(*descs)
            xf = np.ascontiguousarray(tm, dtype=np.float32)
            out = (np.empty(10 * len(q), np.float32), np.empty((10 * len(q), 3), np.float32),
                   np.empty(10 * len(q), np.int32))
            hs.lib().simclear_serial_pairs(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(10), _p(q),
                                           ctypes.c_longlong(len(q)), ctypes.c_int(first), *[_p(a) for a in out])
            for a, b, what in zip(out, ref, ("val", "grad", "which")):
                assert np.array_equal(a, b), (name, first, what, int(np.sum(a != b)))


# ---------------------------------------------------------------- 4. C ABI refusals (no kernel launch involved)
def test_abi_refuses_invalid_clearance_queries(built_lib):
    near, tri, keep = hs.table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_seg=10, seg_len=100, keys=fake,
             val=fake, grad=fake):
        return L.pvb_composed_query_clearance(descs, n_sdf, 0, xf, n_cfg, begin, count, pts, n_seg, seg_len,
                                              nat.PVB_MESH_DEFAULT, keys, val, grad, None, None, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    bad_kind = near.copy()
    bad_kind.kind = 7
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(val=None), dict(grad=None), dict(keys=None),
             dict(n_sdf=0), dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0), dict(begin=2, count=3),
             dict(n_seg=-1), dict(seg_len=-1), dict(seg_len=0), dict(seg_len=1 << 31, n_seg=1),
             dict(n_seg=1 << 62, seg_len=4), dict(descs=nat.desc_array([near] * 129), n_sdf=129),
             dict(descs=nat.desc_array([near, gt])), dict(descs=nat.desc_array([near, bad_kind]))]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_clearance"), (kw, msg)
    assert b"empty configuration slab" in (call(count=0), L.pvb_last_error())[1]
    assert b"empty segment" in (call(seg_len=0), L.pvb_last_error())[1]
    assert b"keys" in (call(keys=None), L.pvb_last_error())[1]
    assert b"128" in (call(descs=nat.desc_array([near] * 129), n_sdf=129), L.pvb_last_error())[1]
    assert b"bounding-box" in (call(descs=nat.desc_array([near, gt])), L.pvb_last_error())[1]
    # no segments: nothing to do, whatever the slab, without pointers to points, keys or outputs
    assert call(n_seg=0, pts=None, keys=None, val=None, grad=None) == 0
    assert call(n_seg=0, count=0, pts=None, keys=None, val=None, grad=None) == 0
    assert call(n_seg=0, seg_len=0, pts=None, keys=None, val=None, grad=None) == 0
    # empty segments and no configurations: no outputs to write
    assert call(seg_len=0, count=0, pts=None, keys=None, val=None, grad=None) == 0


# ---------------------------------------------------------------- shape rules, before any device work
def test_clearance_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(3,))
    for shape in ((5, 2), (3,), (4, 5, 4), (), (0,)):
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.clearance(torch.zeros(shape))
        with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
            comp.query_clearance(torch.zeros(shape))
    for shape in ((0, 3), (2, 0, 3)):
        with pytest.raises(ValueError, match="empty segment"):
            comp.clearance(torch.zeros(shape))
        with pytest.raises(ValueError, match="empty segment"):
            comp.query_clearance(torch.zeros(shape))
    with pytest.raises(ValueError, match="empty configuration slab"):
        comp.query_clearance(torch.zeros(10, 3), cfg_begin=1, cfg_count=0)
    from pytorch_volumetric_b200 import distributed as pd
    robot = type("R", (), {"sdf": comp})()
    with pytest.raises(ValueError, match="gather=True or gather=False"):
        pd.sharded_robot_query(robot, torch.zeros(10, 3), gather="peer", clearance=True)
    with pytest.raises(ValueError, match="cannot be combined"):
        pd.sharded_robot_query(robot, torch.zeros(10, 3), paired=True, clearance=True)
    with pytest.raises(ValueError, match=r"\[\.\.\., N, 3\]"):
        pd.sharded_robot_query(robot, torch.zeros(10, 2), clearance=True)
