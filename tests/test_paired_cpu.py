"""CPU tier for paired composed queries (ComposedSDF.paired / RobotSDF.paired / pvb_composed_query_paired): every
configuration evaluated at its own points.

1. The device arithmetic (composed_point and paired_index of pvb_device.cuh, compiled for the host by
   tests/hostsim/hostsim_paired.cpp): a paired evaluation equals the diagonal of the cross product on the golden
   composition -- nearest, trilinear and mixed grid sets with the sphere, probe and drill tables -- bit for bit, with
   pruning on or off, in any visiting order and with or without the nearest-bound-first order.
2. The 64-bit pair index arithmetic near and above 2^31 pairs.
3. The C ABI refusals, and the shape rules of the Python layer, without a GPU."""
import ctypes
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from helpers import golden
from pytorch_volumetric_b200 import _native as nat
from test_trilinear_composed_cpu import _grid_desc, _sim_composed, _unpruned

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_paired.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_paired.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_paired.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
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


def _sim_paired(descs, xforms, n_cfg, points, cfg_begin=0, order=None, nearest_first=1):
    """(val, grad, which) of configurations cfg_begin.. at their own points [cfg_count, P, 3]."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count, P = p.shape[0], p.shape[1]
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4)
    order = hs.bit_reversed_order(S) if order is None else list(order)
    od = np.asarray(order, dtype=np.uint8)
    margin_max = max([0.0] + [float(d.prune_margin) for d in descs])
    n = cfg_count * P
    val, grad, which = np.empty(n, np.float32), np.empty((n, 3), np.float32), np.empty(n, np.int32)
    _simlib().simpair_composed(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                               ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(P), ctypes.c_int(nearest_first),
                               ctypes.c_float(margin_max), _p(val), _p(grad), _p(which))
    return val, grad, which


def _table_descs(name):
    z = golden(f"ref_cachedsdf_{name}")
    shape = tuple(int(s) for s in z["table_shape"])
    args = (torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"]),
            [tuple(r) for r in z["ranges"]], z["bb"])
    near, k1 = _grid_desc(*args, interpolation="nearest")
    tri, k2 = _grid_desc(*args, interpolation="trilinear")
    return near, tri, (k1, k2)


def _sets():
    zc = golden("ref_composed")
    sph = hs.sphere_desc(float(zc["sphere_radius"]))
    pn, pt, k1 = _table_descs("probe")
    dn, dt, k2 = _table_descs("drill")
    return zc, [("nearest", [pn, pn, sph, pn]), ("trilinear", [pt, pt, sph, pt]), ("mixed", [pn, pt, sph, dt]),
                ("drill", [dn, dt, dn, sph])], (k1, k2)


def _own_points(q, A, seed):
    """[A, P, 3]: the golden points, shuffled and shifted differently for every configuration."""
    g = np.random.default_rng(seed)
    q = np.asarray(q, dtype=np.float32)
    return np.stack([q[g.permutation(len(q))] + g.normal(0.0, 0.01, 3).astype(np.float32) for _ in range(A)])


def test_paired_equals_the_cross_product_diagonal(built_lib):
    zc, sets, keep = _sets()
    S, A = int(zc["S"]), int(zc["A"])
    own = _own_points(zc["q"], A, 0)
    P = own.shape[1]
    for name, descs in sets:
        # the cross product over all A * P points, then configuration a's own block on its diagonal
        cv, cg, cw = _sim_composed(descs, zc["tmat"], A, own.reshape(-1, 3))
        cv, cg, cw = cv.reshape(A, A, P), cg.reshape(A, A, P, 3), cw.reshape(A, A, P)
        dv = np.stack([cv[a, a] for a in range(A)]).reshape(-1)
        dg = np.stack([cg[a, a] for a in range(A)]).reshape(-1, 3)
        dw = np.stack([cw[a, a] for a in range(A)]).reshape(-1)
        for nearest_first in (1, 0):
            v, g, w = _sim_paired(descs, zc["tmat"], A, own, nearest_first=nearest_first)
            assert np.array_equal(v, dv) and np.array_equal(g, dg) and np.array_equal(w, dw), (name, nearest_first)
        # pruning off, other visiting orders
        for order in (range(S), list(range(S))[::-1], [2, 0, 3, 1]):
            for d in (descs, _unpruned(descs)):
                v, g, w = _sim_paired(d, zc["tmat"], A, own, order=order, nearest_first=0)
                assert np.array_equal(v, dv) and np.array_equal(g, dg) and np.array_equal(w, dw), (name, order)
        # a slab of the configurations, indexed by the absolute configuration
        v, g, w = _sim_paired(descs, zc["tmat"], A, own[1:3], cfg_begin=1)
        assert np.array_equal(v, dv[P:3 * P]) and np.array_equal(w, dw[P:3 * P]), name


def test_paired_on_shared_points_equals_the_cross_product(built_lib):
    """The same points for every configuration: the paired query is the cross product itself."""
    zc, sets, keep = _sets()
    A = int(zc["A"])
    q = np.asarray(zc["q"], dtype=np.float32)
    for name, descs in sets:
        ref = _sim_composed(descs, zc["tmat"], A, q)
        got = _sim_paired(descs, zc["tmat"], A, np.broadcast_to(q, (A,) + q.shape))
        assert all(np.array_equal(a, b) for a, b in zip(ref, got)), name


@pytest.mark.parametrize("P", [1, 3, 64, 2 ** 31 - 1])
def test_pair_index_arithmetic_is_64_bit(built_lib, P):
    S, s, cfg_begin = 8, 5, 7
    # more than 2^31 pairs wherever int32 configuration indices allow it (cfg_begin + cfg_count <= n_cfg < 2^31)
    cfg_count = min(2 ** 31 - 1 - cfg_begin, max(4, (2 ** 33) // P + 3))
    n_pairs = cfg_count * P
    assert n_pairs > 2 ** 31 or (P == 1 and n_pairs == 2 ** 31 - 1 - cfg_begin)
    cand = [0, 1, P - 1, P, 2 ** 31 - 2, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7,
            n_pairs - P, n_pairs - 1]
    t = np.array(sorted({x for x in cand if 0 <= x < n_pairs}), dtype=np.int64)
    c, i = np.empty_like(t), np.empty_like(t)
    jit = np.empty(len(t), dtype=np.uint64)
    _simlib().simpair_index(_p(t), ctypes.c_longlong(len(t)), ctypes.c_longlong(P), ctypes.c_int(cfg_begin),
                            ctypes.c_int(S), ctypes.c_int(s), _p(c), _p(i), _p(jit))
    for k, tk in enumerate(t.tolist()):
        assert (int(c[k]), int(i[k])) == divmod(tk, P), tk
        cfg = cfg_begin + tk // P
        assert int(jit[k]) == ((cfg * P + tk % P) * S + s) % 2 ** 64, tk


# ---------------------------------------------------------------- C ABI refusals (no kernel launch involved)
def test_abi_refuses_invalid_paired_queries(built_lib):
    near, tri, keep = _table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near])

    def call(descs=arr, n_sdf=2, xf=fake, n_cfg=4, begin=0, count=4, pts=fake, n_pts=100, val=fake, grad=fake):
        return L.pvb_composed_query_paired(descs, n_sdf, 0, xf, n_cfg, begin, count, pts, n_pts, nat.PVB_MESH_DEFAULT,
                                           val, grad, None, None)

    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    cases = [dict(descs=None), dict(xf=None), dict(pts=None), dict(val=None), dict(grad=None), dict(n_sdf=0),
             dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(begin=2, count=3), dict(n_pts=-1),
             dict(descs=nat.desc_array([near] * 129), n_sdf=129), dict(descs=nat.desc_array([near, gt])),
             dict(count=4, n_pts=2 ** 62)]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_paired"), (kw, msg)
    assert b"128" in (call(descs=nat.desc_array([near] * 129), n_sdf=129), L.pvb_last_error())[1]
    assert b"bounding-box" in (call(descs=nat.desc_array([near, gt])), L.pvb_last_error())[1]
    assert b"overflow" in (call(n_pts=2 ** 62), L.pvb_last_error())[1]
    # empty queries do nothing and succeed, without pointers to points or outputs
    assert call(n_pts=0, pts=None, val=None, grad=None) == 0
    assert call(count=0, pts=None, val=None, grad=None) == 0
    # the unfused path's transform
    assert L.pvb_transform_points_paired(None, 4, fake, 10, fake, None) == PVB_ERR_INVALID
    assert L.pvb_transform_points_paired(fake, 4, None, 10, fake, None) == PVB_ERR_INVALID
    assert L.pvb_transform_points_paired(fake, 4, fake, 2 ** 62, fake, None) == PVB_ERR_INVALID
    assert L.pvb_transform_points_paired(fake, 0, None, 10, None, None) == 0


# ---------------------------------------------------------------- shape rules, before any device work
def _composed_cpu(batch):
    import pytorch_volumetric_b200 as pv
    n = int(np.prod(batch))
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2)], pv.Transform3d(matrix=torch.eye(4).repeat(2 * n, 1, 1)))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=tuple(batch))
    return comp


def test_paired_shape_rules_raise_before_device_work(monkeypatch):
    from pytorch_volumetric_b200 import distributed as pd

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = _composed_cpu((3,))
    for shape in ((4, 5, 3), (2, 5, 3), (5, 3, 3, 3), (3, 5, 2), (3,)):
        with pytest.raises(ValueError, match="configuration batch"):
            comp.paired(torch.zeros(shape))
    comp2 = _composed_cpu((2, 3))
    for shape in ((3, 2, 4, 3), (2, 4, 5, 3), (6, 5, 3)):
        with pytest.raises(ValueError, match="configuration batch"):
            comp2.paired(torch.zeros(shape))
    with pytest.raises(ValueError, match="blocks"):
        comp.query_paired(torch.zeros(10, 3))                  # 10 points do not split over 3 configurations
    robot = types.SimpleNamespace(sdf=comp)
    with pytest.raises(ValueError, match="configuration batch"):
        pd.sharded_robot_query(robot, torch.zeros(4, 5, 3), paired=True)
    for gather in ("peer", "multicast", "dma"):
        with pytest.raises(ValueError, match="gather=True or gather=False"):
            pd.sharded_robot_query(robot, torch.zeros(3, 5, 3), gather=gather, paired=True)
