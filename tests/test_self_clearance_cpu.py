"""CPU tier for self-clearance queries (ComposedSDF.self_clearance / RobotSDF.self_clearance /
pvb_composed_query_self_clearance): every configuration's smallest distance between its own sub-SDFs, over the link
points of every source sub-SDF against the sub-SDFs its row of `allowed` names.

1. The key packing: the unsigned order of self_clearance_key is the (value, i, k) order.
2. The device arithmetic, compiled for the host by tests/hostsim/hostsim_self_clearance.cpp in the order the kernels
   run it: robot_self_clearance_kernel's sequence under every chunk size, unit order, seeding, sharing and first visit,
   then self_clearance_finish_kernel -- equal bit for bit (value, gradient, i, k, j) to the composition route, which
   is the definition: every source's points posed with W_i (pvb_transform_points_paired's arithmetic), the host build
   of the paired clearance query on the allowed sub-composition, reduced over i by (value, i).  On the nearest,
   trilinear, mixed, primitive and primitive+grid golden sets; with duplicated points and sub-SDFs; with an empty row,
   an empty matrix and an asymmetric matrix.  A masked link is never visited.
3. RobotSDF.self_collision_pairs and the analytic surface samples of link_surface_points.
4. The C ABI refusals and the Python shape rules, without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from hostsim_lib import PVB_ERR_INVALID, _p
from pytorch_volumetric_b200 import _native as nat


def _fused(descs, xf, inv, n_cfg, lp, allowed, cfg_begin=0, cfg_count=None, chunk=None, lanes=32, share=1,
           unit_order=0, shuffle_seed=0, seeded=1, first=-1):
    """(keys [cfg_count], visits [8, 8]) of robot_self_clearance_kernel's sequence."""
    S, K = lp.shape[:2]
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    keys = np.empty(cfg_count, np.uint64)
    visits = np.zeros(64, np.int64)
    hs.lib().simscl_fused((nat.SdfDesc * S)(*descs), ctypes.c_int(S), _p(xf), _p(inv), ctypes.c_int(n_cfg),
                          ctypes.c_int(cfg_begin), ctypes.c_int(cfg_count), _p(lp), ctypes.c_int(K),
                          _p(hs.masks(allowed)), ctypes.c_int(chunk or K), ctypes.c_int(lanes), ctypes.c_int(share),
                          ctypes.c_int(unit_order), ctypes.c_int(shuffle_seed), ctypes.c_int(seeded),
                          ctypes.c_int(first), _p(keys), _p(visits))
    return keys, visits.reshape(8, 8)


def _finish(descs, xf, inv, n_cfg, lp, allowed, keys, cfg_begin=0):
    S, K = lp.shape[:2]
    R = len(keys)
    out = (np.empty(R, np.float32), np.empty((R, 3), np.float32), np.empty(R, np.int32), np.empty(R, np.int32),
           np.empty(R, np.int32))
    hs.lib().simscl_finish((nat.SdfDesc * S)(*descs), ctypes.c_int(S), _p(xf), _p(inv), ctypes.c_int(n_cfg),
                           ctypes.c_int(cfg_begin), ctypes.c_int(R), _p(lp), ctypes.c_int(K), _p(hs.masks(allowed)),
                           _p(np.ascontiguousarray(keys)), *[_p(a) for a in out])
    return out


def _pose(inv, n_cfg, i, lp_i, cfg_begin, cfg_count):
    """[cfg_count, K, 3]: link points of source i posed by W_i with composed_xform's fused multiply-adds (the host
    build, so that the rounding is the kernels')."""
    S = len(inv) // n_cfg
    w = np.asarray(inv, dtype=np.float32).reshape(S, n_cfg, 4, 4)[i, cfg_begin:cfg_begin + cfg_count]
    w = np.ascontiguousarray(w)
    p = np.ascontiguousarray(lp_i, dtype=np.float32)
    out = np.empty((cfg_count, len(p), 3), np.float32)
    hs.lib().simscl_pose(_p(w), ctypes.c_int(cfg_count), _p(p), ctypes.c_int(len(p)), _p(out))
    return out


def _composition_route(descs, xf, inv, n_cfg, lp, allowed, cfg_begin=0, cfg_count=None):
    """The definition: per source i with an allowed row, its points posed with W_i, the host build of the paired
    clearance query (robot_paired_clearance_kernel + paired_clearance_finish_kernel) on the allowed sub-composition,
    which mapped back; then the minimum over i by (value, i)."""
    S, K = lp.shape[:2]
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    tm = np.asarray(xf, dtype=np.float32).reshape(S, n_cfg, 4, 4)
    per = []
    for i in range(S):
        js = [j for j in range(S) if allowed[i][j] and j != i]
        if not js:
            continue
        x = _pose(inv, n_cfg, i, lp[i], cfg_begin, cfg_count)[:, None]              # [cfg_count, 1, K, 3]
        sub = [descs[j] for j in js]
        sub_xf = np.ascontiguousarray(tm[js].reshape(len(js) * n_cfg, 4, 4))
        keys = hs.pcl_keys(sub, sub_xf, n_cfg, x, cfg_begin=cfg_begin)[0]
        v, g, pt, w = hs.pcl_finish(sub, sub_xf, n_cfg, x, keys, cfg_begin=cfg_begin)
        per.append((i, v, g, pt, np.asarray(js, np.int32)[w]))
    if not per:
        return (np.full(cfg_count, np.inf, np.float32), np.zeros((cfg_count, 3), np.float32),
                *[np.full(cfg_count, -1, np.int32) for _ in range(3)])
    v = np.stack([r[1] for r in per], 1)
    vz = np.where(v == 0, 0.0, v)                                               # -0 == +0
    vz = np.where(np.isnan(vz), np.inf, vz)
    pos = np.argmax(vz == vz.min(axis=1, keepdims=True), axis=1)               # first source on ties
    rows = np.arange(cfg_count)
    return (v[rows, pos], np.stack([r[2] for r in per], 1)[rows, pos],
            np.asarray([r[0] for r in per], np.int32)[pos], np.stack([r[3] for r in per], 1)[rows, pos],
            np.stack([r[4] for r in per], 1)[rows, pos])


def _assert_same(got, ref, what):
    for a, b, name in zip(got, ref, ("val", "grad", "src", "point", "which")):
        assert np.array_equal(a, b), (what, name, int(np.sum(a != b)))


def _key_of(ref):
    return np.array([hs.lib().simscl_key(float(v), int(i), int(k)) for v, i, k in zip(ref[0], ref[2], ref[3])],
                    np.uint64)


# ---------------------------------------------------------------- 1. key packing
def test_self_clearance_key_orders_value_then_source_then_point():
    values = [-np.inf, -1.5, -1e-30, -0.0, 0.0, 1e-30, 0.25, 0.25000003, np.inf, np.nan]
    ks = [0, 1, 2, (1 << 24) - 2, (1 << 24) - 1]
    cands = [(v, i, k) for v in values for i in range(8) for k in ks]
    keys = [hs.lib().simscl_key(v, i, k) for v, i, k in cands]

    def rank(c):
        v, i, k = c
        vv = math.inf if math.isnan(v) else (0.0 if v == 0 else v)
        return (1 if math.isnan(v) else 0, vv, i, k)
    ranks = [rank(c) for c in cands]
    order = sorted(range(len(cands)), key=lambda t: ranks[t])
    for a, b in zip(order, order[1:]):
        assert (keys[a] < keys[b]) == (ranks[a] < ranks[b]) and (keys[a] == keys[b]) == (ranks[a] == ranks[b]), \
            (cands[a], cands[b])
    assert len(set(keys)) == len(set(ranks))                     # -0 and +0 give the same key, nothing else collides


# ---------------------------------------------------------------- 2. the fused sequence against the composition
@pytest.mark.parametrize("A", [3, 37])
def test_fused_self_clearance_equals_the_composition_route(built_lib, A):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else hs.trajectory(zc["tmat"], S, A0, A, seed=A)
    tm = np.ascontiguousarray(tm, dtype=np.float32)
    inv = hs.inverse(tm)
    for name, descs in sets:
        S = len(descs)
        for K in (1, 45, 130):
            lp = hs.link_points(zc, tm, S, A, K, seed=K + A)
            for case, allowed in hs.allowed_cases(S).items():
                ref = _composition_route(descs, tm, inv, A, lp, allowed)
                keys, visits = _fused(descs, tm, inv, A, lp, allowed)
                _assert_same(_finish(descs, tm, inv, A, lp, allowed, keys), ref, (name, K, case))
                if case == "empty":
                    assert (keys == np.uint64(~np.uint64(0))).all() and (ref[2] == -1).all() and np.isinf(ref[0]).all()
                    continue
                assert np.array_equal(keys, _key_of(ref)), (name, K, case)
                # a masked link is never visited
                m = hs.masks(allowed)
                for i in range(S):
                    for j in range(8):
                        if not (int(m[i]) >> j) & 1:
                            assert visits[i, j] == 0, (name, case, i, j)
                # chunk sizes, unit widths, sharing, unit orders, seeding and first visits: the same keys
                for chunk in sorted({1, 7, 32, 64, K}):
                    for order, seed in ((0, 0), (1, 0), (2, chunk + K)):
                        got = _fused(descs, tm, inv, A, lp, allowed, chunk=chunk, share=(order + 1) & 1,
                                     unit_order=order, shuffle_seed=seed, seeded=(chunk + order) & 1)[0]
                        assert np.array_equal(got, keys), (name, K, case, chunk, order)
                for first in range(S):
                    got = _fused(descs, tm, inv, A, lp, allowed, chunk=32, first=first, lanes=64)[0]
                    assert np.array_equal(got, keys), (name, K, case, first)
            # slabs: the absolute configuration picks the transforms
            allowed = hs.allowed_cases(S)["full"]
            for begin, count in ((1, A - 1), (A // 2, 1), (A - 2, 2)):
                ks = _fused(descs, tm, inv, A, lp, allowed, cfg_begin=begin, cfg_count=count, chunk=32)[0]
                _assert_same(_finish(descs, tm, inv, A, lp, allowed, ks, cfg_begin=begin),
                             _composition_route(descs, tm, inv, A, lp, allowed, begin, count), (name, begin, count))


def test_self_clearance_argmins_vary(built_lib):
    """The golden sub-SDFs overlap: configurations in collision, values that differ, and an argmin that moves."""
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    tm = np.ascontiguousarray(hs.trajectory(zc["tmat"], S, A0, 40, seed=5), dtype=np.float32)
    inv = hs.inverse(tm)
    for name, descs in sets:
        S = len(descs)
        lp = hs.link_points(zc, tm, S, 40, 64, seed=9)
        ref = _composition_route(descs, tm, inv, 40, lp, hs.allowed_cases(S)["full"])
        assert (ref[0] < 0).any() and len(set(ref[0].tolist())) > 1, name
        assert len(set(zip(ref[2].tolist(), ref[3].tolist()))) > 1, name


def test_ties_report_the_first_source_and_point(built_lib):
    zc, sets, keep = hs.all_sets()
    S, A0 = int(zc["S"]), int(zc["A"])
    base = hs.trajectory(zc["tmat"], S, A0, 6, seed=7).reshape(S, 6, 4, 4)
    descs = sets[0][1]
    # sub-SDF 0 listed twice (positions 0 and 2) under the same transforms, with the same link points; every link's
    # points twice in a row
    dup = [descs[0], descs[1], descs[0], descs[2]]
    tm = np.ascontiguousarray(np.concatenate([base[0:1], base[1:2], base[0:1], base[2:3]]).reshape(24, 4, 4),
                              dtype=np.float32)
    inv = hs.inverse(tm)
    lp = hs.link_points(zc, tm, 4, 6, 50, seed=3)
    lp[2] = lp[0]
    lp = np.ascontiguousarray(np.concatenate([lp, lp], axis=1))
    allowed = [[i != j and {i, j} != {0, 2} for j in range(4)] for i in range(4)]
    ref = _composition_route(dup, tm, inv, 6, lp, allowed)
    assert (ref[3] < 50).all() and (ref[2] != 2).all()              # first point, first of two equal sources
    assert (ref[4] != 2).all()                                       # first of two equal targets
    for kw in ({}, dict(chunk=7, unit_order=1, share=0), dict(chunk=32, unit_order=2, shuffle_seed=3, seeded=0)):
        keys = _fused(dup, tm, inv, 6, lp, allowed, **kw)[0]
        _assert_same(_finish(dup, tm, inv, 6, lp, allowed, keys), ref, kw)


# ---------------------------------------------------------------- 3. RobotSDF defaults
_FIXED_CHAIN = """<robot name="r">
<link name="base"><visual><origin xyz="0 0 0.05"/><geometry><box size="0.2 0.2 0.1"/></geometry></visual></link>
<link name="upper"><visual><origin xyz="0 0 0.1"/><geometry><cylinder radius="0.04" length="0.2"/></geometry></visual>
  <visual><origin xyz="0 0 0.2"/><geometry><sphere radius="0.05"/></geometry></visual></link>
<link name="bracket"><visual><origin xyz="0 0.03 0"/><geometry><box size="0.05 0.05 0.05"/></geometry></visual></link>
<link name="fore"><visual><origin xyz="0 0 0.1"/><geometry><box size="0.05 0.06 0.2"/></geometry></visual></link>
<link name="hand"><visual><geometry><sphere radius="0.04"/></geometry></visual></link>
<joint name="j1" type="revolute"><parent link="base"/><child link="upper"/><origin xyz="0 0 0.1"/>
  <axis xyz="0 0 1"/></joint>
<joint name="jf" type="fixed"><parent link="upper"/><child link="bracket"/><origin xyz="0 0 0.2"/></joint>
<joint name="j2" type="revolute"><parent link="bracket"/><child link="fore"/><origin xyz="0 0 0.02"/>
  <axis xyz="0 1 0"/></joint>
<joint name="j3" type="revolute"><parent link="fore"/><child link="hand"/><origin xyz="0 0 0.2"/>
  <axis xyz="1 0 0"/></joint>
</robot>"""


def _robot(urdf_text, end, **kw):
    from pytorch_volumetric_b200 import kinematics
    from pytorch_volumetric_b200.model_to_sdf import RobotSDF
    chain = kinematics.build_serial_chain_from_urdf(urdf_text, end)
    robot = RobotSDF.__new__(RobotSDF)
    # the constructor installs a configuration (GPU); the link layout and the defaults need none of it
    orig = RobotSDF.set_joint_configuration
    try:
        RobotSDF.set_joint_configuration = lambda self, q=None: None
        RobotSDF.__init__(robot, chain, **kw)
    finally:
        RobotSDF.set_joint_configuration = orig
    return robot


def test_self_collision_pairs_of_the_arm_and_of_fixed_joints(tmp_path):
    import workloads
    path, end = workloads.write_primitive_arm(str(tmp_path))
    with open(path) as fh:
        arm = _robot(fh.read(), end, primitive_visuals=True)
    S = len(arm.sdf_to_link_name)
    assert S == 8
    idx = torch.arange(S)
    assert torch.equal(arm.self_collision_pairs(), (idx[:, None] - idx[None, :]).abs() >= 2)
    r = _robot(_FIXED_CHAIN, "hand", primitive_visuals=True)
    assert r.sdf_to_link_name == ["base", "upper", "upper", "bracket", "fore", "hand"]
    m = torch.tensor([0, 1, 1, 1, 2, 3])                       # movable joints up to each visual's frame
    got = r.self_collision_pairs()
    assert got.dtype == torch.bool and torch.equal(got, (m[:, None] - m[None, :]).abs() >= 2)
    # same rigid body (one link's two visuals, and a link behind a fixed joint) and neighbours: excluded
    for i, j in ((1, 2), (1, 3), (2, 3), (0, 1), (3, 4), (4, 5)):
        assert not got[i, j] and not got[j, i]
    assert got[0, 4] and got[1, 5] and got[3, 5]


def test_link_surface_points_of_primitives_lie_on_the_surface(tmp_path):
    import primitive_ref as pr
    r = _robot(_FIXED_CHAIN, "hand", primitive_visuals=True)
    pts = r.link_surface_points(num_points=500, seed=3)
    assert pts.shape == (6, 500, 3) and pts.dtype == torch.float32
    assert r.link_surface_points(num_points=500, seed=3) is pts                   # cached
    assert not torch.equal(r.link_surface_points(num_points=500, seed=4), pts)
    for s, link in enumerate(r.sdf.sdfs):
        q = pts[s].double().numpy()
        if hasattr(link, "size"):
            v = pr.box_ref(np.asarray(link._half), q)[0]
            # area-uniform: every face pair gets points in proportion to its area
            h = np.asarray(link._half)
            on = np.argmax(np.abs(np.abs(q) - h) < 1e-6, axis=1)
            frac = np.bincount(on, minlength=3) / len(q)
            area = np.array([h[1] * h[2], h[0] * h[2], h[0] * h[1]])
            assert np.allclose(frac, area / area.sum(), atol=0.08), (s, frac)
        elif hasattr(link, "length"):
            v = pr.cylinder_ref(link.radius, 0.5 * link.length, q)[0]
        else:
            v = pr.sphere_ref(link.radius, q)[0]
        assert np.abs(v).max() <= 1e-6, (s, np.abs(v).max())


# ---------------------------------------------------------------- 4. C ABI refusals (no kernel launch involved)
def test_abi_refuses_invalid_self_clearance_queries(built_lib):
    near, tri, keep = hs.table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near, tri])
    rows3 = (ctypes.c_uint8 * 3)(0b110, 0b101, 0b011)

    def call(descs=arr, n_sdf=3, xf=fake, inv=fake, n_cfg=4, begin=0, count=4, pts=fake, K=100, allowed=rows3,
             keys=fake, val=fake, grad=fake):
        return L.pvb_composed_query_self_clearance(descs, n_sdf, xf, inv, n_cfg, begin, count, pts, K, allowed, keys,
                                                   val, grad, None, None, None, None)

    gt = near.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    mesh = near.copy()
    mesh.kind = nat.PVB_KIND_MESH
    bad_kind = near.copy()
    bad_kind.kind = 7
    nine = (ctypes.c_uint8 * 9)()
    cases = [dict(descs=None), dict(xf=None), dict(inv=None), dict(pts=None), dict(val=None), dict(grad=None),
             dict(keys=None), dict(allowed=None), dict(n_sdf=0), dict(n_cfg=0), dict(begin=-1), dict(count=-1),
             dict(count=0), dict(begin=2, count=3), dict(K=0), dict(K=-1), dict(K=1 << 24),
             dict(allowed=(ctypes.c_uint8 * 3)(0b1110, 0, 0)), dict(allowed=(ctypes.c_uint8 * 3)(0, 0, 0x80)),
             dict(descs=nat.desc_array([near] * 9), n_sdf=9, allowed=nine),
             dict(descs=nat.desc_array([near] * 129), n_sdf=129),
             dict(descs=nat.desc_array([near, mesh, near])), dict(descs=nat.desc_array([near, gt, near])),
             dict(descs=nat.desc_array([near, bad_kind, near]))]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_self_clearance"), (kw, msg)
    assert b"2^24" in (call(K=1 << 24), L.pvb_last_error())[1]
    assert b"empty configuration slab" in (call(count=0), L.pvb_last_error())[1]
    assert b"beyond n_sdf" in (call(allowed=(ctypes.c_uint8 * 3)(0b1000, 0, 0)), L.pvb_last_error())[1]
    assert b"keys" in (call(keys=None), L.pvb_last_error())[1]
    assert b"at most 8" in (call(descs=nat.desc_array([near] * 9), n_sdf=9, allowed=nine), L.pvb_last_error())[1]
    assert b"no mesh" in (call(descs=nat.desc_array([near, mesh, near])), L.pvb_last_error())[1]
    assert b"no mesh" in (call(descs=nat.desc_array([near, gt, near])), L.pvb_last_error())[1]


# ---------------------------------------------------------------- shape rules, before any device work
def test_self_clearance_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2), pv.SphereSDF(0.3)],
                          pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    ok = torch.ones(3, 3, dtype=torch.bool)
    for shape in ((3, 4), (2, 4, 3), (4, 4, 3), (3, 0, 3), (3, 4, 2), (1, 3, 4, 3), (3, 1 << 24, 3)):
        lp = torch.zeros(1).expand(*shape) if len(shape) else torch.zeros(())
        with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
            comp.query_self_clearance(lp, ok)
        with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
            comp.self_clearance(lp, ok)
    lp = torch.zeros(3, 5, 3)
    for bad in (torch.ones(3, 3), torch.ones(3, 4, dtype=torch.bool), torch.ones(2, 2, dtype=torch.bool),
                np.ones((3, 3), dtype=np.int64), [[True] * 3] * 2):
        with pytest.raises(ValueError, match="bool matrix"):
            comp.query_self_clearance(lp, bad)
    for begin, count in ((0, 0), (2, 0), (1, 2), (-1, 1), (0, -1)):
        with pytest.raises(ValueError, match="slab"):
            comp.query_self_clearance(lp, ok, cfg_begin=begin, cfg_count=count)
    with pytest.raises(ValueError, match="slab"):
        comp.query_self_clearance(lp, ok, cfg_begin=2)
    # RobotSDF delegates
    from pytorch_volumetric_b200.model_to_sdf import RobotSDF
    robot = RobotSDF.__new__(RobotSDF)
    robot.sdf = comp
    with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
        robot.self_clearance(torch.zeros(2, 5, 3), ok)
    with pytest.raises(ValueError, match="bool matrix"):
        robot.self_clearance(lp, ok.int())
