"""CPU tier of the scene queries (ComposedSDF.scene_clearance / scene_collision_cost, RobotSDF.scene_clearance /
scene_collision_cost, pvb_composed_query_scene_clearance / _collision_cost).

1. The host build of the kernels' per-configuration body (tests/hostsim/hostsim_scene.cpp) against an fp64
   definition written here, on a rotated and translated scene of a box, a sphere and a cylinder: clearance value,
   source and point, cost and twist.
2. Planted ties in (d, i, k): a duplicated source and duplicated points resolve to the first; -0 and +0 values of a
   grid scene tie through the host build, and in the composition route's reduction.
3. links masks, all links masked (+inf, -1, cost 0), a margin nothing is inside (exactly 0), K = 1 and K = 37.
4. The Python ValueErrors, raised before any device work; which scenes take the fused route.
5. The C entry points' refusals without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from hostsim_lib import PVB_ERR_INVALID, _p
from primitive_ref import box_ref, cylinder_ref
from pytorch_volumetric_b200 import _native as nat


def _rigid(n, seed, t=0.2):
    g = np.random.default_rng(seed)
    out = np.tile(np.eye(4), (n, 1, 1))
    for a in range(n):
        w = g.normal(0.0, 1.0, 3)
        th = np.linalg.norm(w)
        k = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
        out[a, :3, :3] = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        out[a, :3, 3] = g.uniform(-t, t, 3)
    return out.astype(np.float32)


def _scene():
    """(descriptors, fp64 evaluators in the sub-frame, scene transforms [3, 4, 4] fp32): a box, a sphere and a
    cylinder, rotated and translated."""
    import pytorch_volumetric_b200 as pv
    box, sph, cyl = pv.BoxSDF([0.2, 0.1, 0.15]), pv.SphereSDF(0.08), pv.CylinderSDF(0.05, 0.3)
    descs = [box.native_desc("cpu"), sph.native_desc("cpu"), cyl.native_desc("cpu")]

    def sphere(q):
        r = np.linalg.norm(q, axis=1)
        return r - 0.08, q / (r[:, None] + 1e-300)
    evals = [lambda q: box_ref([0.1, 0.05, 0.075], q), sphere, lambda q: cylinder_ref(0.05, 0.15, q)]
    return descs, evals, _rigid(3, seed=1, t=0.15)


def _sim(descs, sxf, inv, n_cfg, lp, links, margin, cfg_begin=0, cfg_count=None):
    S, K = lp.shape[:2]
    C = n_cfg - cfg_begin if cfg_count is None else cfg_count
    n = len(descs)
    arr = (nat.SdfDesc * n)(*descs)
    od = np.asarray(hs.bit_reversed_order(n), dtype=np.uint8)
    out = dict(val=np.empty(C, np.float32), grad=np.empty((C, 3), np.float32), link=np.empty(C, np.int32),
               point=np.empty(C, np.int32), cost=np.empty(C, np.float32), twist=np.empty((C, S, 6), np.float32))
    skipped = ctypes.c_longlong(0)
    hs.lib().simscene_fused(arr, ctypes.c_int(n), _p(od), _p(np.ascontiguousarray(sxf, np.float32)),
                            _p(np.ascontiguousarray(inv, np.float32)), ctypes.c_int(S), ctypes.c_int(n_cfg),
                            ctypes.c_int(cfg_begin), ctypes.c_int(C), _p(np.ascontiguousarray(lp, np.float32)),
                            ctypes.c_int(K), _p(np.asarray(links, np.uint8)), ctypes.c_float(margin),
                            *[_p(out[k]) for k in ("val", "grad", "link", "point", "cost", "twist")],
                            ctypes.byref(skipped))
    return out, skipped.value


def _fp64(evals, sxf, inv, n_cfg, lp, links, m):
    """The definition in fp64 from the fp32 inputs: per configuration the (d, i, k) minimum and its gradient, cost
    and twists, with sum|term| bounds."""
    S, K = lp.shape[:2]
    M = sxf.astype(np.float64)
    W = inv.astype(np.float64).reshape(S, n_cfg, 4, 4)
    res = {k: [] for k in ("val", "grad", "link", "point", "cost", "twist", "bc", "bt")}
    for a in range(n_cfg):
        best, cost = (np.inf, None, -1, -1), 0.0
        twist, bt, bc = np.zeros((S, 6)), np.zeros((S, 6)), 0.0
        for i in range(S):
            if not links[i]:
                continue
            x = lp[i].astype(np.float64) @ W[i, a, :3, :3].T + W[i, a, :3, 3]
            v, g = np.full(K, np.inf), np.zeros((K, 3))
            for s, ev in enumerate(evals):
                vs, gs = ev(x @ M[s, :3, :3].T + M[s, :3, 3])
                better = vs < v
                v, g = np.where(better, vs, v), np.where(better[:, None], gs @ M[s, :3, :3], g)
            k = int(np.argmin(v))
            if v[k] < best[0]:
                best = (v[k], g[k], i, k)
            h = np.maximum(m - v, 0.0)
            tau = np.concatenate([g, np.cross(x, g)], axis=1) * (2 * h)[:, None]
            cost += (h * h).sum()
            twist[i] = -tau.sum(0)
            bt[i] = np.abs(tau).sum(0) + 2 * h.sum() * (1 + np.abs(x).sum(1).max())
            bc += 2 * h.sum()
        for key, val in zip(("val", "grad", "link", "point", "cost", "twist", "bc", "bt"),
                            (best[0], best[1] if best[1] is not None else np.zeros(3), best[2], best[3], cost, twist,
                             bc, bt)):
            res[key].append(val)
    return {k: np.asarray(v) for k, v in res.items()}


def _inputs(S, n_cfg, K, seed):
    """W [S * n_cfg, 4, 4] (rigid, fp32) and link points [S, K, 3] that the poses carry about the scene."""
    g = np.random.default_rng(seed)
    inv = _rigid(S * n_cfg, seed=seed + 10, t=0.1)
    lp = g.normal(0.0, 0.12, (S, K, 3)).astype(np.float32)
    return inv, lp


# ---------------------------------------------------------------- 1. the host build against fp64
@pytest.mark.parametrize("K", [1, 37, 96])
@pytest.mark.parametrize("margin", [0.02, 0.1])
def test_host_build_against_fp64(K, margin):
    descs, evals, sxf = _scene()
    S, n_cfg = 3, 6
    inv, lp = _inputs(S, n_cfg, K, seed=K)
    links = [1, 1, 1]
    m = float(np.float32(margin))
    got, _ = _sim(descs, sxf, inv, n_cfg, lp, links, m)
    ref = _fp64(evals, sxf, inv, n_cfg, lp, links, m)
    assert np.abs(got["val"] - ref["val"]).max() <= 1e-5
    # the same (i, k) unless the fp64 runner-up is within the fp32 noise
    same = (got["link"] == ref["link"]) & (got["point"] == ref["point"])
    assert same.mean() >= 0.8
    assert np.abs(got["grad"][same] - ref["grad"][same]).max() <= 1e-4
    assert (np.abs(got["cost"] - ref["cost"]) <= 1e-5 * ref["bc"] + 1e-12).all()
    assert (np.abs(got["twist"] - ref["twist"]) <= 1e-5 * ref["bt"] + 1e-12).all()
    assert (got["cost"] > 0).any() or (ref["cost"] == 0).all()


# ---------------------------------------------------------------- 2. ties
def test_planted_ties_resolve_to_the_first_source_and_point():
    descs, _, sxf = _scene()
    S, n_cfg, K = 3, 4, 40
    inv, lp = _inputs(S, n_cfg, K, seed=5)
    inv = inv.reshape(S, n_cfg, 4, 4)
    inv[1] = inv[0]                                    # source 1 is source 0: every value ties
    lp[1] = lp[0]
    lp[:, 33] = lp[:, 7]                               # point 33 repeats point 7 of every source
    got, _ = _sim(descs, sxf, inv.reshape(-1, 4, 4), n_cfg, lp, [1, 1, 0], 0.05)
    assert (got["link"] == 0).all()
    assert not (got["point"] == 33).any()
    # -0 and +0 tie through the host build: a grid scene storing -0 at voxel (1, 1, 1) and +0 at (2, 2, 2), 1
    # elsewhere, read at voxel centres under identity poses; the first (i, k) at a zero wins, whichever sign it has
    tv = torch.ones(5, 5, 5)
    tv[1, 1, 1], tv[2, 2, 2] = -0.0, 0.0
    grid, keep = hs.grid_desc(tv, torch.zeros(125, 3), [(0.0, 4.0)] * 3, np.array([[0.0, 4.0]] * 3))
    eye = np.tile(np.eye(4, dtype=np.float32), (2 * 2, 1, 1))
    neg, pos, one = (1.0, 1.0, 1.0), (2.0, 2.0, 2.0), (3.0, 3.0, 3.0)
    for pts, want in ((([one, neg, pos], [pos, one, neg]), (0, 1, True)),
                      (([one, pos, neg], [neg, one, pos]), (0, 1, False)),
                      (([one, one, one], [one, neg, pos]), (1, 1, True)),
                      (([one, one, one], [one, pos, neg]), (1, 1, False))):
        tie, _ = _sim([grid], np.eye(4, dtype=np.float32)[None], eye, 2, np.array(pts, np.float32), [1, 1], 0.5)
        assert (tie["val"] == 0).all() and (np.signbit(tie["val"]) == want[2]).all(), (pts, tie["val"])
        assert (tie["link"] == want[0]).all() and (tie["point"] == want[1]).all(), (pts, tie["link"], tie["point"])
    # the same key order in the composition route's reduction
    from pytorch_volumetric_b200.sdf import ComposedSDF
    v = torch.tensor([[0.5, 0.0, -0.0, 0.0], [0.5, -0.0, 0.0, 1.0], [float("nan"), 2.0, -0.0, -0.0]])
    assert ComposedSDF._first_minimum(v).tolist() == [1, 1, 2]
    assert hs.lib().simscl_key(-0.0, 3, 9) == hs.lib().simscl_key(0.0, 3, 9)
    assert hs.lib().simscl_key(0.0, 2, 9) < hs.lib().simscl_key(0.0, 3, 0)


# ---------------------------------------------------------------- 3. masks, empty margins
def test_links_masks_and_margins():
    descs, evals, sxf = _scene()
    S, n_cfg, K = 3, 5, 50
    inv, lp = _inputs(S, n_cfg, K, seed=7)
    full, _ = _sim(descs, sxf, inv, n_cfg, lp, [1, 1, 1], 0.1)
    part, _ = _sim(descs, sxf, inv, n_cfg, lp, [0, 1, 1], 0.1)
    assert (part["link"] != 0).all() and (part["twist"][:, 0] == 0).all()
    assert (part["val"] >= full["val"]).all()
    ref = _fp64(evals, sxf, inv, n_cfg, lp, [0, 1, 1], float(np.float32(0.1)))
    assert (np.abs(part["cost"] - ref["cost"]) <= 1e-5 * ref["bc"] + 1e-12).all()
    none, _ = _sim(descs, sxf, inv, n_cfg, lp, [0, 0, 0], 0.1)
    assert np.isinf(none["val"]).all() and (none["val"] > 0).all() and (none["grad"] == 0).all()
    assert (none["link"] == -1).all() and (none["point"] == -1).all()
    assert (none["cost"] == 0).all() and (none["twist"] == 0).all()
    # nothing inside the margin: exactly 0, every step skipped, the clearance unchanged
    far, skipped = _sim(descs, sxf, inv, n_cfg, lp, [1, 1, 1], -10.0)
    assert (far["cost"] == 0).all() and (far["twist"] == 0).all() and not np.signbit(far["twist"]).any()
    assert skipped == n_cfg * S * 2
    assert np.array_equal(far["val"], full["val"]) and np.array_equal(far["point"], full["point"])
    # a slab reproduces the rows of the full call
    sl, _ = _sim(descs, sxf, inv, n_cfg, lp, [1, 1, 1], 0.1, cfg_begin=2, cfg_count=2)
    for k in sl:
        assert np.array_equal(sl[k], full[k][2:4]), k


# ---------------------------------------------------------------- 4. Python rules
def _comp(S=3, A=2):
    import pytorch_volumetric_b200 as pv
    comp = pv.ComposedSDF([pv.SphereSDF(0.1)] * S, pv.Transform3d(matrix=torch.eye(4).repeat(S * A, 1, 1)))
    comp.set_transforms(pv.Transform3d(matrix=torch.eye(4).repeat(S * A, 1, 1)), batch_dim=(A,))
    return comp


def test_scene_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = _comp()
    scene = pv.BoxSDF([0.1, 0.1, 0.1])
    for shape in ((3, 4), (2, 4, 3), (3, 0, 3), (3, 4, 2), (1, 3, 4, 3), (3, 1 << 24, 3)):
        lp = torch.zeros(1).expand(*shape)
        for call in (lambda: comp.query_scene_clearance(scene, lp), lambda: comp.scene_clearance(scene, lp),
                     lambda: comp.query_scene_collision_cost(scene, lp, 0.1),
                     lambda: comp.scene_collision_cost(scene, lp, 0.1)):
            with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
                call()
    lp = torch.zeros(3, 5, 3)
    for bad in (torch.ones(3), torch.ones(2, dtype=torch.bool), np.ones(3, dtype=np.int64),
                torch.ones(3, 3, dtype=torch.bool)):
        with pytest.raises(ValueError, match="bool mask"):
            comp.query_scene_clearance(scene, lp, bad)
        with pytest.raises(ValueError, match="bool mask"):
            comp.scene_collision_cost(scene, lp, 0.1, bad)
    for margin in (float("nan"), float("inf"), "x", None, torch.tensor([0.1, 0.2])):
        with pytest.raises(ValueError, match="margin"):
            comp.query_scene_collision_cost(scene, lp, margin)
    for begin, count in ((0, 0), (2, 0), (1, 2), (-1, 1), (0, -1)):
        with pytest.raises(ValueError, match="slab"):
            comp.query_scene_clearance(scene, lp, cfg_begin=begin, cfg_count=count)
        with pytest.raises(ValueError, match="slab"):
            comp.query_scene_collision_cost(scene, lp, 0.1, cfg_begin=begin, cfg_count=count)
    with pytest.raises(ValueError, match="one pose"):
        comp.scene_clearance(_comp(1, 2), lp)
    with pytest.raises(ValueError, match="ObjectFrameSDF"):
        comp.scene_collision_cost(lambda p: p, lp, 0.1)
    from pytorch_volumetric_b200.model_to_sdf import RobotSDF
    robot = RobotSDF.__new__(RobotSDF)
    robot.sdf = comp
    with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
        robot.scene_collision_cost(scene, 0.1, torch.zeros(2, 5, 3))
    with pytest.raises(ValueError, match="margin"):
        robot.scene_collision_cost(scene, float("nan"), lp)
    with pytest.raises(ValueError, match="bool mask"):
        robot.scene_clearance(scene, lp, torch.ones(3))


def test_which_scenes_take_the_fused_route():
    import pytorch_volumetric_b200 as pv
    from helpers import opaque_sdfs
    comp = _comp()
    box, sph, cyl = pv.BoxSDF([0.1, 0.2, 0.3]), pv.SphereSDF(0.1), pv.CylinderSDF(0.1, 0.2)
    T = pv.Transform3d(matrix=torch.from_numpy(_rigid(3, seed=2)))
    for scene in (box, sph, cyl, pv.ComposedSDF([box, sph, cyl], T), pv.ComposedSDF([box] * 128, pv.Transform3d(
            matrix=torch.eye(4).repeat(128, 1, 1)))):
        fused = comp._scene_fused(scene, "cpu")
        assert fused is not None
        descs, n, xf = fused
        n_expect = len(scene.sdfs) if isinstance(scene, pv.ComposedSDF) else 1
        assert n == n_expect and tuple(xf.reshape(-1, 4, 4).shape) == (n_expect, 4, 4)
    assert torch.equal(comp._scene_fused(box, "cpu")[2], torch.eye(4))

    class GtGrid(pv.ObjectFrameSDF):               # stands in for a LOOKUP_GT_SDF CachedSDF: its descriptor flag
        def __call__(self, p):
            return box(p)

        def surface_bounding_box(self, **kw):
            return box.surface_bounding_box(**kw)

        def native_desc(self, device):
            d = box.native_desc(device)
            d.kind, d.flags = nat.PVB_KIND_GRID, nat.PVB_GRID_OOB_GT
            return d

    class MeshLike(GtGrid):
        def native_desc(self, device):
            d = box.native_desc(device)
            d.kind = nat.PVB_KIND_MESH
            return d
    for scene in (opaque_sdfs(pv, [box])[0], GtGrid(), MeshLike(), pv.ComposedSDF([box, MeshLike()], pv.Transform3d(
            matrix=torch.eye(4).repeat(2, 1, 1))), pv.ComposedSDF([box] * 129, pv.Transform3d(
            matrix=torch.eye(4).repeat(129, 1, 1)))):
        assert comp._scene_fused(scene, "cpu") is None
    # any sub-SDF kind in the robot, up to 255 of them
    assert _comp(3, 1).__class__(opaque_sdfs(pv, [box]) * 255, pv.Transform3d(
        matrix=torch.eye(4).repeat(255, 1, 1)))._scene_fused(box, "cpu") is not None
    assert _comp(3, 1).__class__([box] * 256, pv.Transform3d(
        matrix=torch.eye(4).repeat(256, 1, 1)))._scene_fused(box, "cpu") is None


# ---------------------------------------------------------------- 5. C ABI refusals
def test_abi_refuses_invalid_scene_queries(built_lib):
    import pytorch_volumetric_b200 as pv
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    box = pv.BoxSDF([0.1, 0.1, 0.1]).native_desc("cpu")
    arr = nat.desc_array([box, box])
    on3 = (ctypes.c_uint8 * 3)(1, 1, 1)
    gt = box.copy()
    gt.kind, gt.flags = nat.PVB_KIND_GRID, nat.PVB_GRID_OOB_GT
    mesh = box.copy()
    mesh.kind = nat.PVB_KIND_MESH
    bad_kind = box.copy()
    bad_kind.kind = 7

    def clearance(scene=arr, n_scene=2, sxf=fake, inv=fake, n_sdf=3, n_cfg=4, begin=0, count=4, pts=fake, K=100,
                  links=on3, a=fake, b=fake, margin=None):
        return L.pvb_composed_query_scene_clearance(scene, n_scene, sxf, inv, n_sdf, n_cfg, begin, count, pts, K,
                                                    links, a, b, None, None, None)

    def cost(margin=0.05, scene=arr, n_scene=2, sxf=fake, inv=fake, n_sdf=3, n_cfg=4, begin=0, count=4, pts=fake,
             K=100, links=on3, a=fake, b=fake):
        return L.pvb_composed_query_scene_collision_cost(scene, n_scene, sxf, inv, n_sdf, n_cfg, begin, count, pts,
                                                         K, links, margin, a, b, None)

    cases = [dict(scene=None), dict(sxf=None), dict(inv=None), dict(pts=None), dict(a=None), dict(b=None),
             dict(links=None), dict(n_scene=0), dict(n_sdf=0), dict(n_sdf=256, links=(ctypes.c_uint8 * 256)()),
             dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0), dict(begin=2, count=3), dict(K=0),
             dict(K=-1), dict(K=1 << 24), dict(scene=nat.desc_array([box] * 129), n_scene=129),
             dict(scene=nat.desc_array([box, mesh])), dict(scene=nat.desc_array([box, gt])),
             dict(scene=nat.desc_array([box, bad_kind]))]
    for fn, name in ((clearance, b"pvb_composed_query_scene_clearance"),
                     (cost, b"pvb_composed_query_scene_collision_cost")):
        for kw in cases:
            rc = fn(**kw)
            msg = L.pvb_last_error()
            assert rc == PVB_ERR_INVALID and msg.startswith(name), (name, kw, msg)
        assert b"2^24" in (fn(K=1 << 24), L.pvb_last_error())[1]
        assert b"no mesh" in (fn(scene=nat.desc_array([box, mesh])), L.pvb_last_error())[1]
        assert b"no mesh" in (fn(scene=nat.desc_array([box, gt])), L.pvb_last_error())[1]
        assert b"255" in (fn(n_sdf=256, links=(ctypes.c_uint8 * 256)()), L.pvb_last_error())[1]
    for margin in (float("nan"), float("inf"), -math.inf):
        assert cost(margin=margin) == PVB_ERR_INVALID and b"finite" in L.pvb_last_error()
