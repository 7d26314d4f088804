"""GPU: collision-cost queries (ComposedSDF.collision_cost / query_collision_cost, RobotSDF.collision_cost,
pvb_composed_query_collision_cost).

For every configuration and segment, cost = sum_p max(0, m - d)^2 and the twist gradient per sub-SDF; for a robot the
joint gradient.  Every route is compared with the fp64 sum of the fp32 per-pair query(..., return_which=True)
outputs, within 1e-5 * sum|term|: the fused kernel on the golden nearest, trilinear and primitive sets and the 8-link
arm, the composition route on meshes, LOOKUP_GT_SDF grids, more than 8 sub-SDFs and sub-SDFs without descriptors.
Far clouds cost exactly 0; calls repeat bit for bit; slabs reproduce the rows of the full call bit for bit; the joint
gradient matches fp64 finite differences on a general chain and the fp64 Jacobian transpose on the cached arm."""
import numpy as np
import pytest
import torch

import workloads
from helpers import arm_points, arm_robot, cached_arm, cached_from_golden, golden, golden_sets, opaque_sdfs, pv_factory
from robot_ref import build_robot, joint_values

pytestmark = pytest.mark.gpu


def _no_composition(monkeypatch, comp):
    def boom(*a, **k):
        raise AssertionError("composition route taken")
    monkeypatch.setattr(comp, "_composed_collision_cost", boom)
    monkeypatch.setattr(comp, "_generic_query", boom)


def _reference(comp, pts, m, cfg_begin=0, cfg_count=None):
    """fp64 (cost [C * n_seg], twist [C * n_seg, S, 6], sum|cost term|, sum|twist term|) from the fp32 per-pair
    query(..., return_which=True) outputs."""
    S = len(comp.sdfs)
    m = float(np.float32(m))                       # the margin every route computes with
    n_cfg = 1 if comp.tsf_batch is None else int(np.prod(comp.tsf_batch))
    C = n_cfg - cfg_begin if cfg_count is None else cfg_count
    L = pts.shape[-2]
    p = pts.reshape(-1, L, 3).double()
    n_seg = p.shape[0]
    cost = torch.zeros(C, n_seg, dtype=torch.float64, device="cuda")
    twist = torch.zeros(C, n_seg, S, 6, dtype=torch.float64, device="cuda")
    abs_tw = torch.zeros_like(twist)
    for c0 in range(0, C, 32):
        cc = min(32, C - c0)
        v, g, w = comp.query(pts.reshape(-1, 3), cfg_begin + c0, cc, return_which=True)
        v, g, w = v.reshape(cc, n_seg, L).double(), g.reshape(cc, n_seg, L, 3).double(), w.reshape(cc, n_seg, L)
        h = (m - v).clamp_min(0.0)
        cost[c0:c0 + cc] = (h * h).sum(-1)
        terms = torch.cat([g, torch.linalg.cross(p.expand_as(g), g, dim=-1)], -1) * (2 * h)[..., None]
        for s in range(S):
            mask = (w == s)[..., None]
            twist[c0:c0 + cc, :, s] = (terms * mask).sum(-2)
            abs_tw[c0:c0 + cc, :, s] = (terms.abs() * mask).sum(-2)
    return cost.reshape(-1), twist.reshape(-1, S, 6), cost.reshape(-1), abs_tw.reshape(-1, S, 6)


def _assert_close(got, ref, what):
    cost, twist = got
    rc, rt, ac, at = ref
    ec = (cost.double() - rc).abs() - 1e-5 * ac
    et = (twist.double() - rt).abs() - 1e-5 * at
    assert float(ec.max()) <= 1e-30, (what, "cost", float((cost.double() - rc).abs().max()))
    assert float(et.max()) <= 1e-30, (what, "twist", float((twist.double() - rt).abs().max()))


def _check(comp, pts, m, cfg_begin=0, cfg_count=None, what=""):
    got = comp.query_collision_cost(pts, m, cfg_begin, cfg_count)
    _assert_close(got, _reference(comp, pts, m, cfg_begin, cfg_count), what)
    again = comp.query_collision_cost(pts, m, cfg_begin, cfg_count)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1]), (what, "repeat")
    return got


def _margins(comp, pts):
    v = comp.query(pts.reshape(-1, 3))[0]
    return [float(torch.quantile(v[:1 << 20].float(), 0.02)), float(torch.quantile(v[:1 << 20].float(), 0.25))]


def test_golden_sets_fused(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    q = torch.from_numpy(z["q"]).cuda()
    prim = [pv.BoxSDF([0.05, 0.03, 0.04]), pv.CylinderSDF(0.015, 0.06), pv.SphereSDF(0.02), pv.BoxSDF([0.02, 0.02, 0.08])]
    for name, sdfs in list(sets.items()) + [("primitive", prim)]:
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        _no_composition(monkeypatch, comp)
        for m in _margins(comp, q):
            assert float(_check(comp, q, m, what=(name, m))[0].sum()) > 0, name
            _check(comp, q.reshape(6, 500, 3), m, cfg_begin=1, cfg_count=2, what=(name, m, "slab"))


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_arm_fused(tmp_path, monkeypatch, kind):
    s = arm_robot(tmp_path, kind)
    s.set_joint_configuration(workloads.arm_configurations(300).cuda())
    _no_composition(monkeypatch, s.sdf)
    pts = arm_points(8000, seed=41)
    for m in (0.02, 0.1):
        full = _check(s.sdf, pts, m, what=(kind, m))
        assert float(full[0].sum()) > 0 and bool(full[1].any()), (kind, m)
        _check(s.sdf, pts.reshape(4, 2000, 3), m, what=(kind, m, "4 segments"))
        # slabs: the rows of the full call, bit for bit
        for begin, count in ((0, 1), (3, 200), (31, 2), (33, 40), (299, 1)):
            c, t = s.sdf.query_collision_cost(pts, m, begin, count)
            assert torch.equal(c, full[0][begin:begin + count]) and torch.equal(t, full[1][begin:begin + count]), \
                (kind, m, begin, count)
    # margins <= 0: penetration only
    for m in (0.0, -0.01):
        v = s.sdf.query(pts)[0]
        if bool((v < m).any()):
            _check(s.sdf, pts, m, what=(kind, m))
        else:
            c, t = s.sdf.query_collision_cost(pts, m)
            assert not c.any() and not t.any()
    # a cloud beyond every link's bound: exactly 0
    far = pts + 100.0
    c, t = s.sdf.query_collision_cost(far, 0.1)
    assert not c.any() and not t.any()


def test_composition_route(tmp_path):
    """Meshes, a LOOKUP_GT_SDF grid, 12 grid links and sub-SDFs without descriptors."""
    import pytorch_volumetric_b200 as pv
    drill = pv_factory("drill")
    A, P = 40, 3000
    pts = (torch.rand(P, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda() * 0.15
    tm = torch.eye(4).repeat(2 * A, 1, 1)
    tm[:, :3, 3] = 0.05 * torch.randn(2 * A, 3, generator=torch.Generator().manual_seed(2))
    comp = pv.ComposedSDF([pv.MeshSDF(drill), pv.MeshSDF(drill)], pv.Transform3d(matrix=tm.cuda()))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
    for m in _margins(comp, pts):
        _check(comp, pts, m, what=("mesh", m))
        _check(comp, pts.reshape(6, 500, 3), m, 7, 20, what=("mesh slab", m))
    z, sets = golden_sets(tmp_path)
    near = sets["nearest"][0]
    zc = golden("ref_cachedsdf_probe")
    gt = cached_from_golden(zc, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    q = torch.from_numpy(z["q"]).cuda()
    for name, sdfs in (("12 links", [near] * 12), ("lookup-gt", [near, gt, near])):
        tm = workloads.random_rigid(len(sdfs) * A, seed=4, t_range=0.03).cuda()
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        for m in _margins(comp, q):
            _check(comp, q, m, what=(name, m))
            _check(comp, q.reshape(10, 300, 3), m, 5, 33, what=(name, m, "slab"))
    s = cached_arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(150).cuda())
    opaque = pv.ComposedSDF(opaque_sdfs(pv, s.sdf.sdfs), s.sdf.obj_frame_to_link_frame)
    apts = arm_points(2000, seed=23)
    _check(opaque, apts, 0.05, what="opaque")
    _check(opaque, apts.reshape(4, 500, 3), 0.05, 10, 100, what="opaque slab")


def test_shapes(tmp_path):
    s = cached_arm(tmp_path, "nearest")
    pts = arm_points(3000, seed=24)
    S, J = len(s.sdf_to_link_name), len(s.joint_names)
    # no configuration batch: [*B]
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    c, t = s.sdf.collision_cost(pts.reshape(3, 1000, 3), 0.1)
    assert c.shape == (3,) and t.shape == (3, S, 6)
    c, g = s.collision_cost(pts.reshape(3, 1000, 3), 0.1)
    assert c.shape == (3,) and g.shape == (3, J)
    # a 2-D configuration batch and a 2-D segment batch
    s.set_joint_configuration(workloads.arm_configurations(24).cuda().reshape(4, 6, -1))
    bp = pts.reshape(2, 3, 500, 3)
    c, t = s.sdf.collision_cost(bp, 0.1)
    assert c.shape == (4, 6, 2, 3) and t.shape == (4, 6, 2, 3, S, 6)
    rc, rt = s.sdf.query_collision_cost(bp, 0.1)
    assert torch.equal(c.reshape(-1), rc) and torch.equal(t.reshape(-1, S, 6), rt)
    c, g = s.collision_cost(bp, 0.1)
    assert c.shape == (4, 6, 2, 3) and g.shape == (4, 6, 2, 3, J)
    # host in, host out; fp64 in, fp64 out
    ch, gh = s.collision_cost(bp.cpu().double(), 0.1)
    assert ch.device.type == "cpu" and ch.dtype == torch.float64 and gh.dtype == torch.float64
    assert torch.equal(ch, c.cpu().double())
    # N = 0 costs 0; no segments give empty results
    c0, t0 = s.sdf.collision_cost(torch.empty(5, 0, 3, device="cuda"), 0.1)
    assert c0.shape == (4, 6, 5) and t0.shape == (4, 6, 5, S, 6) and not c0.any() and not t0.any()
    c0, g0 = s.collision_cost(torch.empty(0, 7, 3, device="cuda"), 0.1)
    assert c0.shape == (4, 6, 0) and g0.shape == (4, 6, 0, J)


def test_joint_gradient_on_a_general_chain_vs_fp64_finite_differences(tmp_path):
    """The mixed primitive chain of test_gpu_robot_fp64.py: over points whose argmin link and shape rule stay put,
    RobotSDF.collision_cost's joint gradient against central differences of the fp64 cost."""
    robot, ref, text = build_robot("mixed", tmp_path)
    J, S = len(robot.joint_names), len(ref.links)
    A = 6
    qs = joint_values(ref, text, A, seed=9)
    robot.set_joint_configuration(torch.from_numpy(qs).cuda())
    rng = np.random.default_rng(5)
    cloud = rng.uniform(-0.45, 0.45, (20000, 3)) + np.array([0.0, 0.0, 0.45])
    m, h = 0.06, 2.0 ** -16
    per = ref.evaluate(ref.object_to_link(qs), cloud)
    v, g, w = ref.compose(per)
    second = np.sort(per["value"], axis=0)[1]
    gap = np.take_along_axis(per["gap"], w[None], 0)[0]
    cond = np.take_along_axis(per["cond"], w[None], 0)[0]
    for a in range(A):
        stable = (gap[a] > 1e-3) & (second[a] - v[a] > 1e-3) & (cond[a] > 5e-2) & (np.abs(v[a] - m) > 1e-3)
        pts = cloud[stable & (v[a] < m)]
        robot.set_joint_configuration(torch.from_numpy(qs[a:a + 1]).cuda())
        cost, grad = robot.collision_cost(torch.from_numpy(pts.astype(np.float32)).cuda(), m)
        grad = grad.double().cpu().numpy().reshape(-1)
        p32 = pts.astype(np.float32).astype(np.float64)
        twists = robot.joint_twists().cpu().numpy()[0]
        for j in range(J):
            qp, qm = qs[a:a + 1].astype(np.float64), qs[a:a + 1].astype(np.float64)
            qp[0, j] += h
            qm[0, j] -= h
            cp = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qp), p32))[0][0], 0) ** 2
            cm = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qm), p32))[0][0], 0) ** 2
            fd = (cp.sum() - cm.sum()) / (2 * h)
            hinge = np.maximum(m - v[a][stable & (v[a] < m)], 0)
            scale = (2 * hinge * (np.linalg.norm(twists[j, :3]) + np.linalg.norm(pts, axis=1) *
                                  np.linalg.norm(twists[j, 3:]))).sum()
            assert abs(grad[j] - fd) <= 5e-4 * scale + 1e-9, (a, j, grad[j], fd, scale)


def test_joint_gradient_on_the_cached_arm_vs_fp64_jacobian(tmp_path):
    """The cached 8-link arm: the joint gradient against the fp64 Jacobian transpose of the fp32 per-pair outputs,
    through the fp64 joint twists of the same configurations."""
    s = cached_arm(tmp_path, "nearest")
    A = 100
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    pts = arm_points(20000, seed=42).reshape(2, 10000, 3)
    m = 0.05
    cost, grad = s.collision_cost(pts, m)
    rc, rt, ac, at = _reference(s.sdf, pts, m)
    jt = s.joint_twists()
    moves = s.joint_moves_link()
    ref = s.joint_gradient(rt.reshape(A, 2, -1, 6), jt, moves)
    bound = s.joint_gradient(at.reshape(A, 2, -1, 6), jt.abs(), moves)
    assert cost.shape == (A, 2) and grad.shape == (A, 2, len(s.joint_names))
    assert float(((grad.double() - ref).abs() - 1e-5 * bound).max()) <= 1e-12
    assert float(((cost.double() - rc.reshape(A, 2)).abs() - 1e-5 * ac.reshape(A, 2)).max()) <= 1e-30
    assert float(ref.abs().max()) > 0
