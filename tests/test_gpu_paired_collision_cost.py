"""GPU: paired collision-cost queries (ComposedSDF.paired_collision_cost / query_paired_collision_cost,
RobotSDF.paired_collision_cost, pvb_composed_query_paired_collision_cost).

Every configuration against its own cloud: for every segment of its points, the hinge cost and the twist gradient
per sub-SDF; for a robot the joint gradient.  On the fused sets, row (a, b) is compared bit for bit with
query_collision_cost(points[a], m, a, 1)[b] -- the definition -- and with the rows of slab calls and repeated calls;
every route is compared with the fp64 sum of the fp32 query_paired(..., return_which=True) outputs within
1e-5 * sum|term|."""
import numpy as np
import pytest
import torch

import workloads
from helpers import (arm_points, arm_robot, cached_arm, cached_from_golden, golden, golden_sets, opaque_sdfs,
                     own_points, pv_factory)
from robot_ref import build_robot, joint_values

pytestmark = pytest.mark.gpu

MARGINS = (0.02, 0.1, 0.0, -0.01)


def _no_composition(monkeypatch, comp):
    def boom(*a, **k):
        raise AssertionError("composition route taken")
    monkeypatch.setattr(comp, "_composed_collision_cost", boom)
    monkeypatch.setattr(comp, "_generic_query", boom)


def _reference(comp, own, m, cfg_begin=0):
    """own [C, *B, N, 3]: fp64 (cost [C * n_seg], twist [C * n_seg, S, 6], sum|cost term|, sum|twist term|) from the
    fp32 query_paired(..., return_which=True) outputs at each configuration's own points."""
    S = len(comp.sdfs)
    m = float(np.float32(m))                       # the margin every route computes with
    C, L = own.shape[0], own.shape[-2]
    p = own.reshape(C, -1, L, 3)
    n_seg = p.shape[1]
    cost = torch.zeros(C, n_seg, dtype=torch.float64, device="cuda")
    twist = torch.zeros(C, n_seg, S, 6, dtype=torch.float64, device="cuda")
    abs_tw = torch.zeros_like(twist)
    for c0 in range(0, C, 32):
        cc = min(32, C - c0)
        v, g, w = comp.query_paired(p[c0:c0 + cc], cfg_begin + c0, cc, return_which=True)
        v, g, w = v.reshape(cc, n_seg, L).double(), g.reshape(cc, n_seg, L, 3).double(), w.reshape(cc, n_seg, L)
        h = (m - v).clamp_min(0.0)
        cost[c0:c0 + cc] = (h * h).sum(-1)
        terms = torch.cat([g, torch.linalg.cross(p[c0:c0 + cc].double(), g, dim=-1)], -1) * (2 * h)[..., None]
        for s in range(S):
            mask = (w == s)[..., None]
            twist[c0:c0 + cc, :, s] = (terms * mask).sum(-2)
            abs_tw[c0:c0 + cc, :, s] = (terms.abs() * mask).sum(-2)
    return cost.reshape(-1), twist.reshape(-1, S, 6), cost.reshape(-1), abs_tw.reshape(-1, S, 6)


def _assert_close(got, ref, what):
    cost, twist = got
    rc, rt, ac, at = ref
    assert float(((cost.double() - rc).abs() - 1e-5 * ac).max()) <= 1e-30, \
        (what, "cost", float((cost.double() - rc).abs().max()))
    assert float(((twist.double() - rt).abs() - 1e-5 * at).max()) <= 1e-30, \
        (what, "twist", float((twist.double() - rt).abs().max()))


def _check(comp, own, m, cfg_begin=0, what=""):
    """The slab call over own [C, *B, N, 3]: within the fp64 bound, and repeated bit for bit."""
    got = comp.query_paired_collision_cost(own, m, cfg_begin, own.shape[0])
    _assert_close(got, _reference(comp, own, m, cfg_begin), what)
    again = comp.query_paired_collision_cost(own, m, cfg_begin, own.shape[0])
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1]), (what, "repeat")
    return got


def _assert_single_rows(comp, own, m, got, configs, cfg_begin=0, what=""):
    """Row c * n_seg + b == query_collision_cost(own[c], m, cfg_begin + c, 1)[b], bit for bit."""
    n_seg = len(got[0]) // own.shape[0]
    for c in configs:
        c1, t1 = comp.query_collision_cost(own[c], m, cfg_begin + int(c), 1)
        rows = slice(int(c) * n_seg, (int(c) + 1) * n_seg)
        assert torch.equal(got[0][rows], c1) and torch.equal(got[1][rows], t1), (what, int(c))


def _sample(A, n, seed):
    """At least n configurations of A: 0, 31, 32, the last, and random others."""
    rest = torch.randperm(A, generator=torch.Generator().manual_seed(seed))[:n].tolist()
    return sorted({0, 31, 32, A - 1, *rest} & set(range(A)))


def test_golden_sets_fused(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    own = own_points(torch.from_numpy(z["q"]), A, 5)
    prim = [pv.BoxSDF([0.05, 0.03, 0.04]), pv.CylinderSDF(0.015, 0.06), pv.SphereSDF(0.02), pv.BoxSDF([0.02, 0.02, 0.08])]
    for name, sdfs in (("nearest", sets["nearest"]), ("trilinear", sets["trilinear"]), ("primitive", prim)):
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        _no_composition(monkeypatch, comp)
        for m in MARGINS:
            got = _check(comp, own, m, what=(name, m))
            _assert_single_rows(comp, own, m, got, range(A), what=(name, m))
            seg = own.reshape(A, 6, 500, 3)
            got = _check(comp, seg, m, what=(name, m, "6 segments"))
            _assert_single_rows(comp, seg, m, got, range(A), what=(name, m, "6 segments"))
            sub = _check(comp, seg[1:3], m, cfg_begin=1, what=(name, m, "slab"))
            assert torch.equal(sub[0], got[0][6:18]) and torch.equal(sub[1], got[1][6:18]), (name, m, "slab")
        assert float(comp.query_paired_collision_cost(own, 0.1)[0].sum()) > 0, name


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_arm_fused(tmp_path, monkeypatch, kind):
    s = arm_robot(tmp_path, kind)
    A = 300
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    _no_composition(monkeypatch, s.sdf)
    own = arm_points(A * 1200, seed=51).reshape(A, 1200, 3)          # 3 chunks of 512 points, the last partial
    sample = _sample(A, 40, seed=52)
    assert len(sample) >= 40
    for m in MARGINS:
        full = _check(s.sdf, own, m, what=(kind, m))
        _assert_single_rows(s.sdf, own, m, full, sample, what=(kind, m))
        if m > 0:
            assert float(full[0].sum()) > 0 and bool(full[1].any()), (kind, m)
        # slabs: the rows of the full call, bit for bit
        for begin, count in ((0, 1), (3, 200), (31, 2), (33, 40), (299, 1)):
            c, t = s.sdf.query_paired_collision_cost(own[begin:begin + count], m, begin, count)
            assert torch.equal(c, full[0][begin:begin + count]) and torch.equal(t, full[1][begin:begin + count]), \
                (kind, m, begin, count)
        # segments of 33 and 1 points
        seg = own[:, :1188].reshape(A, 36, 33, 3)
        got = _check(s.sdf, seg, m, what=(kind, m, "N=33"))
        _assert_single_rows(s.sdf, seg, m, got, sample[:10], what=(kind, m, "N=33"))
        got = s.sdf.query_paired_collision_cost(own[:50].reshape(50, 1200, 1, 3), m, 0, 50)
        _assert_single_rows(s.sdf, own[:50].reshape(50, 1200, 1, 3), m, got, (0, 31, 49), what=(kind, m, "N=1"))
    # clouds beyond every link's bound: exactly 0
    c, t = s.sdf.query_paired_collision_cost(own + 100.0, 0.1)
    assert not c.any() and not t.any()


def test_composition_route(tmp_path):
    """Meshes, a LOOKUP_GT_SDF grid, 12 grid links and sub-SDFs without descriptors: within the fp64 bound of the
    same per-pair outputs."""
    import pytorch_volumetric_b200 as pv
    drill = pv_factory("drill")
    A, P = 40, 3000
    own = (torch.rand(A, P, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda() * 0.15
    tm = torch.eye(4).repeat(2 * A, 1, 1)
    tm[:, :3, 3] = 0.05 * torch.randn(2 * A, 3, generator=torch.Generator().manual_seed(2))
    comp = pv.ComposedSDF([pv.MeshSDF(drill), pv.MeshSDF(drill)], pv.Transform3d(matrix=tm.cuda()))
    comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
    for m in (0.02, 0.1):
        assert float(_check(comp, own, m, what=("mesh", m))[0].sum()) > 0
        _check(comp, own[7:27].reshape(20, 6, 500, 3), m, 7, what=("mesh slab", m))
    z, sets = golden_sets(tmp_path)
    near = sets["nearest"][0]
    zc = golden("ref_cachedsdf_probe")
    gt = cached_from_golden(zc, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    gown = own_points(torch.from_numpy(z["q"]), A, 1)
    for name, sdfs in (("12 links", [near] * 12), ("lookup-gt", [near, gt, near])):
        tm = workloads.random_rigid(len(sdfs) * A, seed=4, t_range=0.03).cuda()
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        for m in (0.02, 0.1):
            _check(comp, gown, m, what=(name, m))
            _check(comp, gown[5:38].reshape(33, 10, 300, 3), m, 5, what=(name, m, "slab"))
    s = cached_arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(150).cuda())
    opaque = pv.ComposedSDF(opaque_sdfs(pv, s.sdf.sdfs), s.sdf.obj_frame_to_link_frame)
    apts = arm_points(150 * 400, seed=53).reshape(150, 400, 3)
    _check(opaque, apts, 0.05, what="opaque")
    _check(opaque, apts[10:110].reshape(100, 4, 100, 3), 0.05, 10, what="opaque slab")


def test_shapes(tmp_path):
    s = cached_arm(tmp_path, "nearest")
    pts = arm_points(24 * 6 * 500, seed=54)
    S, J = len(s.sdf_to_link_name), len(s.joint_names)
    # no configuration batch: collision_cost
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    one = pts[:1500].reshape(3, 500, 3)
    for a, b in zip(s.sdf.paired_collision_cost(one, 0.1), s.sdf.collision_cost(one, 0.1)):
        assert torch.equal(a, b)
    for a, b in zip(s.paired_collision_cost(one, 0.1), s.collision_cost(one, 0.1)):
        assert torch.equal(a, b)
    # a 2-D configuration batch and a 2-D segment batch
    s.set_joint_configuration(workloads.arm_configurations(24).cuda().reshape(4, 6, -1))
    own = pts.reshape(4, 6, 2, 3, 500, 3)
    c, t = s.sdf.paired_collision_cost(own, 0.1)
    assert c.shape == (4, 6, 2, 3) and t.shape == (4, 6, 2, 3, S, 6)
    rc, rt = s.sdf.query_paired_collision_cost(own, 0.1)
    assert torch.equal(c.reshape(-1), rc) and torch.equal(t.reshape(-1, S, 6), rt)
    _assert_single_rows(s.sdf, own.reshape(24, 2, 3, 500, 3), 0.1, (rc, rt), (0, 7, 23), what="2-D batch")
    cr, g = s.paired_collision_cost(own, 0.1)
    assert torch.equal(cr, c) and g.shape == (4, 6, 2, 3, J)
    # host in, host out; fp64 in, fp64 out
    ch, gh = s.paired_collision_cost(own.cpu(), 0.1)
    assert ch.device.type == "cpu" and ch.dtype == torch.float32 and torch.equal(ch, c.cpu())
    c64, g64 = s.paired_collision_cost(own.cpu().double(), 0.1)
    assert c64.dtype == torch.float64 and g64.dtype == torch.float64 and torch.equal(c64, c.cpu().double())
    # N = 0 costs 0; no segments give empty results
    c0, t0 = s.sdf.paired_collision_cost(torch.empty(4, 6, 5, 0, 3, device="cuda"), 0.1)
    assert c0.shape == (4, 6, 5) and t0.shape == (4, 6, 5, S, 6) and not c0.any() and not t0.any()
    c0, g0 = s.paired_collision_cost(torch.empty(4, 6, 0, 7, 3, device="cuda"), 0.1)
    assert c0.shape == (4, 6, 0) and g0.shape == (4, 6, 0, J)
    # the configuration batch must lead
    with pytest.raises(ValueError, match="leading"):
        s.paired_collision_cost(own.reshape(6, 4, 2, 3, 500, 3), 0.1)
    with pytest.raises(ValueError, match="leading"):
        s.sdf.paired_collision_cost(own.reshape(24, 6, 500, 3), 0.1)


def test_seventy_thousand_configurations(tmp_path, monkeypatch):
    """70 000 configurations x 64 points: more than 65 535 configuration tiles, on the fused route."""
    s = cached_arm(tmp_path, "nearest")
    A = 70_000
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    _no_composition(monkeypatch, s.sdf)
    own = arm_points(A * 64, seed=55).reshape(A, 64, 3)
    got = s.sdf.query_paired_collision_cost(own, 0.1)
    assert float(got[0].sum()) > 0
    _assert_single_rows(s.sdf, own, 0.1, got, (0, 31, 32, 65_535, 65_536, 69_000, A - 1), what="70000")
    sub = s.sdf.query_paired_collision_cost(own[65_000:], 0.1, 65_000, A - 65_000)
    assert torch.equal(sub[0], got[0][65_000:]) and torch.equal(sub[1], got[1][65_000:])


def test_past_2_31_points(tmp_path, monkeypatch):
    """36 000 configurations x 60 000 own points (2.16e9 points, 26 GB): sampled rows, some past point 2^31, equal
    their single-configuration rows."""
    A, N = 36_000, 60_000
    need = A * N * 12 + A * 118 * 49 * 4 + (2 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GB of free device memory, {free / 2 ** 30:.1f} GB free")
    s = arm_robot(tmp_path, "primitive")
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    _no_composition(monkeypatch, s.sdf)
    own = torch.empty(A, N, 3, device="cuda")
    own.uniform_(generator=torch.Generator(device="cuda").manual_seed(56))
    lo = torch.tensor([r[0] for r in workloads.ARM_QUERY_RANGE], device="cuda")
    hi = torch.tensor([r[1] for r in workloads.ARM_QUERY_RANGE], device="cuda")
    own.mul_(hi - lo).add_(lo)
    got = s.sdf.query_paired_collision_cost(own, 0.1)
    first = (2 ** 31) // N + 1                        # the first configuration whose points start past 2^31
    _assert_single_rows(s.sdf, own, 0.1, got, (0, 1, first - 1, first, first + 1, A - 1), what="2^31")
    assert float(got[0][first:].sum()) > 0
    del own, got
    torch.cuda.empty_cache()


def test_joint_gradient_is_the_twist_through_joint_gradient(tmp_path):
    s = cached_arm(tmp_path, "trilinear")
    A = 64
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    own = arm_points(A * 2 * 800, seed=57).reshape(A, 2, 800, 3)
    cost, grad = s.paired_collision_cost(own, 0.05)
    c, t = s.sdf.paired_collision_cost(own, 0.05)
    ref = s.joint_gradient(t, s.joint_twists(), s.joint_moves_link())
    assert torch.equal(cost, c) and torch.equal(grad, ref.float()) and grad.shape == (A, 2, len(s.joint_names))
    assert float(grad.abs().max()) > 0


def test_joint_gradient_on_a_general_chain_vs_fp64_finite_differences(tmp_path):
    """The mixed primitive chain of test_gpu_robot_fp64.py, every configuration with its own cloud: over points whose
    argmin link and shape rule stay put, RobotSDF.paired_collision_cost's joint gradient against central differences
    of the fp64 cost."""
    robot, ref, text = build_robot("mixed", tmp_path)
    J = len(robot.joint_names)
    A = 6
    qs = joint_values(ref, text, A, seed=9)
    rng = np.random.default_rng(6)
    cloud = rng.uniform(-0.45, 0.45, (20000, 3)) + np.array([0.0, 0.0, 0.45])
    cloud = cloud.astype(np.float32).astype(np.float64)
    m, h = 0.06, 2.0 ** -16
    per = ref.evaluate(ref.object_to_link(qs), cloud)
    v, g, w = ref.compose(per)
    second = np.sort(per["value"], axis=0)[1]
    gap = np.take_along_axis(per["gap"], w[None], 0)[0]
    cond = np.take_along_axis(per["cond"], w[None], 0)[0]
    keep = [np.flatnonzero((gap[a] > 1e-3) & (second[a] - v[a] > 1e-3) & (cond[a] > 5e-2) &
                           (np.abs(v[a] - m) > 1e-3) & (v[a] < m)) for a in range(A)]
    K = min(len(k) for k in keep)
    assert K >= 10
    own = np.stack([cloud[keep[a][rng.permutation(len(keep[a]))[:K]]] for a in range(A)])   # [A, K, 3]
    robot.set_joint_configuration(torch.from_numpy(qs).cuda())
    cost, grad = robot.paired_collision_cost(torch.from_numpy(own.astype(np.float32)).cuda(), m)
    grad = grad.double().cpu().numpy()
    twists = robot.joint_twists().cpu().numpy()
    assert cost.shape == (A,) and grad.shape == (A, J)
    for a in range(A):
        va = ref.compose(ref.evaluate(ref.object_to_link(qs[a:a + 1]), own[a]))[0][0]
        for j in range(J):
            qp, qm = qs[a:a + 1].astype(np.float64), qs[a:a + 1].astype(np.float64)
            qp[0, j] += h
            qm[0, j] -= h
            cp = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qp), own[a]))[0][0], 0) ** 2
            cm = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qm), own[a]))[0][0], 0) ** 2
            fd = (cp.sum() - cm.sum()) / (2 * h)
            hinge = np.maximum(m - va, 0)
            scale = (2 * hinge * (np.linalg.norm(twists[a, j, :3]) + np.linalg.norm(own[a], axis=1) *
                                  np.linalg.norm(twists[a, j, 3:]))).sum()
            assert abs(grad[a, j] - fd) <= 5e-4 * scale + 1e-9, (a, j, grad[a, j], fd, scale)
