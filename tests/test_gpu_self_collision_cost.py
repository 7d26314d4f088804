"""GPU: self-collision-cost queries (ComposedSDF.self_collision_cost / query_self_collision_cost,
RobotSDF.self_collision_cost, pvb_composed_query_self_collision_cost).

For every configuration, cost = sum over (source i, point k) with d < m of (m - d)^2 and the twist gradient per
sub-SDF (+tau to the target j, -tau to the source i); for a robot the joint gradient.
1. The fused route against the composition route (`_composed_self_collision_cost`, the definition) and against the
   fp64 sum of the fp32 per-point query_paired outputs, within 1e-5 * sum|term| per entry for cost, twist and joint
   gradient, on the nearest, trilinear and primitive arms, both margins, 200 and 70 000 configurations -- each route
   checked to have run.  Repeated calls and slabs are bit-identical.
2. Against self_clearance: cost and twists are exactly 0 when the clearance is >= m, and cost > 0 below m - 1e-6.
3. Rigid motions: without the base link's pairs, the first joint moves every remaining link and its derivative is 0;
   the twists of a configuration sum to 0 over the sub-SDFs.
4. The joint gradient on the mixed primitive chain against fp64 central differences.
5. The composition route on meshes, 12 links and opaque sub-SDFs against the fp64 restatement.
6. Shapes: a [3, 20] batch, no batch, a float64 chain, K = 1 and a configuration without allowed pairs."""
import math

import numpy as np
import pytest
import torch

import robot_ref as rr
import workloads
from helpers import allowed_matrix, arm_robot, opaque_sdfs, surface_points, wide_configurations
from robot_ref import build_robot, joint_values

pytestmark = pytest.mark.gpu


def _reference(comp, lp, allowed, m, cfg_begin=0, cfg_count=None, chunk=8192):
    """fp64 (cost [C], twist [C, S, 6], sum|cost term| [C], sum|twist term| [C, S, 6]) of the definition from the fp32
    per-point outputs: per source, its points posed by pvb_transform_points_paired (the library's own posing) and
    query_paired(..., return_which=True) of its allowed sub-composition."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import _native as nat
    S = len(comp.sdfs)
    n_cfg = 1 if comp.tsf_batch is None else math.prod(comp.tsf_batch)
    C = n_cfg - cfg_begin if cfg_count is None else cfg_count
    m = float(np.float32(m))
    dev = torch.device("cuda", torch.cuda.current_device())
    xf = comp._xforms_on(dev).reshape(S, n_cfg, 4, 4)
    inv = comp._inv_xforms_on(dev).reshape(S, n_cfg, 4, 4)
    lp = lp.detach().to(device=dev, dtype=torch.float32)
    K = lp.shape[1]
    al = torch.as_tensor(allowed).cpu().clone()
    al.fill_diagonal_(False)
    cost = torch.zeros(C, dtype=torch.float64, device=dev)
    twist = torch.zeros(C, S, 6, dtype=torch.float64, device=dev)
    abs_tw = torch.zeros_like(twist)
    for i in range(S):
        js = [j for j in range(S) if al[i, j]]
        if not js:
            continue
        sub = pv.ComposedSDF([comp.sdfs[j] for j in js], None)
        sub.set_transforms(pv.Transform3d(matrix=xf[js].reshape(-1, 4, 4)), batch_dim=(n_cfg,))
        jt = torch.tensor(js, device=dev)
        for c0 in range(cfg_begin, cfg_begin + C, chunk):
            cc = min(chunk, cfg_begin + C - c0)
            w_i = inv[i, c0:c0 + cc].contiguous()
            own = lp[i].expand(cc, K, 3).contiguous()
            x = torch.empty(cc, K, 3, device=dev)
            nat.check(nat.lib().pvb_transform_points_paired(nat.ptr(w_i), cc, nat.ptr(own), K, nat.ptr(x),
                                                            nat.stream_ptr(dev)), "pvb_transform_points_paired")
            v, g, w = sub.query_paired(x, cfg_begin=c0, cfg_count=cc, return_which=True)
            v, g, w = v.reshape(cc, K).double(), g.reshape(cc, K, 3).double(), jt[w.long()].reshape(cc, K)
            h = (m - v).clamp_min(0.0)
            tau = torch.cat([g, torch.linalg.cross(x.double(), g, dim=-1)], -1) * (2 * h)[..., None]
            r = slice(c0 - cfg_begin, c0 - cfg_begin + cc)
            cost[r] += (h * h).sum(-1)
            for j in js:
                mask = (w == j)[..., None]
                twist[r, j] += (tau * mask).sum(-2)
                abs_tw[r, j] += (tau.abs() * mask).sum(-2)
            twist[r, i] -= tau.sum(-2)
            abs_tw[r, i] += tau.abs().sum(-2)
    return cost, twist, cost, abs_tw


def _assert_close(got, ref, what, rel=1e-5):
    cost, twist = got
    rc, rt, ac, at = ref
    assert float(((cost.double() - rc).abs() - rel * ac).max()) <= 1e-30, \
        (what, "cost", float((cost.double() - rc).abs().max()))
    assert float(((twist.double() - rt).abs() - rel * at).max()) <= 1e-30, \
        (what, "twist", float((twist.double() - rt).abs().max()))


def _routes(monkeypatch, comp, lp, allowed, m, cfg_begin=0, cfg_count=None):
    """(fused result, composition-route result), after checking which route each call took."""
    from pytorch_volumetric_b200 import sdf as S
    calls = []
    orig = S.ComposedSDF._composed_self_collision_cost

    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(S.ComposedSDF, "_composed_self_collision_cost", spy)
    fused = comp.query_self_collision_cost(lp, allowed, m, cfg_begin=cfg_begin, cfg_count=cfg_count)
    assert not calls, "the fused route fell back to the composition route"
    n_cfg = math.prod(comp.tsf_batch) if comp.tsf_batch is not None else 1
    count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    K, rows = comp._self_clearance_args(lp, allowed)
    p = lp.detach().float().reshape(-1, 3).contiguous()
    ref = comp._composed_self_collision_cost(p, K, rows, comp._collision_cost_margin(m), cfg_begin, count)
    assert calls
    return fused, ref


def _check_arm(monkeypatch, robot, lp, allowed, m, what):
    """Fused against the composition route and the fp64 sum (cost, twist, joint gradient), repeat and the relation
    with self_clearance; returns the fused result and the reference."""
    fused, comp = _routes(monkeypatch, robot.sdf, lp, allowed, m)
    ref = _reference(robot.sdf, lp, allowed, m)
    _assert_close(fused, ref, (what, "fused"))
    _assert_close(comp, ref, (what, "composition"))
    again = robot.sdf.query_self_collision_cost(lp, allowed, m)
    assert torch.equal(again[0], fused[0]) and torch.equal(again[1], fused[1]), (what, "repeat")
    # the joint gradient: within 1e-5 of its bound through the fp64 joint twists
    jt, moves = robot.joint_twists(), robot.joint_moves_link()
    A = fused[0].shape[0]
    grad = robot.joint_gradient(fused[1], jt, moves)
    gref = robot.joint_gradient(ref[1], jt, moves)
    bound = robot.joint_gradient(ref[3], jt.abs(), moves)
    assert grad.shape == (A, len(robot.joint_names))
    assert float(((grad - gref).abs() - 1e-5 * bound).max()) <= 1e-12, (what, "joint gradient")
    # exactly 0 at and above the margin, > 0 clearly below it
    clr = robot.sdf.query_self_clearance(lp, allowed)[0]
    m32 = float(np.float32(m))
    far = clr >= m32
    assert not fused[0][far].any() and not fused[1][far].any(), what
    assert (fused[0][clr < m32 - 1e-6] > 0).all(), what
    # every term is added to its target and subtracted from its source: the twists sum to ~0 over the sub-SDFs
    assert float((fused[1].double().sum(1).abs() - 1e-5 * ref[3].sum(1)).max()) <= 1e-30, (what, "sum over s")
    return fused, ref


# ---------------------------------------------------------------- 1-3. the arm
@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_fused_equals_composition_on_the_arm(tmp_path, monkeypatch, kind):
    robot = arm_robot(tmp_path, kind)
    S = len(robot.sdf.sdfs)
    A, K = 200, 1024
    # half the configurations wide (links pass through one another), half about the nominal pose (most clear)
    q = torch.cat([wide_configurations(A // 2, seed=3), workloads.arm_configurations(A // 2, seed=4)])
    robot.set_joint_configuration(q.cuda())
    lp = robot.link_surface_points(num_points=K, seed=1)
    seen_zero = False
    for m in (0.02, 0.1):
        for which in ("default", "asymmetric"):
            allowed = allowed_matrix(S, which)
            fused, ref = _check_arm(monkeypatch, robot, lp, allowed, m, (kind, m, which))
            assert (fused[0] > 0).any(), (kind, m, which)
            seen_zero |= bool((fused[0] == 0).any())
            # slabs: the rows of the full call, bit for bit
            for begin, count in ((0, 1), (17, 100), (199, 1), (50, 150)):
                c, t = robot.sdf.query_self_collision_cost(lp, allowed, m, begin, count)
                assert torch.equal(c, fused[0][begin:begin + count]) and \
                    torch.equal(t, fused[1][begin:begin + count]), (kind, m, begin, count)
        # rigid motion: without the pairs of the links the first joint does not move, that joint moves every
        # remaining pair together and its derivative is 0
        moves = robot.joint_moves_link()
        moved = moves[0]
        assert not moved.all() and moved.sum() >= 3
        allowed = allowed_matrix(S, "default") & moved[:, None] & moved[None, :]
        fused, ref = _check_arm(monkeypatch, robot, lp, allowed, m, (kind, m, "rigid"))
        assert (fused[0] > 0).any()
        seen_zero |= bool((fused[0] == 0).any())
        jt = robot.joint_twists()
        grad = robot.joint_gradient(fused[1], jt, moves)[:, 0]
        bound = robot.joint_gradient(ref[3], jt.abs(), moves)[:, 0]
        assert float((grad.abs() - 1e-5 * bound).max()) <= 1e-12, (kind, m)
    assert seen_zero, kind                                        # configurations clear of the margin cost exactly 0


def test_fused_equals_composition_at_70000_configurations(tmp_path, monkeypatch):
    for kind in ("nearest", "primitive"):
        robot = arm_robot(tmp_path / kind, kind)
        robot.sdf.composition_chunk = 8192                        # fewer launches for the composition route
        robot.set_joint_configuration(wide_configurations(70_000, seed=5).cuda())
        lp = robot.link_surface_points(num_points=32, seed=1)
        allowed = robot.self_collision_pairs()
        for m in (0.02, 0.1):
            fused, ref = _check_arm(monkeypatch, robot, lp, allowed, m, (kind, "70000", m))
            assert (fused[0] > 0).any()
            for begin, count in ((65_530, 4_470), (69_999, 1), (0, 65_537)):
                c, t = robot.sdf.query_self_collision_cost(lp, allowed, m, begin, count)
                assert torch.equal(c, fused[0][begin:begin + count]) and \
                    torch.equal(t, fused[1][begin:begin + count]), (kind, m, begin, count)


# ---------------------------------------------------------------- 4. the joint gradient against fp64
def _fp64_per_point(ref, q, lp, allowed):
    """fp64 per (configuration, source, point): value, robot-frame gradient, target, gap to the shape rule,
    conditioning, second-best value and the posed point; +inf for empty rows."""
    M = ref.object_to_link(q)
    W = rr.rigid_inverse(M)
    S, A = M.shape[:2]
    K = lp.shape[1]
    out = {k: np.full((A, S, K), np.inf) for k in ("v", "second", "gap", "cond")}
    out["g"], out["x"] = np.zeros((A, S, K, 3)), np.zeros((A, S, K, 3))
    out["w"] = np.full((A, S, K), -1)
    for i in range(S):
        x = np.einsum("aij,kj->aki", W[i, :, :3, :3], lp[i]) + W[i, :, None, :3, 3]
        out["x"][:, i] = x
        if not allowed[i].any():
            continue
        per = ref.evaluate(M, x)
        vals = np.where(allowed[i][:, None, None], per["value"], np.inf)          # [S, A, K]
        w = vals.argmin(0)
        take = lambda t: np.take_along_axis(t, w[None], 0)[0]
        out["v"][:, i], out["w"][:, i] = take(vals), w
        out["second"][:, i] = np.sort(vals, axis=0)[1]
        out["gap"][:, i], out["cond"][:, i] = take(per["gap"]), take(per["cond"])
        out["g"][:, i] = np.take_along_axis(per["grad"], w[None, ..., None], 0)[0]
    return out


def test_joint_gradient_on_a_general_chain_vs_fp64_finite_differences(tmp_path):
    """The mixed primitive chain of test_gpu_robot_fp64.py, one configuration at a time: link points whose target,
    shape rule and side of the margin stay put (the others moved far out of reach), RobotSDF.self_collision_cost's
    joint gradient against central differences of the fp64 cost."""
    robot, ref, text = build_robot("mixed", tmp_path)
    J, S = len(robot.joint_names), len(ref.links)
    qs = joint_values(ref, text, 6, seed=9)
    allowed = robot.self_collision_pairs().numpy().copy()
    np.fill_diagonal(allowed, False)
    lp_all = robot.link_surface_points(num_points=600, seed=3).double().cpu().numpy()
    lp_all = lp_all.astype(np.float32).astype(np.float64)
    m, h = 0.05, 2.0 ** -16
    checked = 0
    for a in range(len(qs)):
        q = qs[a:a + 1].astype(np.float64)
        per = _fp64_per_point(ref, q, lp_all, allowed)
        stable = (per["gap"][0] > 1e-3) & (per["second"][0] - per["v"][0] > 1e-3) & (per["cond"][0] > 5e-2) & \
            (np.abs(per["v"][0] - m) > 1e-3) & (per["v"][0] < m)
        n = int(stable.sum(1).max())
        if n == 0:
            continue
        # per source its stable points, padded with points 100 m away in its own frame
        lp = np.full((S, n, 3), 100.0)
        for i in range(S):
            sel = lp_all[i][stable[i]]
            lp[i, :len(sel)] = sel
        robot.set_joint_configuration(torch.from_numpy(qs[a:a + 1]).cuda())
        cost, grad = robot.self_collision_cost(m, torch.from_numpy(lp.astype(np.float32)).cuda(),
                                               torch.from_numpy(allowed))
        grad = grad.double().cpu().numpy().reshape(-1)
        twists = robot.joint_twists().cpu().numpy()[0]
        base = _fp64_per_point(ref, q, lp, allowed)
        hinge = np.maximum(m - base["v"][0], 0)
        for j in range(J):
            qp, qm = q.copy(), q.copy()
            qp[0, j] += h
            qm[0, j] -= h
            cp = (np.maximum(m - _fp64_per_point(ref, qp, lp, allowed)["v"], 0) ** 2).sum()
            cm = (np.maximum(m - _fp64_per_point(ref, qm, lp, allowed)["v"], 0) ** 2).sum()
            fd = (cp - cm) / (2 * h)
            scale = 2 * (2 * hinge * (np.linalg.norm(twists[j, :3]) + np.linalg.norm(base["x"][0], axis=-1) *
                                      np.linalg.norm(twists[j, 3:]))).sum()
            assert abs(grad[j] - fd) <= 5e-4 * scale + 1e-9, (a, j, grad[j], fd, scale)
        checked += n
    assert checked > 20


# ---------------------------------------------------------------- 5. the composition route
def test_composition_route_on_meshes_12_links_and_opaque(tmp_path):
    import pytorch_volumetric_b200 as pv
    robot, ref, text = build_robot("mixed_mesh", tmp_path / "mesh")
    robot.set_joint_configuration(torch.from_numpy(joint_values(ref, text, 20, seed=3)).cuda())
    dev = torch.device("cuda", torch.cuda.current_device())
    assert not robot.sdf._self_clearance_fused(dev)
    lp = robot.link_surface_points(num_points=40, seed=2)
    allowed = robot.self_collision_pairs()
    for m in (0.02, 0.1):
        got = robot.sdf.query_self_collision_cost(lp, allowed, m)
        _assert_close(got, _reference(robot.sdf, lp, allowed, m), ("mesh", m))
    cost, grad = robot.self_collision_cost(0.1, lp, allowed)
    assert cost.shape == (20,) and grad.shape == (20, len(robot.joint_names)) and bool((cost > 0).any())
    # 12 primitive links: the composition route
    prim = [pv.BoxSDF([0.1, 0.05, 0.04]), pv.CylinderSDF(0.03, 0.12), pv.SphereSDF(0.04)] * 4
    A = 40
    tsf = pv.Transform3d(matrix=workloads.random_rigid(12 * A, seed=4, t_range=0.12).cuda())
    comp = pv.ComposedSDF(prim, tsf)
    comp.set_transforms(tsf, batch_dim=(A,))
    lp12 = torch.cat([torch.from_numpy(surface_points(s, 24, k)) for k, s in enumerate(prim)])
    lp12 = lp12.reshape(12, 24, 3).float()
    lp12 = lp12.cuda()
    allowed12 = torch.ones(12, 12, dtype=torch.bool)
    got = comp.query_self_collision_cost(lp12, allowed12, 0.05)
    _assert_close(got, _reference(comp, lp12, allowed12, 0.05), "12 links")
    assert bool((got[0] > 0).any())
    # an opaque 8-link prefix (composition route) against the same links made native (fused route)
    opaque = pv.ComposedSDF(opaque_sdfs(pv, prim[:8]), None)
    native = pv.ComposedSDF(prim[:8], None)
    m8 = pv.Transform3d(matrix=tsf.get_matrix().reshape(12, A, 4, 4)[:8].reshape(-1, 4, 4))
    for c in (opaque, native):
        c.set_transforms(m8, batch_dim=(A,))
    assert not opaque._self_clearance_fused(dev) and native._self_clearance_fused(dev)
    a = opaque.query_self_collision_cost(lp12[:8], allowed12[:8, :8], 0.05)
    b = native.query_self_collision_cost(lp12[:8], allowed12[:8, :8], 0.05)
    ref8 = _reference(native, lp12[:8], allowed12[:8, :8], 0.05)
    _assert_close(b, ref8, "native prefix")
    # the opaque links rotate their gradient back with a torch matmul: the same sums to rounding
    assert torch.allclose(a[0], b[0], rtol=1e-5, atol=1e-9) and torch.allclose(a[1], b[1], rtol=1e-4, atol=1e-6)


# ---------------------------------------------------------------- 6. shapes
def test_shapes_float64_and_empty_rows(tmp_path):
    import pytorch_volumetric_b200 as pv
    robot = arm_robot(tmp_path, "primitive")
    S, J = len(robot.sdf.sdfs), len(robot.joint_names)
    q = wide_configurations(60, seed=9)
    robot.set_joint_configuration(q.cuda().reshape(3, 20, 7))
    c, g = robot.self_collision_cost(0.05)
    assert c.shape == (3, 20) and g.shape == (3, 20, J)
    cs, ts = robot.sdf.self_collision_cost(robot.link_surface_points(), robot.self_collision_pairs(), 0.05)
    assert cs.shape == (3, 20) and ts.shape == (3, 20, S, 6)
    flat = robot.sdf.query_self_collision_cost(robot.link_surface_points(), robot.self_collision_pairs(), 0.05)
    assert torch.equal(cs.reshape(-1), flat[0]) and torch.equal(ts.reshape(-1, S, 6), flat[1])
    # no configuration batch: 0-d / [S, 6] / [J]
    robot.set_joint_configuration(q[7].cuda())
    c1, g1 = robot.self_collision_cost(0.05)
    assert c1.shape == () and g1.shape == (J,)
    assert torch.equal(c1, c.reshape(-1)[7])
    c1s, t1s = robot.sdf.self_collision_cost(robot.link_surface_points(), robot.self_collision_pairs(), 0.05)
    assert c1s.shape == () and t1s.shape == (S, 6) and torch.equal(t1s, ts.reshape(-1, S, 6)[7])
    # K = 1, and no allowed pair: exactly 0
    robot.set_joint_configuration(q.cuda())
    lp1 = robot.link_surface_points(num_points=1, seed=2)
    c, t = robot.sdf.query_self_collision_cost(lp1, robot.self_collision_pairs(), 0.3)
    _assert_close((c, t), _reference(robot.sdf, lp1, robot.self_collision_pairs(), 0.3), "K=1")
    c, g = robot.self_collision_cost(10.0, allowed=torch.zeros(S, S, dtype=torch.bool))
    assert not c.any() and not g.any()
    # one source only (a single non-empty row): its twist is minus the sum of its targets'
    one = torch.zeros(S, S, dtype=torch.bool)
    one[S - 1, :S - 3] = True
    c, t = robot.sdf.query_self_collision_cost(robot.link_surface_points(), one, 0.1)
    assert bool((c > 0).any())
    assert torch.allclose(t[:, S - 1].double(), -t[:, :S - 3].double().sum(1), rtol=1e-5, atol=1e-7)
    assert not t[:, S - 3:S - 1].any()
    # a float64 chain: float64 results, within fp32 noise of the float32 chain
    urdf, end = workloads.write_primitive_arm(str(tmp_path / "f64"))
    r64 = pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(dtype=torch.float64, device="cuda"),
                      primitive_visuals=True)
    r64.set_joint_configuration(q.double().cuda())
    c64, g64 = r64.self_collision_cost(0.05)
    c32, g32 = robot.self_collision_cost(0.05)
    assert c64.dtype == torch.float64 and g64.dtype == torch.float64 and c64.shape == (60,)
    assert torch.allclose(c64.float(), c32, rtol=1e-3, atol=1e-6)
