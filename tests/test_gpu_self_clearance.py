"""GPU: self-clearance queries (ComposedSDF.self_clearance / query_self_clearance / RobotSDF.self_clearance).

1. The fused route (pvb_composed_query_self_clearance) equals the composition route (`_composed_self_clearance`,
   the definition) bit for bit in value, gradient, source, point and target, on the nearest, trilinear and primitive
   arms, over configuration counts, link point counts, slabs and `allowed` matrices -- each route checked to have run.
2. The composition route on the sets the fused kernel does not take: mesh links, 12 links, an opaque sub-SDF.
3. Against the fp64 robot of tests/robot_ref.py with the same link points posed in fp64: values within the FK-derived
   bounds of tests/test_gpu_robot_fp64.py, the argmin and gradient where the fp64 gap decides them.
4. A 2-D configuration batch, a float64 chain and repeated calls."""
import math

import numpy as np
import pytest
import torch

import robot_ref as rr
import workloads
from test_gpu_robot_fp64 import build_robot, joint_values, link_tolerances, point_bound
from test_gpu_swept import _arm_robot
from test_gpu_trilinear_composed import _opaque

pytestmark = pytest.mark.gpu


def _wide_configurations(A, seed, dtype=torch.float32):
    """Joint values uniform in +-pi: wide enough that the arm's links pass through one another."""
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(A, 7, generator=g, dtype=torch.float64) * 2 - 1) * math.pi).to(dtype)


def _routes(monkeypatch, comp, lp, allowed, cfg_begin=0, cfg_count=None):
    """(fused result, composition-route result), each with every index, after checking which route each call took."""
    from pytorch_volumetric_b200 import sdf as S
    calls = []
    orig = S.ComposedSDF._composed_self_clearance

    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(S.ComposedSDF, "_composed_self_clearance", spy)
    fused = comp.query_self_clearance(lp, allowed, cfg_begin=cfg_begin, cfg_count=cfg_count, return_which=True)
    assert not calls, "the fused route fell back to the composition route"
    n_cfg = math.prod(comp.tsf_batch) if comp.tsf_batch is not None else 1
    count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    K, rows = comp._self_clearance_args(lp, allowed)
    p = lp.detach().float().reshape(-1, 3).contiguous()
    ref = comp._composed_self_clearance(p, K, rows, cfg_begin, count, True)
    assert calls
    return fused, ref


def _assert_same(got, ref, what):
    for a, b, name in zip(got, ref, ("val", "grad", "src", "point", "which")):
        assert torch.equal(a, b), (what, name, int((a != b).sum()))


def _allowed(S, kind):
    i = torch.arange(S)
    if kind == "default":
        return (i[:, None] - i[None, :]).abs() >= 2
    if kind == "asymmetric":
        return (i[None, :] - i[:, None] >= 3) | ((i[:, None] == S - 1) & (i[None, :] == 0))
    return torch.zeros(S, S, dtype=torch.bool)


# ---------------------------------------------------------------- 1. fused == composition
@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_fused_equals_composition_on_the_arm(tmp_path, monkeypatch, kind):
    robot = _arm_robot(tmp_path, kind)
    S = len(robot.sdf.sdfs)
    cases = [(A, 33) for A in (1, 7, 31, 32, 33, 200, 1000)] + [(200, K) for K in (1, 31, 32, 256, 1000)]
    signs = set()
    for A, K in cases:
        robot.set_joint_configuration(_wide_configurations(A, seed=A + K).cuda())
        lp = robot.link_surface_points(num_points=K, seed=K)
        assert lp.shape == (S, K, 3)
        for which in ("default", "asymmetric", "empty"):
            if which != "default" and (A, K) not in ((33, 33), (200, 256)):
                continue
            allowed = _allowed(S, which)
            fused, ref = _routes(monkeypatch, robot.sdf, lp, allowed)
            _assert_same(fused, ref, (kind, A, K, which))
            if which == "empty":
                assert torch.isinf(fused[0]).all() and (fused[2] == -1).all() and (fused[1] == 0).all()
            else:
                signs.update(torch.sign(fused[0]).cpu().tolist())
                m = allowed.cuda()[fused[2].long(), fused[4].long()]
                assert m.all() and (fused[2] != fused[4]).all()
        if A == 200 and K == 256:
            for begin, count in ((0, 1), (17, 100), (199, 1), (50, 150)):
                fused, ref = _routes(monkeypatch, robot.sdf, lp, _allowed(S, "default"), begin, count)
                _assert_same(fused, ref, (kind, begin, count))
    assert {-1.0, 1.0} <= signs, (kind, signs)               # links really intersect, and really clear one another


def test_fused_equals_composition_at_70000_configurations(tmp_path, monkeypatch):
    robot = _arm_robot(tmp_path, "primitive")
    robot.set_joint_configuration(_wide_configurations(70_000, seed=5).cuda())
    lp = robot.link_surface_points(num_points=32, seed=1)
    fused, ref = _routes(monkeypatch, robot.sdf, lp, robot.self_collision_pairs())
    _assert_same(fused, ref, "70000")
    assert (fused[0] < 0).any() and (fused[0] > 0).any()


# ---------------------------------------------------------------- 2. the sets the fused kernel does not take
def test_composition_route_on_meshes_12_links_and_opaque(tmp_path):
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import sdf as S
    # mesh links (MeshSDF): the composition route, equal to the per-source paired clearance done by hand
    robot, ref, text = build_robot("mixed_mesh", tmp_path / "mesh")
    robot.set_joint_configuration(torch.from_numpy(joint_values(ref, text, 20, seed=3)).cuda())
    assert not robot.sdf._self_clearance_fused(torch.device("cuda", torch.cuda.current_device()))
    lp = robot.link_surface_points(num_points=40, seed=2)
    allowed = robot.self_collision_pairs()
    v, g, src, pt, which = robot.self_clearance(lp, allowed, return_argmin=True)
    Sn = len(robot.sdf.sdfs)
    inv = S._affine_inverse(robot.sdf._xforms_on(v.device)).reshape(Sn, 20, 4, 4)
    xf = robot.sdf._xforms_on(v.device).reshape(Sn, 20, 4, 4)
    best = None
    for i in range(Sn):
        js = [j for j in range(Sn) if allowed[i, j] and j != i]
        if not js:
            continue
        x = (inv[i, :, None, :3, :3] @ lp[i][None, :, :, None]).squeeze(-1) + inv[i, :, None, :3, 3]
        sub = pv.ComposedSDF([robot.sdf.sdfs[j] for j in js], pv.Transform3d(matrix=xf[js].reshape(-1, 4, 4)))
        sv = sub.query_paired_clearance(x, return_which=True)[0]
        best = sv if best is None else torch.minimum(best, sv)
    # the posing by hand rounds differently from pvb_transform_points_paired: values agree to fp32 noise
    assert torch.allclose(v.cuda(), best, atol=1e-5), (v.cuda() - best).abs().max()
    assert (allowed[src.cpu(), which.cpu()]).all()
    # 12 links and an opaque sub-SDF: the composition route, and where the fused route also serves (an 8-link prefix
    # with the opaque link made native), the two agree bit for bit
    prim = [pv.BoxSDF([0.1, 0.05, 0.04]), pv.CylinderSDF(0.03, 0.12), pv.SphereSDF(0.04)] * 4
    A = 40
    tsf = pv.Transform3d(matrix=workloads.random_rigid(12 * A, seed=4, t_range=0.12).cuda())
    comp = pv.ComposedSDF(prim, tsf)
    comp.set_transforms(tsf, batch_dim=(A,))
    lp12 = torch.cat([torch.from_numpy(_surface(s, 24, k)) for k, s in enumerate(prim)]).reshape(12, 24, 3).float()
    lp12 = lp12.cuda()
    allowed12 = torch.ones(12, 12, dtype=torch.bool)
    out12 = comp.self_clearance(lp12, allowed12, return_argmin=True)
    assert out12[0].shape == (A,) and (out12[2] != out12[4]).all()
    opaque = pv.ComposedSDF(_opaque(pv, prim[:8]), None)
    native = pv.ComposedSDF(prim[:8], None)
    m8 = pv.Transform3d(matrix=tsf.get_matrix().reshape(12, A, 4, 4)[:8].reshape(-1, 4, 4))
    for c in (opaque, native):
        c.set_transforms(m8, batch_dim=(A,))
    dev = torch.device("cuda", torch.cuda.current_device())
    assert not opaque._self_clearance_fused(dev) and native._self_clearance_fused(dev)
    a = opaque.query_self_clearance(lp12[:8], allowed12[:8, :8], return_which=True)
    b = native.query_self_clearance(lp12[:8], allowed12[:8, :8], return_which=True)
    # the opaque links evaluate through their own __call__ (the same primitive arithmetic) and rotate their gradient
    # back with a torch matmul: equal values and indices, gradients to rounding
    for t, u, name in zip(a, b, ("val", "grad", "src", "point", "which")):
        assert torch.equal(t, u) if name != "grad" else torch.allclose(t, u, atol=1e-6), name


def _surface(link_sdf, n, seed):
    from pytorch_volumetric_b200.model_to_sdf import _primitive_surface
    return _primitive_surface(link_sdf, n, np.random.default_rng(seed))


# ---------------------------------------------------------------- 3. against fp64
def _fp64_truth(ref, q, lp, allowed):
    """Per configuration: the fp64 minimum over (i, k, allowed j) with the link points posed in fp64, its (i, k, j),
    gradient, the gap to the second-best (i, k) candidate, and the value / gradient tolerances."""
    M = ref.object_to_link(q)                                        # [S, A, 4, 4] fp64
    W = rr.rigid_inverse(M)
    S, A = M.shape[:2]
    lp = np.asarray(lp, dtype=np.float64)
    K = lp.shape[1]
    cand_v, cand_g, cand_j, cand_tol, cand_gtol, cand_dec = [], [], [], [], [], []
    for i in range(S):
        x = np.einsum("aij,kj->aki", W[i, :, :3, :3], lp[i]) + W[i, :, None, :3, 3]     # [A, K, 3]
        per = ref.evaluate(M, x)
        pb, vt = link_tolerances(ref, q, x)
        # the posing of x in fp32: W_i's error (the inverse of M_i's) applied to the link point
        nf = ref.links[i].frame + 1
        pose = 2 * point_bound(nf, ref.reach(q)[i][:, None], np.linalg.norm(lp[i], axis=1)[None])   # [A, K]
        v = np.where(np.asarray(allowed)[i][:, None, None] & (np.arange(S) != i)[:, None, None], per["value"], np.inf)
        j = v.argmin(0)
        take = lambda t: np.take_along_axis(t, j[None], 0)[0]
        tol = vt.max(0) + pose
        second = np.sort(v, axis=0)[1] if S > 1 else np.full(v.shape[1:], np.inf)
        cand_v.append(take(v)); cand_j.append(j)
        cand_g.append(np.take_along_axis(per["grad"], j[None, ..., None], 0)[0])
        cand_tol.append(tol)
        cand_gtol.append(1e-6 + 2 * (take(pb) + pose) + 2 * (take(vt) + pose) / take(per["cond"]))
        # fp64 decides the target link, the shape's rule and the gradient's direction (as analyse does)
        cand_dec.append((second - take(v) > 2 * tol) & (take(per["gap"]) > take(vt) + pose) &
                        (take(per["cond"]) > 100 * (take(pb) + pose)))
    v = np.stack(cand_v, 1).reshape(A, S * K)                       # candidates (i, k), i-major
    order = np.argsort(v, axis=1, kind="stable")
    rows = np.arange(A)
    best = order[:, 0]
    tol = np.stack(cand_tol, 1).reshape(A, S * K)
    tmax = np.where(np.isfinite(v), tol, 0).max(1)
    gap = v[rows, order[:, 1]] - v[rows, best]
    g = np.stack(cand_g, 1).reshape(A, S * K, 3)[rows, best]
    jj = np.stack(cand_j, 1).reshape(A, S * K)[rows, best]
    gtol = np.stack(cand_gtol, 1).reshape(A, S * K)[rows, best]
    dec = np.stack(cand_dec, 1).reshape(A, S * K)[rows, best] & (gap > 2 * tmax)
    return dict(value=v[rows, best], src=best // K, point=best % K, which=jj, grad=g, decided=dec, tol=tmax,
                gtol=gtol)


@pytest.mark.parametrize("kind", ["mixed", "prim_arm"])
def test_self_clearance_against_fp64(tmp_path, kind):
    robot, ref, text = build_robot(kind, tmp_path)
    A = 300
    q = joint_values(ref, text, A, seed=21)
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    lp = robot.link_surface_points(num_points=128, seed=5)
    allowed = robot.self_collision_pairs()
    v, g, src, pt, which = (t.cpu().numpy() for t in robot.self_clearance(lp, allowed, return_argmin=True))
    truth = _fp64_truth(ref, q, lp.cpu().numpy(), allowed.numpy())
    err = np.abs(v - truth["value"])
    ok = truth["decided"]
    gerr = np.abs(g - truth["grad"]).max(1)
    print(f"{kind} self-clearance A={A}: max |value error| {err.max():.3g}, error / bound max "
          f"{(err / truth['tol']).max():.3f}, decided {int(ok.sum())} of {A}, gradient error / bound max "
          f"{(gerr / truth['gtol'])[ok].max():.3f}")
    assert (err <= truth["tol"]).all(), np.argmax(err / truth["tol"])
    assert (v < 0).any() and (v > 0).any()                          # links intersect in some configurations
    assert ok.mean() > 0.7
    assert (src[ok] == truth["src"][ok]).all() and (pt[ok] == truth["point"][ok]).all()
    assert (which[ok] == truth["which"][ok]).all()
    assert (gerr[ok] <= truth["gtol"][ok]).all(), (gerr / truth["gtol"])[ok].max()


# ---------------------------------------------------------------- 4. shapes, dtypes, repeatability
def test_batch_float64_and_repeat(tmp_path):
    robot = _arm_robot(tmp_path, "primitive")
    q = _wide_configurations(60, seed=9)
    robot.set_joint_configuration(q.cuda().reshape(3, 20, 7))
    v, g, src, pt, which = robot.self_clearance(return_argmin=True)
    assert v.shape == (3, 20) and g.shape == (3, 20, 3) and src.dtype == torch.int64 and pt.shape == (3, 20)
    flat = robot.sdf.query_self_clearance(robot.link_surface_points(), robot.self_collision_pairs(),
                                          return_which=True)
    assert torch.equal(v.reshape(-1), flat[0]) and torch.equal(which.reshape(-1), flat[4].long())
    for _ in range(2):                                              # identical bits on every call
        again = robot.self_clearance(return_argmin=True)
        assert all(torch.equal(a, b) for a, b in zip(again, (v, g, src, pt, which)))
    # one configuration without a batch: 0-d results
    robot.set_joint_configuration(q[7].cuda())
    one = robot.self_clearance(return_argmin=True)
    assert one[0].shape == () and one[1].shape == (3,)
    assert torch.equal(one[0], v.reshape(-1)[7]) and torch.equal(one[2], src.reshape(-1)[7])
    # a float64 chain: float64 results, within fp32 noise of the float32 chain
    import pytorch_volumetric_b200 as pv
    urdf, end = workloads.write_primitive_arm(str(tmp_path / "f64"))
    r64 = pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(dtype=torch.float64, device="cuda"),
                      primitive_visuals=True)
    r64.set_joint_configuration(q.double().cuda())
    v64, g64 = r64.self_clearance()
    assert v64.dtype == torch.float64 and v64.shape == (60,)
    assert torch.allclose(v64.float(), v.reshape(-1), atol=1e-4)
