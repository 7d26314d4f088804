"""GPU: RobotSDF on kinematic trees (build_chain_from_urdf) against the fp64 tree reference (tests/tree_ref.py).

1. Forward kinematics: the native tree kernel (pvb_fk_tree), the eager fp32 path and a float64 chain against fp64 at
   1, 37 and 100 000 configurations, on the mixed chain read as a tree, the hand (primitives and meshes), the gripper,
   a generated tree at exactly 64 frames and 64 links (native) and one of 65 frames (eager); batches of any shape.
2. Serial URDFs parsed as a tree give SerialChain's bits: transforms on the native and eager paths, and queries.
3. Branches are independent: moving one finger leaves every link off its subtree bit for bit where it was.
4. Every query form on trees against fp64: the gripper (8 links) on the fused kernels, the hand on the composition
   routes; the fused and composition self_clearance agree bit for bit on the gripper.
5. The joint gradients of collision_cost, paired_collision_cost and self_collision_cost against central differences
   of the fp64 cost, and a cloud at one finger gives every other finger's joints exactly 0."""
import numpy as np
import pytest
import torch

import workloads
from robot_ref import U32, build_robot, fk_bound, joint_values
from test_gpu_self_clearance import _fp64_truth, _routes
from test_gpu_self_collision_cost import _fp64_per_point
from tree_ref import NATIVE, TREES, analyse, build_tree, check, sample_points

pytestmark = pytest.mark.gpu


def _urdf(tmp_path, kind):
    """The URDF build_tree wrote for the hand or the gripper."""
    return str(tmp_path / ("gripper_tree.urdf" if kind == "gripper" else "hand.urdf"))


def _frames(robot, S):
    return robot.object_to_link_frames.get_matrix().reshape(S, -1, 4, 4)


# ---------------------------------------------------------------- 1. forward kinematics against fp64
@pytest.mark.parametrize("kind", TREES)
def test_forward_kinematics_against_fp64(tmp_path, kind):
    robot, ref, text = build_tree(kind, tmp_path)
    assert (robot._fk_plan is not None) == NATIVE[kind]
    S = len(ref.links)
    nf = ref.path_frames()[:, None]
    for A in (1, 37, 100_000):
        q = joint_values(ref, text, A, seed=A)
        mref = np.concatenate([ref.object_to_link(q.reshape(-1, ref.n_joints)[i:i + 10_000])
                               for i in range(0, max(A, 1), 10_000)], axis=1)
        reach = np.concatenate([ref.reach(q.reshape(-1, ref.n_joints)[i:i + 10_000])
                                for i in range(0, max(A, 1), 10_000)], axis=1)
        bound = fk_bound(nf, reach)
        for native in (True, False):
            robot.native_fk = native
            robot.set_joint_configuration(torch.from_numpy(q).cuda())
            assert robot.configuration_batch == (None if A == 1 else torch.Size([A]))
            m = _frames(robot, S).double().cpu().numpy()
            err = np.abs(m - mref)[..., :3, :].max((-1, -2))
            path = "native" if native and robot._fk_plan is not None else "eager"
            print(f"{kind} A={A} {path}: max fk error {err.max():.3g}, error / bound max {(err / bound).max():.3f}")
            assert (err <= bound).all(), (kind, A, path)
            assert (m[..., 3, :] == np.array([0.0, 0.0, 0.0, 1.0])).all()
    # batches of any shape: the rows of the flat batch
    robot.native_fk = True
    q = torch.from_numpy(joint_values(ref, text, 20, seed=1)).cuda()
    robot.set_joint_configuration(q)
    flat = robot.object_to_link_frames.get_matrix().clone()
    robot.set_joint_configuration(q.reshape(4, 5, -1))
    assert robot.configuration_batch == torch.Size([4, 5])
    assert torch.equal(robot.object_to_link_frames.get_matrix(), flat)
    # float64: the eager path in fp64
    r64, _, _ = build_tree(kind, tmp_path / "f64", dtype=torch.float64)
    q = joint_values(ref, text, 37, seed=2)
    r64.set_joint_configuration(torch.from_numpy(q).double().cuda())
    err = np.abs(_frames(r64, S).cpu().numpy() - ref.object_to_link(q))[..., :3, :].max((-1, -2))
    assert (err <= 3 * U32 * (1 + ref.reach(q))).all()


# ---------------------------------------------------------------- 2. serial URDFs keep their bits
@pytest.mark.parametrize("kind", ["limit32", "arm", "prim_arm"])
def test_serial_urdf_as_a_tree_gives_the_serial_bits(tmp_path, kind):
    import pytorch_volumetric_b200 as pv
    serial, ref, text = build_robot(kind, tmp_path)
    tree = pv.RobotSDF(pv.build_chain_from_urdf(text).to(device="cuda"), path_prefix=str(tmp_path),
                       primitive_visuals=serial._link_factories[0] is None)
    assert tree._fk_plan is not None and tree._fk_plan[2] is not None and serial._fk_plan[2] is None
    q = torch.from_numpy(joint_values(ref, text, 300, seed=6)).cuda()
    pts = torch.from_numpy(sample_points(ref, ref.object_to_link(q.cpu().numpy()[:20]), 500, seed=2)).float().cuda()
    for native in (True, False):
        serial.native_fk = tree.native_fk = native
        serial.set_joint_configuration(q)
        tree.set_joint_configuration(q)
        assert torch.equal(serial.object_to_link_frames.get_matrix(), tree.object_to_link_frames.get_matrix()), native
        for a, b in zip(serial.sdf.query(pts, return_which=True), tree.sdf.query(pts, return_which=True)):
            assert torch.equal(a, b), native


# ---------------------------------------------------------------- 3. branches are independent
@pytest.mark.parametrize("kind,finger", [("hand", "finger2"), ("gripper", "finger_b")])
def test_moving_one_finger_leaves_the_other_links(tmp_path, kind, finger):
    robot, ref, text = build_tree(kind, tmp_path)
    S = len(ref.links)
    q = torch.from_numpy(joint_values(ref, text, 500, seed=3)).cuda()
    cols = [k for k, n in enumerate(robot.joint_names) if n.startswith(finger)]
    assert cols
    q2 = q.clone()
    q2[:, cols] = torch.rand(len(q), len(cols), device="cuda")
    on_finger = np.array([robot.sdf_to_link_name[s].startswith(finger) for s in range(S)])
    assert on_finger.any() and not on_finger.all()
    for native in (True, False):
        robot.native_fk = native
        robot.set_joint_configuration(q)
        m1 = _frames(robot, S).clone()
        robot.set_joint_configuration(q2)
        m2 = _frames(robot, S)
        assert torch.equal(m1[~on_finger], m2[~on_finger]), native
        assert not torch.equal(m1[on_finger], m2[on_finger])


# ---------------------------------------------------------------- 4. every query form against fp64
def _reduced(label, value, grad, idx, which, v, tol, dec, gref, gtol, wref, axis):
    """swept / clearance / paired_clearance against the fp64 per-(configuration, point) truth reduced over `axis`."""
    best = v.argmin(axis)
    srt = np.sort(v, axis=axis)
    tmax = tol.max(axis)
    take = lambda x: np.take_along_axis(x, np.expand_dims(best, axis), axis).squeeze(axis)
    lo, nxt = np.take(srt, 0, axis), np.take(srt, 1, axis)
    ok = (nxt - lo > 2 * tmax) & take(dec)
    err = np.abs(value - lo)
    print(f"{label}: max |value error| {err.max():.3g}, error / bound max {(err / tmax).max():.3f}, "
          f"skipped {int((~ok).sum())} of {ok.size}")
    assert (err <= tmax).all() and ok.mean() > 0.7
    assert (idx[ok] == best[ok]).all() and (which[ok] == take(wref)[ok]).all()
    g = np.take_along_axis(gref, np.expand_dims(best, axis)[..., None], axis).squeeze(axis)
    assert (np.abs(grad - g).max(-1) <= take(gtol))[ok].all()


@pytest.mark.parametrize("kind,A", [("gripper", 200), ("hand", 40)])
def test_query_forms_against_fp64(tmp_path, monkeypatch, kind, A):
    robot, ref, text = build_tree(kind, tmp_path)
    q = workloads.tree_configurations(_urdf(tmp_path, kind), A, seed=A).numpy()
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    pts = sample_points(ref, ref.object_to_link(q), 600, seed=A)
    P = len(pts)
    pts_t = torch.from_numpy(pts).float().cuda()
    truth = analyse(ref, q, pts)
    v, g, w = robot.sdf.query(pts_t, return_which=True)
    check(f"{kind} A={A} __call__", truth, v.reshape(A, P).cpu().numpy(), g.reshape(A, P, 3).cpu().numpy(),
          w.reshape(A, P).cpu().numpy())
    v2, g2 = robot(pts_t)
    assert torch.equal(v2.reshape(-1), v.reshape(-1))
    own = pts[np.random.default_rng(5).integers(0, P, (A, 300))]
    pv_, pg = robot.paired(torch.from_numpy(own).float().cuda())
    own_truth = analyse(ref, q, own)
    check(f"{kind} A={A} paired", own_truth, pv_.cpu().numpy(), pg.cpu().numpy())
    T = truth
    sv, sg, scfg, swhich = (t.cpu().numpy() for t in robot.swept(pts_t, return_argmin=True))
    # points nearest the root link tie across configurations (the root does not move): skipped as undecided
    best = T["value"].argmin(0)
    srt = np.sort(T["value"], axis=0)
    ok = (srt[1] - srt[0] > 2 * T["tol"].max(0)) & T["decided"][best, np.arange(P)]
    assert (np.abs(sv - srt[0]) <= T["tol"].max(0)).all() and ok.mean() > 0.5
    assert (scfg[ok] == best[ok]).all() and (swhich[ok] == T["which"][best, np.arange(P)][ok]).all()
    cv, cg, cidx, cwhich = (t.cpu().numpy() for t in robot.clearance(pts_t, return_argmin=True))
    _reduced(f"{kind} clearance", cv, cg, cidx, cwhich, T["value"], T["tol"], T["decided"], T["grad"], T["gtol"],
             T["which"], 1)
    O = own_truth
    qv, qg, qidx, qwhich = (t.cpu().numpy() for t in robot.paired_clearance(torch.from_numpy(own).float().cuda(),
                                                                             return_argmin=True))
    _reduced(f"{kind} paired_clearance", qv, qg, qidx, qwhich, O["value"], O["tol"], O["decided"], O["grad"],
             O["gtol"], O["which"], 1)
    # self_clearance with the tree's default pairs
    lp = robot.link_surface_points(num_points=96, seed=5)
    allowed = robot.self_collision_pairs()
    sv, sg, src, spt, swh = (t.cpu().numpy() for t in robot.self_clearance(lp, allowed, return_argmin=True))
    st = _fp64_truth(ref, q, lp.cpu().numpy(), allowed.numpy())
    err = np.abs(sv - st["value"])
    ok = st["decided"]
    print(f"{kind} self_clearance: error / bound max {(err / st['tol']).max():.3f}, decided {int(ok.sum())} of {A}")
    assert (err <= st["tol"]).all() and ok.mean() > 0.5
    assert (src[ok] == st["src"][ok]).all() and (spt[ok] == st["point"][ok]).all() and (swh[ok] == st["which"][ok]).all()
    assert (np.abs(sg - st["grad"]).max(1) <= st["gtol"])[ok].all()
    if kind == "gripper":
        fused, comp = _routes(monkeypatch, robot.sdf, lp, allowed)
        for a, b in zip(fused, comp):
            assert torch.equal(a, b)


# ---------------------------------------------------------------- 5. joint gradients
def _cost_fd(ref, q, pts, m, h):
    """fp64 central differences of the collision cost over points [P, 3] (or [A, P, 3]) at one configuration."""
    out = []
    for j in range(ref.n_joints):
        qp, qm = q.copy(), q.copy()
        qp[0, j] += h
        qm[0, j] -= h
        cp = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qp), pts))[0], 0) ** 2
        cm = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(qm), pts))[0], 0) ** 2
        out.append((cp.sum() - cm.sum()) / (2 * h))
    return np.array(out)


def _stable(ref, q, cloud, m):
    per = ref.evaluate(ref.object_to_link(q), cloud)
    v, _, w = ref.compose(per)
    second = np.sort(per["value"], axis=0)[1]
    gap = np.take_along_axis(per["gap"], w[None], 0)[0]
    cond = np.take_along_axis(per["cond"], w[None], 0)[0]
    keep = (gap[0] > 1e-3) & (second[0] - v[0] > 1e-3) & (cond[0] > 5e-2) & (np.abs(v[0] - m) > 1e-3) & (v[0] < m)
    return cloud[keep]


@pytest.mark.parametrize("kind", ["gripper", "hand"])
def test_cost_joint_gradients_against_fp64_differences(tmp_path, kind):
    robot, ref, text = build_tree(kind, tmp_path)
    J = len(robot.joint_names)
    qs = workloads.tree_configurations(_urdf(tmp_path, kind), 4, seed=11).numpy()
    m, h = (0.04, 2.0 ** -16) if kind == "gripper" else (0.015, 2.0 ** -16)
    rng = np.random.default_rng(7)
    lo, hi = (np.array([-0.4, -0.4, -0.05]), np.array([0.4, 0.4, 0.6])) if kind == "gripper" else \
        (np.array([-0.2, -0.2, -0.1]), np.array([0.2, 0.2, 0.3]))
    cloud = rng.uniform(lo, hi, (40000, 3)).astype(np.float32).astype(np.float64)
    checked = 0
    for a in range(1, len(qs)):
        q = qs[a:a + 1].astype(np.float64)
        pts = _stable(ref, q, cloud, m)
        if len(pts) < 5:
            continue
        robot.set_joint_configuration(torch.from_numpy(qs[a:a + 1]).cuda())
        twists = robot.joint_twists().cpu().numpy()[0]
        hinge = np.maximum(m - ref.compose(ref.evaluate(ref.object_to_link(q), pts))[0][0], 0)
        scale = np.array([(2 * hinge * (np.linalg.norm(twists[j, :3]) + np.linalg.norm(pts, axis=1) *
                                        np.linalg.norm(twists[j, 3:]))).sum() for j in range(J)])
        fd = _cost_fd(ref, q, pts, m, h)
        p32 = torch.from_numpy(pts.astype(np.float32)).cuda()
        _, grad = robot.collision_cost(p32, m)
        assert (np.abs(grad.double().cpu().numpy().reshape(-1) - fd) <= 5e-4 * scale + 1e-9).all(), (kind, a)
        _, pgrad = robot.paired_collision_cost(p32[None], m)
        assert (np.abs(pgrad.double().cpu().numpy().reshape(-1) - fd) <= 5e-4 * scale + 1e-9).all(), (kind, a)
        checked += len(pts)
    assert checked > 50
    # self_collision_cost: link points whose target, rule and side of the margin stay put, the rest moved away
    allowed = robot.self_collision_pairs().numpy().copy()
    lp_all = robot.link_surface_points(num_points=400, seed=3).double().cpu().numpy().astype(np.float32)
    lp_all = lp_all.astype(np.float64)
    S = len(ref.links)
    # joint values across their whole range, so that the links come within the margin of one another
    qs = joint_values(ref, text, 6 if kind == "gripper" else 3, seed=9)
    ms = 0.05 if kind == "gripper" else 0.02
    done = 0
    for a in range(1, len(qs)):
        q = qs[a:a + 1].astype(np.float64)
        per = _fp64_per_point(ref, q, lp_all, allowed)
        stable = (per["gap"][0] > 1e-3) & (per["second"][0] - per["v"][0] > 1e-3) & (per["cond"][0] > 5e-2) & \
            (np.abs(per["v"][0] - ms) > 1e-3) & (per["v"][0] < ms)
        n = int(stable.sum(1).max())
        if n == 0:
            continue
        lp = np.full((S, n, 3), 100.0)
        for i in range(S):
            sel = lp_all[i][stable[i]]
            lp[i, :len(sel)] = sel
        robot.set_joint_configuration(torch.from_numpy(qs[a:a + 1]).cuda())
        _, grad = robot.self_collision_cost(ms, torch.from_numpy(lp.astype(np.float32)).cuda(),
                                            torch.from_numpy(allowed))
        grad = grad.double().cpu().numpy().reshape(-1)
        twists = robot.joint_twists().cpu().numpy()[0]
        base = _fp64_per_point(ref, q, lp, allowed)
        hinge = np.maximum(ms - base["v"][0], 0)
        for j in range(J):
            qp, qm = q.copy(), q.copy()
            qp[0, j] += h
            qm[0, j] -= h
            fd = ((np.maximum(ms - _fp64_per_point(ref, qp, lp, allowed)["v"], 0) ** 2).sum() -
                  (np.maximum(ms - _fp64_per_point(ref, qm, lp, allowed)["v"], 0) ** 2).sum()) / (2 * h)
            scale = 2 * (2 * hinge * (np.linalg.norm(twists[j, :3]) + np.linalg.norm(base["x"][0], axis=-1) *
                                      np.linalg.norm(twists[j, 3:]))).sum()
            assert abs(grad[j] - fd) <= 5e-4 * scale + 1e-9, (kind, a, j, grad[j], fd)
        done += n
    assert done > 0


@pytest.mark.parametrize("kind,finger,palm", [("hand", "thumb", ["wrist_pitch", "wrist_roll"]),
                                              ("gripper", "finger_b", ["j1", "j2", "j3"])])
def test_a_cloud_at_one_finger_moves_only_its_joints_and_the_arm(tmp_path, kind, finger, palm):
    """Points near the last finger in frame order only: under a serial reading of the frame order every earlier
    finger's joints would be credited with its links; on the tree they are exactly 0."""
    robot, ref, text = build_tree(kind, tmp_path)
    q = workloads.tree_configurations(_urdf(tmp_path, kind), 3, seed=2).numpy()
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    m = 0.01
    on = np.array([robot.sdf_to_link_name[s].startswith(finger) for s in range(len(ref.links))])
    M = ref.object_to_link(q)
    lp = robot.link_surface_points(num_points=200, seed=1).double().cpu().numpy()
    # the finger's surface points pushed 5 mm outward along the gradient, in the robot frame of every configuration
    W = np.linalg.inv(M)
    rows = []
    for a in range(len(q)):
        x = np.concatenate([lp[s] @ W[s, a, :3, :3].T + W[s, a, :3, 3] for s in np.flatnonzero(on)])
        per = ref.evaluate(M[:, a:a + 1], x)
        v, g, _ = ref.compose(per)
        x = x + 0.005 * g[0]
        per = ref.evaluate(M[:, a:a + 1], x)
        far = np.where(on[:, None], np.inf, per["value"][:, 0]).min(0) > m + 1e-3
        rows.append(x[far][:2000])
    n = min(len(r) for r in rows)
    assert n > 50
    cloud = torch.from_numpy(np.stack([r[:n] for r in rows]).astype(np.float32)).cuda()     # [A, n, 3]
    results = [("paired_collision_cost", robot.paired_collision_cost(cloud, m))]
    robot.set_joint_configuration(torch.from_numpy(q[:1]).cuda())
    results.append(("collision_cost", robot.collision_cost(cloud[0], m)))
    for name, (cost, grad) in results:
        grad = grad.reshape(-1, len(robot.joint_names)).cpu()
        assert (cost > 0).all(), name
        for k, jn in enumerate(robot.joint_names):
            if jn.startswith(finger) or jn in palm:
                continue
            assert (grad[:, k] == 0).all(), (name, jn, grad[:, k])
        for jn in palm:
            assert (grad[:, robot.joint_names.index(jn)] != 0).all(), (name, jn)
