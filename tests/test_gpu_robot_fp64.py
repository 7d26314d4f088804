"""GPU: RobotSDF end to end against the fp64 reference robot (tests/robot_ref.py): URDF -> forward kinematics -> link
frames -> link SDFs -> minimum, on general serial chains and on every kernel route the link and configuration counts
select.

Chains (written into tmp_path by robot_ref.write_chain):
  mixed        7 movable joints (revolute with unnormalised, non-axis-aligned axes, a continuous and a prismatic
               joint), two fixed joints inside the chain, nonzero rpy on every origin, links without visuals, a link
               with two visuals, a visual on the root, and a side branch off the path; 8 links.  Built with box,
               cylinder and sphere visuals, and with closed convex OBJ meshes (a tessellated box and an icosahedron,
               placed with a `scale`) through the default MeshSDF links.
  limit32      32 frames and 16 visuals: native forward kinematics at both of its limits.
  frames33     33 frames; links17: 17 visuals.  Both past a limit: the eager forward kinematics.
  arm, prim_arm  workloads.write_arm / write_primitive_arm (bench.py's C4 chain).

Tolerances follow from fp32 arithmetic (robot_ref.fk_bound, point_bound, link_tolerances); tests/test_robot_ref_cpu.py
checks that they cover the fp32 error of the package's eager forward kinematics with at most a 10x margin."""
import numpy as np
import pytest
import torch

from helpers import no_generic
from robot_ref import CHAINS, NATIVE, U32, analyse, build_robot, check, fk_bound, joint_values, sample_points


# ------------------------------------------------------------------------------------------------------- the tests
pytestmark = pytest.mark.gpu


def _fp64_object_to_link(ref, q, chunk=10_000):
    q2 = np.asarray(q).reshape(-1, ref.n_joints)
    return (np.concatenate([ref.object_to_link(q2[i:i + chunk]) for i in range(0, len(q2), chunk)], axis=1),
            np.concatenate([ref.reach(q2[i:i + chunk]) for i in range(0, len(q2), chunk)], axis=1))


@pytest.mark.parametrize("kind", CHAINS)
def test_forward_kinematics_against_fp64(tmp_path, kind):
    """object_to_link_frames against the fp64 reference: the native kernel (where the chain is within its limits),
    the eager fp32 path, and a float64 chain, at 1 (no batch), 37 and 100 000 configurations."""
    robot, ref, text = build_robot(kind, tmp_path)
    assert (robot._fk_plan is not None) == NATIVE[kind]
    S = len(ref.links)
    nf = np.array([l.frame + 1 for l in ref.links])[:, None]
    for A in (1, 37, 100_000):
        q = joint_values(ref, text, A, seed=A)
        mref, reach = _fp64_object_to_link(ref, q)
        bound = fk_bound(nf, reach)
        for native in (True, False):
            robot.native_fk = native
            robot.set_joint_configuration(torch.from_numpy(q).cuda())
            assert robot.configuration_batch == (None if A == 1 else torch.Size([A]))
            m = robot.object_to_link_frames.get_matrix().reshape(S, -1, 4, 4).double().cpu().numpy()
            err = np.abs(m - mref)[..., :3, :].max((-1, -2))
            path = "native" if native and robot._fk_plan is not None else "eager"
            print(f"{kind} A={A} {path}: max fk error {err.max():.3g}, error / fk_bound max {(err / bound).max():.3f}")
            assert (err <= bound).all(), (kind, A, path, np.unravel_index(np.argmax(err / bound), err.shape))
            assert (m[..., 3, :] == np.array([0.0, 0.0, 0.0, 1.0])).all()
    # float64: the eager path in fp64; only the fp32 visual origins (pk's convention) round, by u32 each
    r64, _, _ = build_robot(kind, tmp_path / "f64", dtype=torch.float64)
    q = joint_values(ref, text, 37, seed=2)
    mref, reach = _fp64_object_to_link(ref, q)
    r64.set_joint_configuration(torch.from_numpy(q).double().cuda())
    m = r64.object_to_link_frames.get_matrix().reshape(S, -1, 4, 4).cpu().numpy()
    err = np.abs(m - mref)[..., :3, :].max((-1, -2))
    print(f"{kind} float64 chain: max fk error {err.max():.3g}, error / bound max "
          f"{(err / (3 * U32 * (1 + reach))).max():.3f}")
    assert (err <= 3 * U32 * (1 + reach)).all()


# (chain, configurations, the kernel pvb_composed_query selects for that link set and count)
ROUTES = [
    ("mixed", 1, "point-major"),
    ("mixed", 5, "point-major"),
    ("mixed", 8, "robot_serial_kernel"),
    ("mixed", 33, "robot_serial_kernel, lane-split remainder"),
    ("mixed", 200, "robot_serial_kernel, lane-split remainder"),
    ("prim_arm", 200, "robot_serial_kernel"),
    ("limit32", 64, "configuration-major, primitives"),
    ("links17", 8, "point-major, 128 sub-SDF slots"),
    ("mixed_mesh", 5, "mesh point-major"),
    ("mixed_mesh", 40, "mesh point-major"),
]


@pytest.mark.parametrize("kind,A,route", ROUTES, ids=[f"{k}-{a}" for k, a, _ in ROUTES])
def test_query_against_fp64(tmp_path, monkeypatch, kind, A, route):
    """Values everywhere, gradients and the argmin link where fp64 decides them, on every route."""
    robot, ref, text = build_robot(kind, tmp_path)
    S = len(ref.links)
    assert robot._fk_plan is not None or S > 16
    q = joint_values(ref, text, A, seed=7 + A)
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    n = 400 if kind == "mixed_mesh" else (1500 if A >= 64 else 4000)
    pts = sample_points(ref, ref.object_to_link(q), n, seed=A)
    no_generic(monkeypatch, robot.sdf)
    v, g, w = robot.sdf.query(torch.from_numpy(pts).float().cuda(), return_which=True)
    P = len(pts)
    truth = analyse(ref, q, pts)
    check(f"{kind} A={A} [{route}] S={S} P={P}", truth, v.reshape(-1, P).cpu().numpy(),
          g.reshape(-1, P, 3).cpu().numpy(), w.reshape(-1, P).cpu().numpy())


def test_paired_swept_clearance_against_fp64(tmp_path):
    """paired, swept and clearance on the mixed primitive robot at 33 configurations against the fp64 reductions of
    the same per-(configuration, point) truth; the argmin where the fp64 gap decides it."""
    robot, ref, text = build_robot("mixed", tmp_path)
    A = 33
    q = joint_values(ref, text, A, seed=11)
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    pts = sample_points(ref, ref.object_to_link(q), 1000, seed=12)
    P = len(pts)
    # paired: configuration a at its own 700 points
    own = pts[np.random.default_rng(13).integers(0, P, (A, 700))]
    pv_, pg = robot.paired(torch.from_numpy(own).float().cuda())
    check("mixed paired A=33", analyse(ref, q, own), pv_.cpu().numpy(), pg.cpu().numpy())
    truth = analyse(ref, q, pts)
    rv, tol, dec = truth["value"], truth["tol"], truth["decided"]
    pts_t = torch.from_numpy(pts).float().cuda()
    # swept: the first configuration attaining the minimum at every point
    sv, sg, scfg, swhich = (t.cpu().numpy() for t in robot.swept(pts_t, return_argmin=True))
    a_best = rv.argmin(0)
    cols = np.arange(P)
    srt = np.sort(rv, axis=0)
    tmax = tol.max(0)
    ok = (srt[1] - srt[0] > 2 * tmax) & dec[a_best, cols]
    err = np.abs(sv - srt[0])
    print(f"mixed swept A=33: max |value error| {err.max():.3g}, error / bound max {(err / tmax).max():.3f}, "
          f"skipped {int((~ok).sum())} of {P}")
    # points nearest the root link tie across every configuration (the root does not move): their argmin is the
    # first configuration by the tie rule, not by fp64, and they are skipped
    assert (err <= tmax).all() and ok.mean() > 0.8
    assert (scfg[ok] == a_best[ok]).all() and (swhich[ok] == truth["which"][a_best, cols][ok]).all()
    assert (np.abs(sg - truth["grad"][a_best, cols]).max(1) <= truth["gtol"][a_best, cols])[ok].all()
    # clearance: the first point attaining the minimum for every configuration
    cv, cg, cidx, cwhich = (t.cpu().numpy() for t in robot.clearance(pts_t, return_argmin=True))
    assert cv.shape == (A,)
    p_best = rv.argmin(1)
    rows = np.arange(A)
    srt = np.sort(rv, axis=1)
    tmax = tol.max(1)
    ok = (srt[:, 1] - srt[:, 0] > 2 * tmax) & dec[rows, p_best]
    err = np.abs(cv - srt[:, 0])
    print(f"mixed clearance A=33: max |value error| {err.max():.3g}, error / bound max {(err / tmax).max():.3f}, "
          f"skipped {int((~ok).sum())} of {A}")
    assert (err <= tmax).all() and ok.mean() > 0.8
    assert (cidx[ok] == p_best[ok]).all() and (cwhich[ok] == truth["which"][rows, p_best][ok]).all()
    assert (np.abs(cg - truth["grad"][rows, p_best]).max(1) <= truth["gtol"][rows, p_best])[ok].all()
