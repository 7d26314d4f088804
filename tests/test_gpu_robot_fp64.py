"""GPU: RobotSDF end to end against the fp64 reference robot (tests/robot_ref.py): URDF -> forward kinematics -> link
frames -> link SDFs -> minimum, on general serial chains and on every kernel route the link and configuration counts
select.

Chains (written into tmp_path by the helpers below):
  mixed        7 movable joints (revolute with unnormalised, non-axis-aligned axes, a continuous and a prismatic
               joint), two fixed joints inside the chain, nonzero rpy on every origin, links without visuals, a link
               with two visuals, a visual on the root, and a side branch off the path; 8 links.  Built with box,
               cylinder and sphere visuals, and with closed convex OBJ meshes (a tessellated box and an icosahedron,
               placed with a `scale`) through the default MeshSDF links.
  limit32      32 frames and 16 visuals: native forward kinematics at both of its limits.
  frames33     33 frames; links17: 17 visuals.  Both past a limit: the eager forward kinematics.
  arm, prim_arm  workloads.write_arm / write_primitive_arm (bench.py's C4 chain).

Tolerances follow from fp32 arithmetic (fk_bound, point_bound, link_tolerances); tests/test_robot_ref_cpu.py checks
that they cover the fp32 error of the package's eager forward kinematics with at most a 10x margin."""
import math
import os

import numpy as np
import pytest
import torch

import robot_ref as rr
import workloads

U32 = rr.EPS32 / 2          # fp32 unit roundoff


# ------------------------------------------------------------------------------------------------ tolerance model
def fk_bound(n_frames, reach):
    """Bound on every entry of [R | t] of an object->link transform computed in fp32.  Each of the n_frames joint
    steps T @ origin @ motion(q), the rigid inverse and the visual-offset product rounds 3-term dot products
    (gamma_3 ~ 3 u32 each), and lever arms up to `reach` carry the rounding of the rotation block into the
    translation."""
    return 3 * U32 * (np.asarray(n_frames) + 2) * (1 + np.asarray(reach))


def point_bound(n_frames, reach, pnorm):
    """Bound on |q - q_fp64| of the link-frame point q = R p + t: the transform's error applied to p, and the fp32
    rounding of R p + t itself (3 terms of magnitude up to |p| and reach)."""
    return fk_bound(n_frames, reach) * (1 + pnorm) + 3 * U32 * (pnorm + reach)


def link_tolerances(ref, q, pts):
    """[S, A, P] (point_bound, value tolerance) of every link: point_bound plus the fp32 evaluation of the link SDF at
    |q| <= |p| + reach, and for mesh links the 5e-6 x scale the fp32 mesh path is allowed."""
    reach = ref.reach(q)[..., None]                                            # [S, A, 1]
    nf = np.array([l.frame + 1 for l in ref.links])[:, None, None]
    pnorm = np.linalg.norm(np.asarray(pts, dtype=np.float64), axis=-1)
    pnorm = pnorm[None, :, :] if pnorm.ndim == 2 else pnorm[None, None, :]
    pb = point_bound(nf, reach, pnorm)
    mesh = np.array([5e-6 * max(1.0, l.extent) if l.kind == "mesh" else 0.0 for l in ref.links])[:, None, None]
    return pb, pb + 3 * U32 * (pnorm + reach) + mesh


# ------------------------------------------------------------------------------------------------------ the chains
def _o(xyz, rpy):
    return f'<origin xyz="{xyz}" rpy="{rpy}"/>'


# (link, joint (type, origin xyz, origin rpy, axis) or None for the root, visuals [(kind, dims, xyz, rpy)])
MIXED_CHAIN = [
    ("base", None, [("box", (0.24, 0.2, 0.1), "0 0 0.05", "0 0 0.3")]),
    ("l1", ("revolute", "0.02 -0.01 0.12", "0.1 -0.2 0.3", "0.3 -0.5 0.8"),
     [("cylinder", (0.05, 0.18), "0 0 0.09", "0.2 0 0")]),
    ("l2", ("revolute", "0 0.03 0.2", "-0.3 0.1 0.2", "1 1 0"), []),
    ("l3", ("fixed", "0.05 0 0.08", "0.4 -0.1 0.25", None),
     [("box", (0.08, 0.1, 0.2), "0 0 0.1", "0 0.15 0.6"), ("sphere", (0.06,), "0.03 0 0.21", "0.3 0.2 0.1")]),
    ("l4", ("prismatic", "0 0 0.22", "0.2 0.3 -0.1", "0.2 1 -0.4"),
     [("cylinder", (0.045, 0.2), "0 0 0.1", "0.1 -0.1 0.9")]),
    ("l5", ("continuous", "0.01 0.02 0.2", "-0.2 0.25 0.1", "-1 0.5 2"),
     [("box", (0.09, 0.07, 0.16), "0 0 0.08", "-0.2 0 1.2")]),
    ("l6", ("revolute", "0 0 0.17", "0.15 0.1 -0.3", "0 0.6 0.8"), []),
    ("l7", ("fixed", "0.02 0 0.05", "0 -0.3 0.2", None), [("sphere", (0.05,), "0 0 0.04", "0.1 0 -0.2")]),
    ("l8", ("revolute", "0 0.01 0.12", "0.3 0 0.1", "1 0 0.3"), []),
    ("l9", ("revolute", "0 0 0.1", "-0.1 0.2 0.3", "0.2 -0.7 0.4"),
     [("cylinder", (0.03, 0.1), "0 0 0.05", "0 0.25 1.5")]),
]
MIXED_SIDE = ("side", ("revolute", "0.1 0 0", "0 0 0.5", "0 0 1"), "l4")       # off the path: ignored
PRISMATIC_RANGE = 0.3        # metres; revolute joints are drawn in +-pi


def _geometry(kind, dims, meshes):
    if meshes:      # a unit box / unit icosahedron scaled to the primitive's extents
        if kind == "box":
            return f'<mesh filename="box.obj" scale="{dims[0]} {dims[1]} {dims[2]}"/>'
        r, hz = (dims[0], dims[0]) if kind == "sphere" else (dims[0], dims[1] / 2)
        return f'<mesh filename="ico.obj" scale="{r} {r} {hz}"/>'
    if kind == "box":
        return f'<box size="{dims[0]} {dims[1]} {dims[2]}"/>'
    if kind == "cylinder":
        return f'<cylinder radius="{dims[0]}" length="{dims[1]}"/>'
    return f'<sphere radius="{dims[0]}"/>'


def _write_urdf(dirname, name, chain, meshes=False, extra=""):
    os.makedirs(dirname, exist_ok=True)
    parts = [f'<robot name="{name}">']
    for link, _, visuals in chain:
        vis = "".join(f'<visual>{_o(xyz, rpy)}<geometry>{_geometry(k, d, meshes)}</geometry></visual>'
                      for k, d, xyz, rpy in visuals)
        parts.append(f'<link name="{link}">{vis}</link>')
    for (parent, _, _), (link, joint, _) in zip(chain, chain[1:]):
        jt, xyz, rpy, axis = joint
        ax = f'<axis xyz="{axis}"/>' if axis else ""
        parts.append(f'<joint name="j_{link}" type="{jt}"><parent link="{parent}"/><child link="{link}"/>'
                     f'{_o(xyz, rpy)}{ax}<limit lower="-3.2" upper="3.2"/></joint>')
    parts.append(extra + "</robot>")
    path = os.path.join(dirname, name + ".urdf")
    with open(path, "w") as fh:
        fh.write("\n".join(parts))
    if meshes:
        from pytorch_volumetric_b200.meshio import write_obj
        write_obj(os.path.join(dirname, "box.obj"), *tessellated_box(3))
        write_obj(os.path.join(dirname, "ico.obj"), *icosahedron())
    return path, chain[-1][0]


def write_mixed(dirname, meshes=False):
    side, (jt, xyz, rpy, axis), parent = MIXED_SIDE
    extra = (f'<link name="{side}"><visual><geometry><box size="0.3 0.3 0.3"/></geometry></visual></link>'
             f'<joint name="j_{side}" type="{jt}"><parent link="{parent}"/><child link="{side}"/>{_o(xyz, rpy)}'
             f'<axis xyz="{axis}"/></joint>')
    return _write_urdf(dirname, "mixed_mesh" if meshes else "mixed", MIXED_CHAIN, meshes, extra)


def write_long_chain(dirname, n_frames, n_visuals, seed=0):
    """n_frames frames, every 6th joint fixed and every 7th prismatic, the others revolute about random
    unnormalised axes, origins of about 6 cm with random rpy; n_visuals box / cylinder / sphere visuals spread
    over the frames (the root included)."""
    rng = np.random.default_rng(seed)
    fmt = lambda v: " ".join(f"{x:.6f}" for x in v)
    on = set(np.linspace(0, n_frames - 1, n_visuals).round().astype(int).tolist())
    assert len(on) == n_visuals
    shapes = [("box", (0.05, 0.04, 0.06)), ("cylinder", (0.02, 0.07)), ("sphere", (0.025,))]
    chain = []
    for f in range(n_frames):
        jt = "fixed" if f % 6 == 5 else ("prismatic" if f % 7 == 3 else "revolute")
        joint = None if f == 0 else (jt, fmt(rng.uniform(-0.02, 0.02, 2).tolist() + [0.06]),
                                     fmt(rng.uniform(-0.6, 0.6, 3)), None if jt == "fixed" else fmt(rng.normal(size=3)))
        vis = []
        if f in on:
            kind, dims = shapes[f % 3]
            vis.append((kind, dims, fmt([0, 0, 0.03]), fmt(rng.uniform(-0.5, 0.5, 3))))
        chain.append((f"f{f}", joint, vis))
    return _write_urdf(dirname, f"chain{n_frames}_{n_visuals}", chain)


def tessellated_box(k):
    """Closed unit cube [-0.5, 0.5]^3, every side a k x k grid of quads (2 k^2 triangles), wound outward."""
    v, f = [], []
    g = np.linspace(-0.5, 0.5, k + 1)
    for axis in range(3):
        for side in (-0.5, 0.5):
            base = len(v)
            for a in g:
                for b in g:
                    p = [0.0, 0.0, 0.0]
                    p[axis], p[(axis + 1) % 3], p[(axis + 2) % 3] = side, a, b
                    v.append(p)
            for i in range(k):
                for j in range(k):
                    c = [base + i * (k + 1) + j, base + (i + 1) * (k + 1) + j, base + (i + 1) * (k + 1) + j + 1,
                         base + i * (k + 1) + j + 1]
                    f += [[c[0], c[1], c[2]], [c[0], c[2], c[3]]]
    return _outward(np.array(v), np.array(f, dtype=np.int32))


def icosahedron():
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                  [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int32)
    return _outward(v / np.linalg.norm(v[0]), f)


def _outward(v, f):
    """Wind every triangle of a convex mesh around the origin so that its normal points away from the origin."""
    tri = v[f]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    flip = (n * tri.mean(1)).sum(1) < 0
    f = f.copy()
    f[flip] = f[flip][:, ::-1]
    return v, f


def write_chain(kind, dirname):
    """(urdf path, end link, primitive_visuals) of a named chain."""
    d = str(dirname)
    if kind == "mixed":
        return (*write_mixed(d), True)
    if kind == "mixed_mesh":
        return (*write_mixed(d, meshes=True), False)
    if kind == "limit32":
        return (*write_long_chain(d, 32, 16), True)
    if kind == "frames33":
        return (*write_long_chain(d, 33, 16, seed=1), True)
    if kind == "links17":
        return (*write_long_chain(d, 24, 17, seed=2), True)
    if kind == "arm":
        return (*workloads.write_arm(d), False)
    assert kind == "prim_arm", kind
    return (*workloads.write_primitive_arm(d), True)


CHAINS = ["mixed", "mixed_mesh", "limit32", "frames33", "links17", "arm", "prim_arm"]
NATIVE = {"mixed": True, "mixed_mesh": True, "limit32": True, "frames33": False, "links17": False, "arm": True,
          "prim_arm": True}


def joint_values(ref, urdf_text, A, seed):
    """fp32 joint values [A, J] (A = 1: [J]): uniform in +-pi (prismatic joints +-PRISMATIC_RANGE m), about 10 % of
    them exactly 0, every configuration 0 all zeros, and continuous joints at +-50 rad in configurations 1 and 2."""
    import xml.etree.ElementTree as ET
    rng = np.random.default_rng(seed)
    movable = [t for t in ref.types if t != "fixed"]
    joints = {j.find("child").get("link"): j.get("type") for j in ET.fromstring(urdf_text).findall("joint")}
    kinds = [joints[n] for n, t in zip(ref.names, ref.types) if t != "fixed"]
    q = rng.uniform(-math.pi, math.pi, (A, len(movable)))
    q[:, [t == "prismatic" for t in movable]] *= PRISMATIC_RANGE / math.pi
    q[rng.random(q.shape) < 0.1] = 0.0
    cont = [k == "continuous" for k in kinds]
    if A > 1:
        q[0] = 0.0
    q[1:2, cont] = 50.0
    q[2:3, cont] = -50.0
    if A == 1:
        q[0, cont] = 50.0
        return q[0].astype(np.float32)
    return q.astype(np.float32)


def build_robot(kind, dirname, dtype=torch.float32, device="cuda"):
    """(RobotSDF, RefRobot, URDF text) of a named chain."""
    import pytorch_volumetric_b200 as pv
    urdf, end, prim = write_chain(kind, dirname)
    text = open(urdf).read()
    chain = pv.build_serial_chain_from_urdf(text, end).to(dtype=dtype, device=device)
    robot = pv.RobotSDF(chain, path_prefix=str(dirname), primitive_visuals=prim)
    return robot, rr.RefRobot(text, end, primitive_visuals=prim, path_prefix=str(dirname)), text


# ------------------------------------------------------------------------------------------ points and comparison
def _half_extents(link):
    if link.kind == "box":
        return np.asarray(link.half)
    if link.kind == "cylinder":
        return np.array([link.radius, link.radius, link.half_length])
    if link.kind == "sphere":
        return np.full(3, link.radius)
    return np.abs(link.vertices).max(0)


def sample_points(ref, M, n, seed):
    """fp32-representable robot-frame points [P, 3] (fp64) in four groups of the fp64 geometry under the
    object->link transforms M [S, A, 4, 4]: n within +-1 cm of a link's surface, n inside a link (each for a random
    link and configuration), n uniform over the box around every link origin, and n // 4 + 1 at 1-3 m."""
    rng = np.random.default_rng(seed)
    S, A = M.shape[:2]
    to_world = rr.rigid_inverse(M)
    shell, inside = [], []
    for s, link in enumerate(ref.links):
        m = 3 * n // S + 8
        q = rng.uniform(-1.3, 1.3, (m, 3)) * _half_extents(link)
        v, g, _, _ = link.evaluate(q)
        on = q - v[:, None] * g                                     # the closest surface point (convex shapes)
        sh = on + rng.uniform(-0.01, 0.01, (m, 1)) * g
        a = rng.integers(0, A, m)
        world = lambda x: np.einsum("mij,mj->mi", to_world[s, a, :3, :3], x) + to_world[s, a, :3, 3]
        shell.append(world(sh))
        inside.append(world(q)[v < 0])
    shell = np.concatenate(shell)
    inside = np.concatenate(inside)
    origins = to_world[..., :3, 3].reshape(-1, 3)
    lo, hi = origins.min(0) - 0.3, origins.max(0) + 0.3
    d = rng.normal(size=(n // 4 + 1, 3))
    far = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(1, 3, (len(d), 1))
    pts = np.concatenate([shell[rng.permutation(len(shell))[:n]], inside[rng.permutation(len(inside))[:n]],
                          rng.uniform(lo, hi, (n, 3)), far])
    return pts.astype(np.float32).astype(np.float64)


def analyse(ref, q, pts):
    """The fp64 truth at every (configuration, point) -- points [P, 3] shared or [A, P, 3] per configuration -- with
    its tolerances: value 'tol' (the largest of the links' value tolerances), gradient 'gtol' of the winning link,
    and 'decided' where fp64 decides the gradient and the link: the best and second-best link values are more than
    2 tol apart, the winning link's rule gap exceeds its value tolerance, and its gradient's conditioning length is
    above 100 x its point bound (off a cylinder's axis, off the surface of an outside rule)."""
    M = ref.object_to_link(q)
    per = ref.evaluate(M, pts)
    rv, rg, rw = ref.compose(per)
    pb, vt = link_tolerances(ref, q, pts)
    take = lambda x: np.take_along_axis(x, rw[None], 0)[0]
    tol = vt.max(0)
    second = np.sort(per["value"], axis=0)[1] if len(ref.links) > 1 else np.full_like(rv, np.inf)
    pbw, vtw, cond = take(pb), take(vt), take(per["cond"])
    why = {"link_tie": second - rv <= 2 * tol, "rule_tie": take(per["gap"]) <= vtw, "conditioning": cond <= 100 * pbw}
    decided = ~(why["link_tie"] | why["rule_tie"] | why["conditioning"])
    # fp32 normalisation, the transform's rotation error carried into the robot frame, and the error of the link's
    # point (or, for a mesh, of its closest point) over the conditioning length
    gtol = 1e-6 + 2 * pbw + 2 * vtw / cond
    return dict(value=rv, grad=rg, which=rw, tol=tol, gtol=gtol, decided=decided,
                skipped={k: int(x.sum()) for k, x in why.items()})


def check(label, truth, v, g, w=None, max_skipped=0.1):
    """Values everywhere, gradients and (with w) the link where decided; prints the observed errors."""
    v, g = np.asarray(v, dtype=np.float64), np.asarray(g, dtype=np.float64)
    err = np.abs(v - truth["value"])
    dec = truth["decided"]
    gerr = np.abs(g - truth["grad"]).max(-1)
    print(f"{label}: max |value error| {err.max():.3g} (bound there {truth['tol'].reshape(-1)[err.argmax()]:.3g}, "
          f"error / bound max {(err / truth['tol']).max():.3f}), gradient error / bound max "
          f"{(gerr / truth['gtol'])[dec].max():.3f}, skipped {int((~dec).sum())} of {dec.size} {truth['skipped']}")
    assert (err <= truth["tol"]).all(), (label, err.max(), np.unravel_index(np.argmax(err / truth["tol"]), err.shape))
    assert (~dec).mean() <= max_skipped, truth["skipped"]
    bad = dec & (gerr > truth["gtol"])
    assert not bad.any(), (label, np.argwhere(bad)[:5], gerr[bad][:5])
    if w is not None:
        bad = dec & (np.asarray(w) != truth["which"])
        assert not bad.any(), (label, np.argwhere(bad)[:5])


def _no_generic(monkeypatch, comp):
    def boom(*a, **k):
        raise AssertionError("generic path taken")
    monkeypatch.setattr(comp, "_generic_query", boom)


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
    _no_generic(monkeypatch, robot.sdf)
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
