"""GPU: scene queries (ComposedSDF.scene_clearance / scene_collision_cost and their query_* slab forms,
RobotSDF.scene_clearance / scene_collision_cost, pvb_composed_query_scene_clearance / _collision_cost).

1. The fused route against the composition route (`_composed_scene_clearance` / `_composed_scene_collision_cost`,
   the definition) on the cached nearest arm, the primitive arm, the arm with MeshSDF links and the 18-visual hand,
   against nearest and trilinear CachedSDF scenes, each primitive and a rotated, translated ComposedSDF of boxes:
   clearance bit for bit (value, link, point; gradient with -0 == +0); cost and twist, and the joint gradient, within
   1e-5 * sum|term| of the fp64 sum of the same fp32 per-point (d, g) -- each route checked to have run.
2. Against fp64, forward kinematics from tests/robot_ref.py (a mixed primitive chain) and tests/tree_ref.py (the
   hand), a primitive scene from tests/primitive_ref.py: clearance within the derived posing and evaluation bound,
   and scene_collision_cost's joint gradient, fused and through the composition route's twists, against fp64 central
   differences of the cost.
3. Determinism: repeated calls and slabs split at odd places are bit-identical; 70 000 configurations stay fused.
4. Locality on the hand: a small object at one finger leaves every joint that moves no contributing link at exactly 0.
5. A MeshSDF and a LOOKUP_GT_SDF scene take the composition route and match the fp64 box they tessellate."""
import math

import numpy as np
import pytest
import torch

import robot_ref as rr
import workloads
from helpers import arm_robot
from primitive_ref import box_ref
from robot_ref import build_robot, joint_values
from tree_ref import build_tree

pytestmark = pytest.mark.gpu

# the tabletop of scripts/c4bench.scene_points: the table slab and six boxes, (lo xyz, size xyz)
BOXES = [(-1.0, -0.5, -0.25, 1.5, 1.0, 0.05), (-0.9, -0.45, -0.2, 0.3, 0.25, 0.35), (0.2, -0.45, -0.2, 0.25, 0.2, 0.6),
         (-0.4, 0.3, -0.2, 0.5, 0.15, 0.25), (0.3, 0.25, -0.2, 0.15, 0.2, 0.9), (-0.95, 0.2, 0.4, 0.2, 0.25, 0.3),
         (-0.3, -0.5, 0.5, 0.6, 0.05, 0.3)]


def _place(rot, t):
    """object -> sub-frame matrix of a sub-SDF whose frame sits at rotation `rot`, origin t."""
    m = np.eye(4)
    m[:3, :3] = rot.T
    m[:3, 3] = -rot.T @ np.asarray(t, dtype=np.float64)
    return m


def tabletop(rotated=False):
    import pytorch_volumetric_b200 as pv
    mats, sdfs = [], []
    g = np.random.default_rng(3)
    for b in BOXES:
        lo, size = np.array(b[:3]), np.array(b[3:])
        rot = np.eye(3)
        if rotated:
            w = g.normal(0, 0.4, 3)
            th = np.linalg.norm(w)
            k = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
            rot = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        sdfs.append(pv.BoxSDF(size))
        mats.append(_place(rot, lo + size / 2))
    return pv.ComposedSDF(sdfs, pv.Transform3d(matrix=torch.tensor(np.stack(mats), dtype=torch.float32).cuda()))


def scenes(tmp_path):
    import pytorch_volumetric_b200 as pv
    table = tabletop()
    out = {"boxes": table, "rotated boxes": tabletop(rotated=True),
           "box": pv.ComposedSDF([pv.BoxSDF([0.3, 0.2, 0.4])], pv.Transform3d(
               matrix=torch.tensor(_place(np.eye(3), (0.1, 0.0, 0.3)), dtype=torch.float32)[None].cuda())),
           "sphere": pv.SphereSDF(0.25), "cylinder": pv.CylinderSDF(0.15, 1.2)}
    rng = [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]]
    for interp in ("nearest", "trilinear"):
        out[f"cached {interp}"] = pv.CachedSDF("table", 0.02, rng, table, device="cuda", clean_cache=True,
                                               cache_path=str(tmp_path / f"table_{interp}.pkl"), interpolation=interp)
    return out


def robot_of(tmp_path, kind):
    import pytorch_volumetric_b200 as pv
    if kind == "hand":
        urdf = workloads.write_hand(str(tmp_path / "hand"))
        robot = pv.RobotSDF(pv.build_chain_from_urdf(open(urdf).read()).to(device="cuda"),
                            path_prefix=str(tmp_path / "hand"), primitive_visuals=True)
        return robot, workloads.tree_configurations(urdf, 200, seed=5).cuda()
    if kind == "mesh":
        urdf, end = workloads.write_primitive_arm(str(tmp_path / "mesh"), mesh_links=workloads.MIXED_ARM_MESH_LINKS)
        robot = pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"),
                            path_prefix=str(tmp_path / "mesh"), primitive_visuals=True)
    else:
        robot = arm_robot(tmp_path, kind)
    g = torch.Generator().manual_seed(7)
    q = torch.cat([workloads.arm_configurations(100, seed=4),
                   ((torch.rand(100, 7, generator=g) * 2 - 1) * math.pi)])
    return robot, q.cuda()


def _spy(monkeypatch, name):
    from pytorch_volumetric_b200 import sdf as S
    calls = []
    orig = getattr(S.ComposedSDF, name)

    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(S.ComposedSDF, name, spy)
    return calls


def _per_point(comp, scene, lp, links):
    """fp64 of the fp32 per-point (d, g) and posed points x of the composition route: [A, n_src, K] each."""
    S, K = lp.shape[:2]
    A = comp._slab(0, None)[1]
    p = lp.detach().float().reshape(-1, 3).contiguous()
    srcs = [i for i in range(S) if links[i]]
    parts = list(comp._scene_chunks(scene, p, K, srcs, 0, A))
    x = torch.cat([c[2] for c in parts]).double()
    return srcs, x, torch.cat([c[3] for c in parts]).double(), torch.cat([c[4] for c in parts]).double()


def _check(monkeypatch, robot, scene, lp, links, m, what):
    comp = robot.sdf
    S = lp.shape[0]
    cl_calls = _spy(monkeypatch, "_composed_scene_clearance")
    cc_calls = _spy(monkeypatch, "_composed_scene_collision_cost")
    fused = comp.query_scene_clearance(scene, lp, links, return_which=True)
    cost = comp.query_scene_collision_cost(scene, lp, m, links)
    assert not cl_calls and not cc_calls, (what, "the fused route fell back")
    K = lp.shape[1]
    mask = [True] * S if links is None else links.tolist()
    p = lp.detach().float().reshape(-1, 3).contiguous()
    A = cost[0].shape[0]
    ref_cl = comp._composed_scene_clearance(scene, p, K, mask, 0, A, True)
    ref_cc = comp._composed_scene_collision_cost(scene, p, K, mask, comp._collision_cost_margin(m), 0, A)
    assert cl_calls and cc_calls
    assert torch.equal(fused[0], ref_cl[0]), (what, "value", float((fused[0] - ref_cl[0]).abs().max()))
    assert torch.equal(fused[2], ref_cl[2]) and torch.equal(fused[3], ref_cl[3]), (what, "link / point")
    assert torch.equal(fused[1], ref_cl[1]), (what, "gradient")       # -0 == +0 in torch.equal
    # cost and twist against the fp64 sum of the per-point (d, g)
    srcs, x, v, g = _per_point(comp, scene, lp, mask)
    m32 = float(np.float32(m))
    h = (m32 - v).clamp_min(0.0)
    tau = torch.cat([g, torch.linalg.cross(x, g, dim=-1)], -1) * (2 * h)[..., None]
    rc = (h * h).sum((-2, -1))
    bc = (h * h).sum((-2, -1))
    rt = torch.zeros(A, S, 6, dtype=torch.float64, device=v.device)
    bt = torch.zeros_like(rt)
    for pos, i in enumerate(srcs):
        rt[:, i] = -tau[:, pos].sum(-2)
        bt[:, i] = tau[:, pos].abs().sum(-2)
    for got, name in ((cost, "fused"), (ref_cc, "composition")):
        assert float(((got[0].double() - rc).abs() - 1e-5 * bc).max()) <= 1e-30, (what, name, "cost")
        assert float(((got[1].double() - rt).abs() - 1e-5 * bt).max()) <= 1e-30, (what, name, "twist")
    jt, moves = robot.joint_twists(), robot.joint_moves_link()
    grad, gref = robot.joint_gradient(cost[1], jt, moves), robot.joint_gradient(rt, jt, moves)
    bound = robot.joint_gradient(bt, jt.abs(), moves)
    assert float(((grad - gref).abs() - 1e-5 * bound).max()) <= 1e-12, (what, "joint gradient")
    assert (cost[0][fused[0] >= m32] == 0).all() and (cost[0][fused[0] < m32 - 1e-6] > 0).all(), what
    return fused, cost


# ---------------------------------------------------------------- 1. fused against the composition route
@pytest.mark.parametrize("kind", ["nearest", "primitive", "mesh", "hand"])
def test_fused_equals_composition(tmp_path, monkeypatch, kind):
    robot, q = robot_of(tmp_path, kind)
    robot.set_joint_configuration(q)
    S = len(robot.sdf.sdfs)
    lp = robot.link_surface_points(num_points=256, seed=1)
    no_base = torch.ones(S, dtype=torch.bool)
    no_base[0] = False
    seen_cost = False
    for name, scene in scenes(tmp_path).items():
        for m in (0.02, 0.1):
            for links in (None, no_base):
                fused, cost = _check(monkeypatch, robot, scene, lp, links, m, (kind, name, m))
                seen_cost |= bool((cost[0] > 0).any())
                if links is not None:
                    assert (fused[2] != 0).all() and not cost[1][:, 0].any()
    assert seen_cost, kind
    # the public forms and RobotSDF
    scene = scenes(tmp_path)["boxes"]
    v, g, i, k = robot.scene_clearance(scene, return_argmin=True)
    assert v.shape == (200,) and g.shape == (200, 3) and i.dtype == torch.int64
    c, jg = robot.scene_collision_cost(scene, 0.1)
    assert c.shape == (200,) and jg.shape == (200, len(robot.joint_names))


# ---------------------------------------------------------------- 2. against fp64
def _posed64(ref, q, lp, n_frames):
    """fp64 posed link points x [A, S, K, 3] from the reference's forward kinematics, and the bound [A, S, K] on
    |x_fp32 - x|: robot_ref.point_bound of the link's frames and reach (two more steps for the fp32 inverse of the
    object->link transform the library poses with)."""
    W = rr.rigid_inverse(ref.object_to_link(q))                                    # [S, A, 4, 4]
    x = np.einsum("sarc,skc->askr", W[..., :3, :3], lp) + W[:, :, None, :3, 3].transpose(1, 0, 2, 3)
    pnorm = np.linalg.norm(lp, axis=-1)[None]                                      # [1, S, K]
    reach = ref.reach(q).T[..., None]                                              # [A, S, 1]
    return x, rr.point_bound(np.asarray(n_frames)[None, :, None] + 2, reach, pnorm)


def _scene_near(x0, rng):
    """A primitive scene about the posed points x0 [S, K, 3] of one configuration: two spheres and a rotated box,
    each centred near a point of another link.  Returns the ComposedSDF on the GPU and its fp64 description
    (kind, size, fp32 object->sub-frame matrix as fp64)."""
    import pytorch_volumetric_b200 as pv
    links = rng.choice(x0.shape[0], 3, replace=False)
    sdfs, mats, specs = [], [], []
    for n, s in enumerate(links):
        c = x0[s, rng.integers(x0.shape[1])] + rng.normal(0.0, 0.015, 3)
        w = rng.normal(0.0, 1.0, 3)
        th = np.linalg.norm(w)
        k = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
        rot = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        m = _place(rot, c).astype(np.float32)
        if n < 2:
            sdfs.append(pv.SphereSDF(0.03))
            specs.append(("sphere", 0.03, m.astype(np.float64)))
        else:
            half = (0.025, 0.035, 0.03)
            sdfs.append(pv.BoxSDF([2 * h for h in half]))
            specs.append(("box", half, m.astype(np.float64)))
        mats.append(m)
    return pv.ComposedSDF(sdfs, pv.Transform3d(matrix=torch.from_numpy(np.stack(mats)).cuda())), specs


def _scene64(specs, x):
    """fp64 scene at points x [N, 3]: value, robot-frame gradient, and whether the point is stable -- its sub-SDF
    wins by more than 1e-3, and its value is smooth there (1e-2 from a sphere's centre; a box point outside by more
    than 1e-3 or inside with its largest axis term ahead of the next by more than 1e-3)."""
    vals, grads, smooth = [], [], []
    for kind, size, m in specs:
        q = x @ m[:3, :3].T + m[:3, 3]
        if kind == "sphere":
            r = np.linalg.norm(q, axis=1)
            v, g, ok = r - np.float32(size), q / np.maximum(r, 1e-300)[:, None], r > 1e-2
        else:
            v, g = box_ref(np.float32(size), q)
            e = np.sort(np.abs(q) - np.float32(size), axis=1)
            ok = (v > 1e-3) | (e[:, 2] - e[:, 1] > 1e-3)
        vals.append(v); grads.append(g @ m[:3, :3]); smooth.append(ok)
    vals, grads, smooth = np.stack(vals), np.stack(grads), np.stack(smooth)
    w = vals.argmin(0)
    take = lambda t: np.take_along_axis(t, w[None, ..., None] if t.ndim == 3 else w[None], 0)[0]
    second = np.sort(vals, axis=0)[1]
    return take(vals), take(grads), take(smooth) & (second - take(vals) > 1e-3)


def _ref_robot(kind, tmp_path):
    """(RobotSDF, fp64 reference, URDF text, frames on each link's root path): robot_ref's mixed primitive chain or
    tree_ref's hand."""
    if kind == "chain":
        robot, ref, text = build_robot("mixed", tmp_path)
        return robot, ref, text, np.array([l.frame + 1 for l in ref.links])
    robot, ref, text = build_tree("hand", tmp_path)
    return robot, ref, text, ref.path_frames()


@pytest.mark.parametrize("kind", ["chain", "hand"])
def test_clearance_and_joint_gradient_against_fp64(tmp_path, monkeypatch, kind):
    """Forward kinematics from robot_ref / tree_ref, a primitive scene from primitive_ref.  Clearance: within the
    posing bound plus the fp32 evaluation of the scene, and the same link and point where the fp64 runner-up is
    beyond twice that.  Joint gradient of scene_collision_cost, on the fused route and through the composition
    route's twists: against fp64 central differences of the cost over stable points (the others moved 100 m out of
    reach), within 5e-4 of sum 2h (|v_j| + |x| |w_j|) as the other cost forms' joint gradients."""
    robot, ref, text, nf = _ref_robot(kind, tmp_path)
    J, S = len(robot.joint_names), len(ref.links)
    qs = joint_values(ref, text, 6, seed=9)
    lp_all = robot.link_surface_points(num_points=400, seed=3).float().cpu().numpy().astype(np.float64)
    K = lp_all.shape[1]
    rng = np.random.default_rng(5)
    m, h = 0.03, 2.0 ** -16
    checked = decided = 0
    for a in range(1, len(qs)):
        q = qs[a:a + 1].astype(np.float64)
        x, xtol = _posed64(ref, q, lp_all, nf)
        scene, specs = _scene_near(x[0], rng)
        v, g, stable = _scene64(specs, x[0].reshape(-1, 3))
        robot.set_joint_configuration(torch.from_numpy(qs[a:a + 1]).cuda())
        # clearance over every point
        t_max = max(np.abs(sp[2][:3, 3]).sum() for sp in specs)
        tol = xtol[0].reshape(-1) + 8 * rr.U32 * (1 + np.abs(x[0]).sum(-1).reshape(-1) + t_max)
        cv, _, cl, ck = (t.cpu().numpy() for t in robot.scene_clearance(
            scene, torch.from_numpy(lp_all.astype(np.float32)).cuda(), return_argmin=True))
        best = int(v.argmin())
        assert abs(float(cv[0]) - v[best]) <= tol.max(), (kind, a, float(cv[0]), v[best], tol.max())
        if np.sort(v)[1] - v[best] > 2 * tol.max():
            assert (int(cl[0]), int(ck[0])) == divmod(best, K), (kind, a)
            decided += 1
        # joint gradient over stable points inside the margin
        keep = (stable & (np.abs(v - m) > 1e-3) & (v < m)).reshape(S, K)
        n = int(keep.sum(1).max())
        if n == 0:
            continue
        lp = np.full((S, n, 3), 100.0)
        for i in range(S):
            lp[i, :int(keep[i].sum())] = lp_all[i][keep[i]]
        lp_t = torch.from_numpy(lp.astype(np.float32)).cuda()
        _, grad = robot.scene_collision_cost(scene, m, lp_t)
        twist_c = robot.sdf._composed_scene_collision_cost(scene, lp_t.reshape(-1, 3), n, [True] * S,
                                                           float(np.float32(m)), 0, 1)[1]
        jt, moves = robot.joint_twists(), robot.joint_moves_link()
        grad_c = robot.joint_gradient(twist_c, jt, moves)
        twists = jt.cpu().numpy()[0]

        def cost64(qq):
            xx, _ = _posed64(ref, qq, lp, nf)
            return (np.maximum(m - _scene64(specs, xx[0].reshape(-1, 3))[0], 0) ** 2).sum()
        x_b = _posed64(ref, q, lp, nf)[0][0].reshape(-1, 3)
        hinge = np.maximum(m - _scene64(specs, x_b)[0], 0)
        for j in range(J):
            qp, qm = q.copy(), q.copy()
            qp[0, j] += h
            qm[0, j] -= h
            fd = (cost64(qp) - cost64(qm)) / (2 * h)
            scale = 2 * (2 * hinge * (np.linalg.norm(twists[j, :3]) + np.linalg.norm(x_b, axis=-1) *
                                      np.linalg.norm(twists[j, 3:]))).sum()
            for got, route in ((grad, "fused"), (grad_c, "composition")):
                gj = float(got.reshape(-1)[j])
                assert abs(gj - fd) <= 5e-4 * scale + 1e-9, (kind, route, a, j, gj, fd, scale)
        checked += int(keep.sum())
    assert checked > 20 and decided >= 1, (checked, decided)


# ---------------------------------------------------------------- 3. determinism, slabs, 70 000 configurations
def test_repeat_slabs_and_70000_configurations(tmp_path, monkeypatch):
    robot, _ = robot_of(tmp_path, "nearest")
    g = torch.Generator().manual_seed(11)
    robot.set_joint_configuration(((torch.rand(70_000, 7, generator=g) * 2 - 1) * math.pi).cuda())
    scene = scenes(tmp_path)["cached nearest"]
    lp = robot.link_surface_points(num_points=64, seed=1)
    calls = (_spy(monkeypatch, "_composed_scene_clearance"), _spy(monkeypatch, "_composed_scene_collision_cost"))
    cl = robot.sdf.query_scene_clearance(scene, lp, return_which=True)
    cc = robot.sdf.query_scene_collision_cost(scene, lp, 0.05)
    assert not any(calls) and (cc[0] > 0).any() and (cc[0] == 0).any()
    for a, b in zip(cl + cc, robot.sdf.query_scene_clearance(scene, lp, return_which=True) +
                    robot.sdf.query_scene_collision_cost(scene, lp, 0.05)):
        assert torch.equal(a, b)
    for begin, count in ((0, 1), (17, 1000), (65_530, 4_470), (69_999, 1), (3, 65_537)):
        s_cl = robot.sdf.query_scene_clearance(scene, lp, cfg_begin=begin, cfg_count=count, return_which=True)
        s_cc = robot.sdf.query_scene_collision_cost(scene, lp, 0.05, cfg_begin=begin, cfg_count=count)
        for a, b in zip(s_cl + s_cc, cl + cc):
            assert torch.equal(a, b[begin:begin + count]), (begin, count)


# ---------------------------------------------------------------- 4. locality on the hand
def test_hand_locality(tmp_path):
    import pytorch_volumetric_b200 as pv
    robot, q = robot_of(tmp_path, "hand")
    robot.set_joint_configuration(q[:1].expand(4, -1).contiguous())
    S = len(robot.sdf.sdfs)
    lp = robot.link_surface_points(num_points=256, seed=1)
    W = robot.sdf._inv_xforms_on(lp.device).reshape(S, -1, 4, 4)[:, 0]
    tip = S - 1                                     # the last link in document order: the thumb's distal segment
    x0 = (W[tip, :3, :3] @ lp[tip, 0].float() + W[tip, :3, 3]).double().cpu().numpy()
    n = x0 / max(np.linalg.norm(x0), 1e-9)
    scene = pv.ComposedSDF([pv.SphereSDF(0.01)], pv.Transform3d(
        matrix=torch.tensor(_place(np.eye(3), x0 + 0.012 * n), dtype=torch.float32)[None].cuda()))
    cost, jg = robot.scene_collision_cost(scene, 0.02)
    twist = robot.sdf.scene_collision_cost(scene, lp, 0.02)[1]
    assert (cost > 0).all()
    hit = twist.abs().sum(-1).sum(0) > 0                                  # links with a contribution
    moves = robot.joint_moves_link().to(hit.device)
    idle = ~(moves & hit[None]).any(1)                                    # joints moving none of them
    assert idle.sum() >= 8, int(idle.sum())                               # the other fingers at least
    assert (jg[:, idle] == 0).all()
    assert (jg[:, ~idle].abs().sum(0) > 0).any()


# ---------------------------------------------------------------- 5. composition-only scenes
def test_mesh_and_lookup_gt_scenes_take_the_composition_route(tmp_path, monkeypatch):
    """A MeshSDF of a tessellated box, and a LOOKUP_GT_SDF CachedSDF over it whose grid lies 2 m away (so every posed
    point takes the ground-truth mesh): both take the composition route, and against the fp64 box
    (primitive_ref.box_ref over the fp32 vertices) with robot_ref's forward kinematics the clearance is within the
    posing bound plus mesh_ref's value and sign bounds, and the cost within sum 2h of that bound."""
    import mesh_ref
    import pytorch_volumetric_b200 as pv
    robot, ref, text = build_robot("prim_arm", tmp_path)
    nf = np.array([l.frame + 1 for l in ref.links])
    size, c = np.array([0.3, 0.2, 0.4]), np.array([0.1, 0.0, 0.3])
    v, f = rr.tessellated_box(4)
    v32 = (v * size + c).astype(np.float32)
    lo, hi = v32.min(0).astype(np.float64), v32.max(0).astype(np.float64)
    obj = pv.MeshObjectFactory("box", mesh=(v32, f))
    mesh = pv.MeshSDF(obj)
    grid = np.array([[2.0, 2.04]] * 3)
    gt = pv.CachedSDF("box", 0.01, grid, mesh, device="cuda", clean_cache=True, cache_path=str(tmp_path / "gt.pkl"),
                      out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    lp = robot.link_surface_points(num_points=64, seed=3).float()
    lp64 = lp.cpu().numpy().astype(np.float64)
    S, K = lp.shape[:2]
    qs = joint_values(ref, text, 60, seed=3).astype(np.float64)
    x, xtol = _posed64(ref, qs, lp64, nf)
    assert (np.abs(x - 2.02).max(-1) > 0.1).all()                                 # no point near the grid
    A = len(qs)
    robot.set_joint_configuration(torch.from_numpy(qs.astype(np.float32)).cuda())
    d64, _ = box_ref((hi - lo) / 2, (x - (lo + hi) / 2).reshape(-1, 3))
    d64 = d64.reshape(A, -1)
    s = np.maximum(np.abs(x).max(-1), np.abs(v32).max()).reshape(A, -1)
    tol = xtol.reshape(A, -1) + mesh_ref.value_bound(4 * s) + 2 * mesh_ref.C_SIGN * mesh_ref.U * s
    m = 0.1
    m32 = float(np.float32(m))
    h = np.maximum(m32 - d64, 0)
    for scene in (mesh, gt):
        calls = (_spy(monkeypatch, "_composed_scene_clearance"), _spy(monkeypatch, "_composed_scene_collision_cost"))
        val = robot.sdf.query_scene_clearance(scene, lp)[0].double().cpu().numpy()
        cost = robot.sdf.query_scene_collision_cost(scene, lp, m)[0].double().cpu().numpy()
        assert all(calls)
        assert (np.abs(val - d64.min(1)) <= tol.max(1)).all(), np.abs(val - d64.min(1)).max()
        assert (np.abs(cost - (h * h).sum(1)) <= (2 * (h + tol) * tol).sum(1) + 1e-12).all()
        assert (cost > 0).any()
