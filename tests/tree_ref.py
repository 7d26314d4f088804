"""fp64 reference for kinematic trees, the tree counterpart of robot_ref.RefRobot: its own URDF tree parser (the root
is the one link no joint names as its child; frames in depth-first pre-order, children in the document order of their
joints) and fp64 forward kinematics with explicit parents, T_f = T_parent(f) @ origin_f @ motion_f(q).  Each frame's
joint and visuals are read by robot_ref's parser (the last frame of the serial path to that link), so the link SDFs,
compose, check and the tolerance model are robot_ref's.  The tolerances count, per link, the frames on its root path
and the largest translation on that path: a tree's other branches add no rounding to a link.
The structure rules RobotSDF states, computed from the explicit parents: a joint moves a link when its frame is on the
link's root path, and two links are a self-collision pair when their root paths differ by at least two movable joints.
Test infrastructure only."""
import copy
import xml.etree.ElementTree as ET

import numpy as np

import robot_ref
from robot_ref import RefRobot, point_bound, U32


def _motion(kind, axis, th):
    """[A, 4, 4] fp64 motion of a movable joint at joint values th [A] (Rodrigues for revolute joints)."""
    A = len(th)
    mot = np.broadcast_to(np.eye(4), (A, 4, 4)).copy()
    x, y, z = axis
    if kind == "revolute":
        c, s = np.cos(th), np.sin(th)
        t = 1 - c
        mot[:, :3, :3] = np.stack([c + x * x * t, x * y * t - z * s, x * z * t + y * s,
                                   y * x * t + z * s, c + y * y * t, y * z * t - x * s,
                                   z * x * t - y * s, z * y * t + x * s, c + z * z * t], 1).reshape(A, 3, 3)
    else:
        mot[:, :3, 3] = np.outer(th, axis)
    return mot


class RefTree(RefRobot):
    """The whole tree of `urdf_text`.  names / parents / origins / axes / types per frame in pre-order, links (robot_ref
    Link, `frame` the pre-order index) in frame order and document order within a frame."""

    def __init__(self, urdf_text, primitive_visuals=True, path_prefix=""):
        robot = ET.fromstring(urdf_text)
        names = [l.get("name") for l in robot.findall("link")]
        children = {n: [] for n in names}
        has_parent = set()
        for j in robot.findall("joint"):
            children[j.find("parent").get("link")].append(j.find("child").get("link"))
            has_parent.add(j.find("child").get("link"))
        roots = [n for n in names if n not in has_parent]
        assert len(roots) == 1, roots
        self.names, self.parents = [], []

        def visit(name, parent):
            self.parents.append(parent)
            self.names.append(name)
            here = len(self.names) - 1
            for c in children[name]:
                visit(c, here)

        visit(roots[0], -1)
        self.origins, self.axes, self.types, self.links = [], [], [], []
        for f, name in enumerate(self.names):
            path = RefRobot(urdf_text, name, primitive_visuals=primitive_visuals, path_prefix=path_prefix)
            self.origins.append(path.origins[-1]); self.axes.append(path.axes[-1]); self.types.append(path.types[-1])
            for link in path.links:
                if link.frame == path.n_frames - 1:
                    link = copy.copy(link)
                    link.frame = f
                    self.links.append(link)
        self.n_frames = len(self.names)
        self.n_joints = sum(t != "fixed" for t in self.types)
        self.depth = []                          # frames on each frame's root path, itself included
        for p in self.parents:
            self.depth.append(1 if p < 0 else self.depth[p] + 1)

    def frames(self, q):
        """World-from-frame transforms [A, n_frames, 4, 4] for joint values q [A, n_joints], rounded to fp32 first."""
        q = np.asarray(q, dtype=np.float32).astype(np.float64).reshape(-1, self.n_joints)
        A = len(q)
        out = np.empty((A, self.n_frames, 4, 4))
        j = 0
        for f in range(self.n_frames):
            p = self.parents[f]
            cur = (np.broadcast_to(np.eye(4), (A, 4, 4)) if p < 0 else out[:, p]) @ self.origins[f]
            if self.types[f] != "fixed":
                cur = cur @ _motion(self.types[f], self.axes[f], q[:, j])
                j += 1
            out[:, f] = cur
        return out

    def reach(self, q):
        """[S, A]: the largest |translation| of the frames on each link's root path, and of the link itself."""
        fr = self.frames(q)
        t = np.linalg.norm(fr[..., :3, 3], axis=-1)                    # [A, F]
        run = np.empty_like(t)
        for f, p in enumerate(self.parents):
            run[:, f] = t[:, f] if p < 0 else np.maximum(run[:, p], t[:, f])
        return np.stack([np.maximum(run[:, l.frame], np.linalg.norm((fr[:, l.frame] @ l.offset)[:, :3, 3], axis=-1))
                         for l in self.links])

    def path_frames(self):
        """[S]: frames on each link's root path."""
        return np.array([self.depth[l.frame] for l in self.links])

    # ------------------------------------------------------------------ structure rules
    def root_path(self, f):
        out = []
        while f >= 0:
            out.append(f)
            f = self.parents[f]
        return out

    def moves(self):
        """[J, S] bool: joint j moves link s when j's frame is on s's root path."""
        joints = [f for f, t in enumerate(self.types) if t != "fixed"]
        return np.array([[fj in self.root_path(l.frame) for l in self.links] for fj in joints], dtype=bool).reshape(
            len(joints), len(self.links))

    def pairs(self):
        """[S, S] bool: the movable joints on one link's root path and not the other's number at least two."""
        movable = [{f for f in self.root_path(l.frame) if self.types[f] != "fixed"} for l in self.links]
        return np.array([[len(a ^ b) >= 2 for b in movable] for a in movable], dtype=bool)


# ------------------------------------------------------------------------------------------------ tolerance model
def link_tolerances(ref, q, pts):
    """robot_ref.link_tolerances with each link's frames and reach counted on its root path."""
    reach = ref.reach(q)[..., None]                                            # [S, A, 1]
    nf = ref.path_frames()[:, None, None]
    pnorm = np.linalg.norm(np.asarray(pts, dtype=np.float64), axis=-1)
    pnorm = pnorm[None, :, :] if pnorm.ndim == 2 else pnorm[None, None, :]
    pb = point_bound(nf, reach, pnorm)
    mesh = np.array([5e-6 * max(1.0, l.extent) if l.kind == "mesh" else 0.0 for l in ref.links])[:, None, None]
    return pb, pb + 3 * U32 * (pnorm + reach) + mesh


def analyse(ref, q, pts):
    """robot_ref.analyse with the tree's tolerances."""
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
    gtol = 1e-6 + 2 * pbw + 2 * vtw / cond
    return dict(value=rv, grad=rg, which=rw, tol=tol, gtol=gtol, decided=decided,
                skipped={k: int(x.sum()) for k, x in why.items()})


check = robot_ref.check
sample_points = robot_ref.sample_points


# ------------------------------------------------------------------------------------------------------- the trees
def write_generated(dirname, n_frames, n_visuals, seed=0):
    """A random tree of n_frames frames (each frame's parent drawn from the frames on the current root path, so the
    document order is a pre-order with branches at every depth), every 5th joint fixed and every 7th prismatic, the
    others revolute about random axes; n_visuals box / cylinder / sphere visuals spread over the frames.  Returns the
    URDF path."""
    import os
    rng = np.random.default_rng(seed)
    fmt = lambda v: " ".join(f"{x:.6f}" for x in v)
    on = set(np.linspace(0, n_frames - 1, n_visuals).round().astype(int).tolist())
    assert len(on) == n_visuals
    shapes = ['<box size="0.04 0.03 0.05"/>', '<cylinder radius="0.015" length="0.05"/>', '<sphere radius="0.02"/>']
    links, joints, stack = [], [], []
    for f in range(n_frames):
        vis = (f'<visual><origin xyz="0 0 0.02" rpy="{fmt(rng.uniform(-0.5, 0.5, 3))}"/><geometry>{shapes[f % 3]}'
               f'</geometry></visual>') if f in on else ""
        links.append(f'<link name="f{f}">{vis}</link>')
        if f > 0:
            stack = stack[:int(rng.integers(1, len(stack) + 1))] if rng.random() < 0.3 else stack
            parent = stack[-1]
            jt = "fixed" if f % 5 == 4 else ("prismatic" if f % 7 == 3 else "revolute")
            ax = "" if jt == "fixed" else f'<axis xyz="{fmt(rng.normal(size=3))}"/>'
            joints.append(f'<joint name="j{f}" type="{jt}"><parent link="f{parent}"/><child link="f{f}"/>'
                          f'<origin xyz="{fmt(rng.uniform(-0.03, 0.03, 2).tolist() + [0.05])}" '
                          f'rpy="{fmt(rng.uniform(-0.6, 0.6, 3))}"/>{ax}<limit lower="-3" upper="3"/></joint>')
        stack.append(f)
    os.makedirs(dirname, exist_ok=True)
    path = os.path.join(dirname, f"tree{n_frames}_{n_visuals}.urdf")
    with open(path, "w") as fh:
        fh.write("\n".join([f'<robot name="tree{n_frames}">'] + links + joints + ["</robot>"]))
    return path


TREES = ["mixed", "hand", "hand_mesh", "gripper", "tree64", "tree65"]
NATIVE = {"mixed": True, "hand": True, "hand_mesh": True, "gripper": True, "tree64": True, "tree65": False}


def write_tree(kind, dirname):
    """(urdf path, primitive_visuals) of a named tree: robot_ref's mixed chain with its side branch, the hand (with
    primitives or meshes), the gripper, and generated trees at the native limits (64 frames and 64 links) and one
    frame past them."""
    import workloads
    d = str(dirname)
    if kind == "mixed":
        return robot_ref.write_mixed(d)[0], True
    if kind == "hand":
        return workloads.write_hand(d), True
    if kind == "hand_mesh":
        return workloads.write_hand(d, meshes=True), False
    if kind == "gripper":
        return workloads.write_gripper_tree(d), True
    if kind == "tree64":
        return write_generated(d, 64, 64, seed=3), True
    assert kind == "tree65", kind
    return write_generated(d, 65, 64, seed=4), True


def build_tree(kind, dirname, dtype=None, device="cuda"):
    """(RobotSDF over build_chain_from_urdf, RefTree, URDF text) of a named tree."""
    import torch
    import pytorch_volumetric_b200 as pv
    urdf, prim = write_tree(kind, dirname)
    text = open(urdf).read()
    chain = pv.build_chain_from_urdf(text).to(dtype=dtype or torch.float32, device=device)
    robot = pv.RobotSDF(chain, path_prefix=str(dirname), primitive_visuals=prim)
    return robot, RefTree(text, primitive_visuals=prim, path_prefix=str(dirname)), text
