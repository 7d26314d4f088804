"""Kinematic chains and trees (URDF -> batched forward kinematics).

`RobotSDF` (model_to_sdf.py in this package; reference
src/pytorch_volumetric/model_to_sdf.py:16-60, 82-115) is duck-typed on the
`pytorch_kinematics.Chain` surface it uses:
  .dtype .device .to() .get_joint_parameter_names() .get_frame_names(exclude_fixed=False)
  .find_frame(name).link.{name, visuals[i].{geom_type, geom_param, offset}}
  .forward_kinematics(q[b, J], end_only=False) -> {link_name: Transform3d}
A real pk chain can be passed instead; this module provides the same surface
when pytorch_kinematics is not installed.

Two builders:
  build_serial_chain_from_urdf(data, end_link) -> SerialChain: the frames on the path from the root to one end link;
    every other branch is dropped.
  build_chain_from_urdf(data) -> Chain: the whole kinematic tree.  Frames are stored in depth-first pre-order from
    the root (the one link no joint names as its child), children in the document order of their joints; column j
    of q is the j-th movable frame in that order.  Chain.frame_parents() states the structure: RobotSDF's joint mask
    and default self-collision pairs, and the native tree forward kinematics (pvb_fk_tree), read it.
Chain is the supported tree.  A foreign pk tree chain runs the eager queries, but RobotSDF has no parents for it and
treats its frame order as a serial chain in joint_moves_link and self_collision_pairs.

FK: T_child = T_parent @ joint_origin @ motion(q);  revolute: Rodrigues
rotation about the axis; prismatic: translation along the axis; fixed: I.
Joint types: continuous is revolute, every type other than revolute and
prismatic is fixed, a missing <axis> is (1, 0, 0), and <mimic> is ignored.
"""
import ctypes
import xml.etree.ElementTree as ET

import torch

from .transforms import Transform3d, axis_angle_to_matrix, rpy_to_matrix


class Visual:
    def __init__(self, offset, geom_type, geom_param):
        self.offset = offset
        self.geom_type = geom_type
        self.geom_param = geom_param

    def __repr__(self):
        return f"Visual({self.geom_type}, {self.geom_param})"


class Link:
    def __init__(self, name, visuals=()):
        self.name = name
        self.visuals = list(visuals)
        self.offset = None


class Joint:
    def __init__(self, name, joint_type="fixed", axis=(0.0, 0.0, 1.0), origin=None):
        self.name = name
        self.joint_type = joint_type
        a = torch.tensor(axis, dtype=torch.float64)
        self.axis = a / a.norm() if float(a.norm()) > 0 else a
        self.origin = origin if origin is not None else torch.eye(4, dtype=torch.float64)


class Frame:
    def __init__(self, name, link, joint):
        self.name = name
        self.link = link
        self.joint = joint
        self.children = []


def _origin_matrix(elem):
    m = torch.eye(4, dtype=torch.float64)
    o = elem.find("origin") if elem is not None else None
    if o is not None:
        xyz = [float(v) for v in o.get("xyz", "0 0 0").split()]
        rpy = [float(v) for v in o.get("rpy", "0 0 0").split()]
        m[:3, :3] = rpy_to_matrix(*rpy)
        m[:3, 3] = torch.tensor(xyz, dtype=torch.float64)
    return m


def _parse_visual(v):
    g = v.find("geometry")
    geom_type, geom_param = None, None
    if g is not None:
        if g.find("mesh") is not None:
            me = g.find("mesh")
            sc = me.get("scale")
            geom_type = "mesh"
            geom_param = (me.get("filename"), [float(s) for s in sc.split()] if sc is not None else None)
        elif g.find("box") is not None:
            geom_type, geom_param = "box", [float(s) for s in g.find("box").get("size").split()]
        elif g.find("cylinder") is not None:
            c = g.find("cylinder")
            geom_type, geom_param = "cylinder", (float(c.get("radius")), float(c.get("length")))
        elif g.find("sphere") is not None:
            geom_type, geom_param = "sphere", float(g.find("sphere").get("radius"))
    offset = Transform3d(matrix=_origin_matrix(v).to(torch.float32).unsqueeze(0))
    return Visual(offset, geom_type, geom_param)


def _parse_link(elem):
    """A <link> element -> Link with its parsed visuals, in document order."""
    return Link(elem.get("name"), [_parse_visual(v) for v in elem.findall("visual")])


def _parse_joint(je):
    """A <joint> element -> Joint: continuous is revolute, every type but revolute and prismatic is fixed, a missing
    <axis> is (1, 0, 0); <mimic> is ignored."""
    jt = je.get("type")
    jt = "revolute" if jt == "continuous" else jt
    if jt not in ("revolute", "prismatic"):
        jt = "fixed"
    ax = je.find("axis")
    axis = [float(v) for v in ax.get("xyz").split()] if ax is not None else [1.0, 0.0, 0.0]
    return Joint(je.get("name"), jt, axis, _origin_matrix(je))


def _joint_motion(joint, q, dtype, device):
    """[b, 4, 4] motion of a movable joint at joint values q [b]."""
    b = q.shape[0]
    axis = joint.axis.to(dtype=dtype, device=device)
    mot = torch.eye(4, dtype=dtype, device=device).repeat(b, 1, 1)
    if joint.joint_type == "revolute":
        mot[:, :3, :3] = axis_angle_to_matrix(axis.expand(b, 3), q)
    else:
        mot[:, :3, 3] = axis.unsqueeze(0) * q.unsqueeze(1)
    return mot


class _Frames:
    """What SerialChain and Chain share: frames in order, the frame and joint names, device and dtype, and the
    pvb_fk_frame packing of the native forward kinematics."""

    def __init__(self, frames, dtype=torch.float32, device="cpu"):
        self._frames = list(frames)
        self.dtype = dtype
        self.device = torch.device(device)
        self._origins = None

    def to(self, dtype=None, device=None):
        if dtype is not None:
            self.dtype = dtype
        if device is not None:
            self.device = torch.device(device)
        self._origins = None
        return self

    @property
    def n_joints(self):
        return len(self.get_joint_parameter_names())

    def get_joint_parameter_names(self, exclude_fixed=True):
        return [f.joint.name for f in self._frames if not (exclude_fixed and f.joint.joint_type == "fixed")]

    def get_frame_names(self, exclude_fixed=True):
        return [f.name for f in self._frames if not (exclude_fixed and f.joint.joint_type == "fixed")]

    def find_frame(self, name):
        for f in self._frames:
            if f.name == name:
                return f
        return None

    def _pack_fk_frames(self):
        """The frames as the pvb_fk_frame array of include/pvb.h: joint origins, unit axes, joint types and the column
        of q each movable joint reads.  fp32, like forward_kinematics on a float32 chain."""
        from . import _native as nat
        arr = (nat.FkFrame * len(self._frames))()
        j = 0
        for i, f in enumerate(self._frames):
            o = f.joint.origin.to(torch.float32)
            for r in range(3):
                for c in range(4):
                    arr[i].origin[4 * r + c] = float(o[r, c])
            ax = f.joint.axis.to(torch.float32)
            for k in range(3):
                arr[i].axis[k] = float(ax[k])
            jt = f.joint.joint_type
            arr[i].joint_type = {"revolute": nat.FK_REVOLUTE, "prismatic": nat.FK_PRISMATIC}.get(jt, nat.FK_FIXED)
            arr[i].q_index = j if jt != "fixed" else -1
            if jt != "fixed":
                j += 1
        return arr

    def _joint_values(self, th):
        th = torch.as_tensor(th, dtype=self.dtype, device=self.device)
        if th.dim() == 1:
            th = th.unsqueeze(0)
        if th.shape[-1] != self.n_joints:
            raise ValueError(f"expected {self.n_joints} joint values, got {th.shape[-1]}")
        if self._origins is None:
            self._origins = [f.joint.origin.to(dtype=self.dtype, device=self.device) for f in self._frames]
        return th


class SerialChain(_Frames):
    def native_fk_frames(self):
        """The chain as the pvb_fk_frame array pvb_fk_serial takes (include/pvb.h), or None past its frame limit."""
        from . import _native as nat
        if len(self._frames) > nat.FK_MAX_FRAMES:
            return None
        return self._pack_fk_frames()

    def forward_kinematics(self, th, end_only=True):
        th = self._joint_values(th)
        b = th.shape[0]
        cur = torch.eye(4, dtype=self.dtype, device=self.device).expand(b, 4, 4)
        out = {}
        j = 0
        for f, origin in zip(self._frames, self._origins):
            cur = cur @ origin
            if f.joint.joint_type != "fixed":
                cur = cur @ _joint_motion(f.joint, th[:, j], self.dtype, self.device)
                j += 1
            out[f.link.name] = Transform3d(matrix=cur)
        if end_only:
            return out[self._frames[-1].link.name]
        return out


class Chain(_Frames):
    """A kinematic tree: frames in depth-first pre-order from the root, each child after its parent
    (build_chain_from_urdf)."""

    def __init__(self, frames, parents, dtype=torch.float32, device="cpu"):
        super().__init__(frames, dtype, device)
        self._parents = list(parents)
        for f, p in zip(self._frames, self._parents):
            if p >= 0:
                self._frames[p].children.append(f)

    def frame_parents(self):
        """The parent index of every frame, in get_frame_names(exclude_fixed=False) order; -1 for the root."""
        return list(self._parents)

    def native_fk_frames(self):
        """(pvb_fk_frame array, int32 parents array) as pvb_fk_tree takes them (include/pvb.h), or None past its
        frame limit."""
        from . import _native as nat
        if len(self._frames) > nat.FK_TREE_MAX_FRAMES:
            return None
        return self._pack_fk_frames(), (ctypes.c_int32 * len(self._parents))(*self._parents)

    def forward_kinematics(self, th, end_only=False):
        """{link name: Transform3d} of every frame: T_parent @ origin @ motion(q), the products SerialChain takes, so a
        serial tree gives SerialChain's bits."""
        if end_only:
            raise ValueError("a kinematic tree has no single end link: call forward_kinematics with end_only=False")
        th = self._joint_values(th)
        b = th.shape[0]
        root = torch.eye(4, dtype=self.dtype, device=self.device).expand(b, 4, 4)
        poses, out = [], {}
        j = 0
        for f, origin, p in zip(self._frames, self._origins, self._parents):
            cur = (root if p < 0 else poses[p]) @ origin
            if f.joint.joint_type != "fixed":
                cur = cur @ _joint_motion(f.joint, th[:, j], self.dtype, self.device)
                j += 1
            poses.append(cur)
            out[f.link.name] = Transform3d(matrix=cur)
        return out


def build_serial_chain_from_urdf(data, end_link_name, root_link_name=""):
    """Parse a URDF string and keep the frames on the path root -> end link."""
    robot = ET.fromstring(data)
    links = {l.get("name"): l for l in robot.findall("link")}
    if end_link_name not in links:
        raise ValueError(f"link {end_link_name} not found in URDF")
    parent_joint = {j.find("child").get("link"): j for j in robot.findall("joint")}
    path = [end_link_name]
    while path[-1] in parent_joint and path[-1] != root_link_name:
        path.append(parent_joint[path[-1]].find("parent").get("link"))
    path.reverse()
    frames = []
    for k, name in enumerate(path):
        joint = Joint(None) if k == 0 else _parse_joint(parent_joint[name])
        frames.append(Frame(name, _parse_link(links[name]), joint))
    return SerialChain(frames)


def build_chain_from_urdf(data):
    """Parse a URDF string into the whole kinematic tree (Chain).  Raises ValueError when there is not exactly one
    root, when a link is the child of two joints, when a joint names a link that does not exist, or when a link cannot
    be reached from the root."""
    robot = ET.fromstring(data)
    links = {l.get("name"): l for l in robot.findall("link")}
    parent_joint, children = {}, {name: [] for name in links}
    for je in robot.findall("joint"):
        parent, child = je.find("parent").get("link"), je.find("child").get("link")
        for name in (parent, child):
            if name not in links:
                raise ValueError(f"joint {je.get('name')} names link {name}, which is not in the URDF")
        if child in parent_joint:
            raise ValueError(f"link {child} is the child of two joints ({parent_joint[child].get('name')} and "
                             f"{je.get('name')})")
        parent_joint[child] = je
        children[parent].append(child)
    roots = [name for name in links if name not in parent_joint]
    if len(roots) != 1:
        raise ValueError(f"a kinematic tree needs exactly one root link (one no joint names as its child), found "
                         f"{roots if roots else 'none'}")
    frames, parents, stack = [], [], [(roots[0], -1)]
    while stack:                                  # depth-first pre-order, children in joint document order
        name, parent = stack.pop()
        joint = Joint(None) if parent < 0 else _parse_joint(parent_joint[name])
        parents.append(parent)
        frames.append(Frame(name, _parse_link(links[name]), joint))
        stack.extend((c, len(frames) - 1) for c in reversed(children[name]))
    if len(frames) != len(links):
        missing = sorted(set(links) - {f.name for f in frames})
        raise ValueError(f"links {missing} cannot be reached from the root link {roots[0]}")
    return Chain(frames, parents)
