"""fp64 reference robot for the CPU and GPU tiers: URDF serial chain -> forward kinematics -> object->link-frame
transforms -> link SDFs from the URDF numbers -> minimum over links.  Numpy only, and independent of the package's
kinematics.py and model_to_sdf.py: it parses the URDF itself and evaluates every link at every (configuration, point).

Conventions (the ones RobotSDF states):
  * the chain runs from the root to the named end link; links off that path are ignored;
  * joint types revolute, continuous (a revolute joint), prismatic and fixed; <origin xyz rpy> with
    R = Rz(yaw) Ry(pitch) Rx(roll); <axis> normalised, (1, 0, 0) when absent;
  * T_child = T_parent @ origin @ motion(q), Rodrigues rotation for revolute joints;
  * the links are the visuals, in frame order and document order within a frame: box, cylinder and sphere visuals
    with primitive_visuals, mesh visuals always; link s of configuration a is posed by (T_frame @ visual_origin)^-1;
  * box: half extents size / 2; cylinder: radius and half length length / 2 along z; sphere: radius; mesh: a closed
    convex OBJ, vertices times `scale`, with the reference's gradient rules (unit vector to / from the closest point,
    the closest face's normal where |d| < 1e-3);
  * the composition takes the first link on ties.
After the reference: the named chains both tiers test (write_chain, build_robot, joint_values), the fp32 tolerance
model (fk_bound, point_bound, link_tolerances), and the sampling and comparison against the reference (sample_points,
analyse, check).
Test infrastructure only."""
import math
import os
import xml.etree.ElementTree as ET

import numpy as np
import torch

import primitive_ref as pr
import workloads

EPS32 = float(np.finfo(np.float32).eps)
U32 = EPS32 / 2          # fp32 unit roundoff
MESH_SHELL = 1e-3          # |d| below which a mesh link's gradient is its closest face's normal


def rpy_matrix(r, p, y):
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return rz @ ry @ rx


def _origin(elem):
    m = np.eye(4)
    o = elem.find("origin") if elem is not None else None
    if o is not None:
        m[:3, :3] = rpy_matrix(*(float(v) for v in o.get("rpy", "0 0 0").split()))
        m[:3, 3] = [float(v) for v in o.get("xyz", "0 0 0").split()]
    return m


def rigid_inverse(m):
    out = np.zeros_like(m)
    rt = np.swapaxes(m[..., :3, :3], -1, -2)
    out[..., :3, :3] = rt
    out[..., :3, 3] = -np.einsum("...ij,...j->...i", rt, m[..., :3, 3])
    out[..., 3, 3] = 1.0
    return out


def read_obj(path):
    """(vertices [V, 3], triangles [F, 3]) of an OBJ with 'v x y z' and triangular 'f a b c' lines."""
    v, f = [], []
    with open(path) as fh:
        for line in fh:
            parts = line.split()
            if parts and parts[0] == "v":
                v.append([float(x) for x in parts[1:4]])
            elif parts and parts[0] == "f":
                f.append([int(x.split("/")[0]) - 1 for x in parts[1:4]])
    return np.array(v, dtype=np.float64), np.array(f, dtype=np.int64)


class Link:
    """One link of the reference robot: a visual of frame `frame`, posed in it by `offset` (4x4)."""

    def __init__(self, frame, offset, kind, **geom):
        self.frame, self.offset, self.kind = frame, offset, kind
        self.__dict__.update(geom)
        if kind == "mesh":
            tri = self.vertices[self.faces]
            n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
            self.normals = n / np.linalg.norm(n, axis=1, keepdims=True)
            self.tri = tri

    @property
    def extent(self):
        """Largest |coordinate| of the shape in its own frame."""
        if self.kind == "box":
            return float(np.linalg.norm(self.half))
        if self.kind == "cylinder":
            return math.hypot(self.radius, self.half_length)
        if self.kind == "sphere":
            return self.radius
        return float(np.linalg.norm(self.vertices, axis=1).max())

    def evaluate(self, q):
        """fp64 (value [n], link-frame gradient [n, 3], gap [n], conditioning length [n]) at link-frame points
        q [n, 3].  The gap is how far q may move before a rule of the shape switches the gradient discontinuously:
        the two largest terms of a box's or cylinder's inside rule, and for a mesh 0 where faces within 1e-7 of the
        closest one give another answer (another closest point, or another normal in the 1e-3 shell) or where |d| is
        within 1e-6 of the shell's edge, +inf otherwise.  The conditioning length c bounds the gradient's
        sensitivity to an error dq of q by dq / c (the outside w / |w|, a cylinder's radial direction, a sphere's
        q / |q|, a mesh's direction to its closest point)."""
        if self.kind == "mesh":
            return self._mesh(q)
        n = len(q)
        inf = np.full(n, np.inf)
        if self.kind == "sphere":
            v, g = pr.sphere_ref(self.radius, q)
            return v, g, inf, np.linalg.norm(q, axis=1)
        if self.kind == "box":
            v, g = pr.box_ref(self.half, q)
            e = np.sort(np.abs(q) - np.asarray(self.half), axis=1)
            gap = np.where(v <= 0, e[:, 2] - e[:, 1], inf)
            return v, g, gap, np.where(v > 0, v, inf)
        v, g = pr.cylinder_ref(self.radius, self.half_length, q)
        rho = np.hypot(q[:, 0], q[:, 1])
        dr, dz = rho - self.radius, np.abs(q[:, 2]) - self.half_length
        gap = np.where(v <= 0, np.abs(dr - dz), inf)
        radial = (v > 0) & (dr > 0) | (v <= 0) & (dr >= dz)
        cond = np.minimum(np.where(v > 0, v, inf), np.where(radial, rho, inf))
        return v, g, gap, cond

    def _mesh(self, q):
        c, d = closest_on_triangles(q, self.tri)                 # [n, F, 3], [n, F]
        k = d.argmin(axis=1)
        rows = np.arange(len(q))
        dist = d[rows, k]
        cbest = c[rows, k]
        inside = np.all(np.einsum("fi,nfi->nf", self.normals, q[:, None, :] - self.tri[None, :, 0]) < 0, axis=1)
        val = np.where(inside, -dist, dist)
        with np.errstate(invalid="ignore", divide="ignore"):
            g = np.where(inside[:, None], cbest - q, q - cbest) / dist[:, None]
        shell = dist < MESH_SHELL
        g = np.where(shell[:, None], self.normals[k], g)
        # how far apart the candidate answers of faces within `tie` of the closest one are: closest points off the
        # shell, face normals in it (coplanar triangles of one side agree on both)
        near = d <= dist[:, None] + 1e-7
        spread_c = np.where(near, np.linalg.norm(c - cbest[:, None], axis=2), 0).max(1)
        spread_n = np.where(near, np.abs(self.normals[None] - self.normals[k][:, None]).max(2), 0).max(1)
        gap = np.where(shell, np.where(spread_n < 1e-9, np.inf, 0.0), np.where(spread_c < 1e-9, np.inf, 0.0))
        # the shell edge: |d| within a hair of 1e-3 may take either rule
        gap = np.where(np.abs(dist - MESH_SHELL) < 1e-6, 0.0, gap)
        return val, g, gap, np.where(shell, np.inf, dist)


def closest_on_triangles(p, tri):
    """Closest points [n, F, 3] and distances [n, F] of points p [n, 3] on triangles tri [F, 3, 3] (fp64; Ericson,
    Real-Time Collision Detection, 5.1.5: Voronoi regions of the vertices, edges and face)."""
    a, b, c = (tri[None, :, i] for i in range(3))
    p = p[:, None, :]
    ab, ac, ap = b - a, c - a, p - a
    dot = lambda x, y: np.einsum("...i,...i->...", x, y)
    d1, d2 = dot(ab, ap), dot(ac, ap)
    bp, cp = p - b, p - c
    d3, d4 = dot(ab, bp), dot(ac, bp)
    d5, d6 = dot(ab, cp), dot(ac, cp)
    va = d3 * d6 - d5 * d4
    vb = d5 * d2 - d1 * d6
    vc = d1 * d4 - d3 * d2
    with np.errstate(invalid="ignore", divide="ignore"):
        denom = 1.0 / (va + vb + vc)
        v_face, w_face = vb * denom, vc * denom
        t_ab = d1 / (d1 - d3)
        t_ac = d2 / (d2 - d6)
        t_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    out = a + ab * v_face[..., None] + ac * w_face[..., None]                      # face interior
    # edges (each only where its Voronoi region applies), then vertices, in the order that makes later regions win
    sel = lambda m, x: np.where(m[..., None], x, out)
    out = sel((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), b + (c - b) * t_bc[..., None])
    out = sel((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + ac * t_ac[..., None])
    out = sel((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + ab * t_ab[..., None])
    out = sel((d6 >= 0) & (d5 <= d6), np.broadcast_to(c, out.shape))
    out = sel((d3 >= 0) & (d4 <= d3), np.broadcast_to(b, out.shape))
    out = sel((d1 <= 0) & (d2 <= 0), np.broadcast_to(a, out.shape))
    return out, np.linalg.norm(p - out, axis=-1)


class RefRobot:
    """The chain of `urdf_text` from its root to `end_link`; mesh files are read from `path_prefix`, and mesh visuals
    are left out when it is None (forward kinematics only)."""

    def __init__(self, urdf_text, end_link, primitive_visuals=True, path_prefix=""):
        robot = ET.fromstring(urdf_text)
        links = {l.get("name"): l for l in robot.findall("link")}
        parent_joint = {j.find("child").get("link"): j for j in robot.findall("joint")}
        path = [end_link]
        while path[-1] in parent_joint:
            path.append(parent_joint[path[-1]].find("parent").get("link"))
        path.reverse()
        self.names = path
        self.origins, self.axes, self.types, self.links = [], [], [], []
        for f, name in enumerate(path):
            if f == 0:
                jt, origin, axis = "fixed", np.eye(4), np.zeros(3)
            else:
                je = parent_joint[name]
                jt = {"continuous": "revolute"}.get(je.get("type"), je.get("type"))
                jt = jt if jt in ("revolute", "prismatic") else "fixed"
                origin = _origin(je)
                ax = je.find("axis")
                axis = np.array([float(v) for v in ax.get("xyz").split()]) if ax is not None else np.array([1., 0, 0])
                axis = axis / np.linalg.norm(axis)
            self.origins.append(origin); self.axes.append(axis); self.types.append(jt)
            for vis in links[name].findall("visual"):
                g = vis.find("geometry")
                off = _origin(vis)
                if g.find("mesh") is not None:
                    if path_prefix is None:
                        continue
                    me = g.find("mesh")
                    v, tris = read_obj(os.path.join(path_prefix, me.get("filename")))
                    scale = np.array([float(s) for s in me.get("scale", "1 1 1").split()])
                    self.links.append(Link(f, off, "mesh", vertices=v * scale, faces=tris))
                elif not primitive_visuals:
                    continue
                elif g.find("box") is not None:
                    size = np.array([float(s) for s in g.find("box").get("size").split()])
                    self.links.append(Link(f, off, "box", half=size / 2))
                elif g.find("cylinder") is not None:
                    c = g.find("cylinder")
                    self.links.append(Link(f, off, "cylinder", radius=float(c.get("radius")),
                                           half_length=float(c.get("length")) / 2))
                elif g.find("sphere") is not None:
                    self.links.append(Link(f, off, "sphere", radius=float(g.find("sphere").get("radius"))))
        self.n_frames = len(path)
        self.n_joints = sum(t != "fixed" for t in self.types)

    def frames(self, q):
        """World-from-frame transforms [A, n_frames, 4, 4] for joint values q [A, n_joints], rounded to fp32 first
        (the kernels' input)."""
        q = np.asarray(q, dtype=np.float32).astype(np.float64).reshape(-1, self.n_joints)
        A = len(q)
        cur = np.broadcast_to(np.eye(4), (A, 4, 4))
        out = np.empty((A, self.n_frames, 4, 4))
        j = 0
        for f in range(self.n_frames):
            cur = cur @ self.origins[f]
            if self.types[f] != "fixed":
                th = q[:, j]
                j += 1
                x, y, z = self.axes[f]
                mot = np.broadcast_to(np.eye(4), (A, 4, 4)).copy()
                if self.types[f] == "revolute":
                    c, s = np.cos(th), np.sin(th)
                    t = 1 - c
                    mot[:, :3, :3] = np.stack([c + x * x * t, x * y * t - z * s, x * z * t + y * s,
                                               y * x * t + z * s, c + y * y * t, y * z * t - x * s,
                                               z * x * t - y * s, z * y * t + x * s, c + z * z * t], 1).reshape(A, 3, 3)
                else:
                    mot[:, :3, 3] = np.outer(th, self.axes[f])
                cur = cur @ mot
            out[:, f] = cur
        return out

    def object_to_link(self, q):
        """[S, A, 4, 4]: the robot frame -> link s frame for every configuration, link-major like
        RobotSDF.object_to_link_frames."""
        fr = self.frames(q)
        return np.stack([rigid_inverse(fr[:, l.frame] @ l.offset) for l in self.links])

    def reach(self, q):
        """[S, A]: the largest |translation| of the frames up to each link's, and of the link itself."""
        fr = self.frames(q)
        t = np.linalg.norm(fr[..., :3, 3], axis=-1)                    # [A, F]
        run = np.maximum.accumulate(t, axis=1)
        return np.stack([np.maximum(run[:, l.frame], np.linalg.norm((fr[:, l.frame] @ l.offset)[:, :3, 3], axis=-1))
                         for l in self.links])

    def evaluate(self, M, pts):
        """Every link at every (configuration, point): M [S, A, 4, 4] from object_to_link, points [P, 3] shared by
        every configuration or [A, P, 3] per configuration.  Returns a dict of [S, A, P] arrays 'value', 'gap',
        'cond' and the robot-frame 'grad' [S, A, P, 3] (see Link.evaluate)."""
        pts = np.asarray(pts, dtype=np.float64)
        S, A = M.shape[:2]
        P = pts.shape[-2]
        own = pts.ndim == 3
        out = {k: np.empty((S, A, P)) for k in ("value", "gap", "cond")}
        out["grad"] = np.empty((S, A, P, 3))
        for s, link in enumerate(self.links):
            R, t = M[s, :, :3, :3], M[s, :, :3, 3]
            q = np.einsum("aij,apj->api" if own else "aij,pj->api", R, pts) + t[:, None]
            if link.kind == "mesh":           # per configuration: the brute-force distance is [P, F] per call
                res = [link.evaluate(q[a]) for a in range(A)]
                v, g, gap, cond = (np.stack([r[i] for r in res]) for i in range(4))
            else:
                v, g, gap, cond = (x.reshape(A, P, *x.shape[1:]) for x in link.evaluate(q.reshape(-1, 3)))
            out["value"][s], out["gap"][s], out["cond"][s] = v, gap, cond
            out["grad"][s] = np.einsum("apj,aji->api", g, R)                    # g @ R: back to the robot frame
        return out

    @staticmethod
    def compose(per_link):
        """(value [A, P], robot-frame gradient [A, P, 3], link [A, P]) of the minimum over links, first on ties."""
        v = per_link["value"]
        w = v.argmin(axis=0)
        take = lambda x: np.take_along_axis(x, w[None, ..., None] if x.ndim == 4 else w[None], 0)[0]
        return take(v), take(per_link["grad"]), w


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
    return robot, RefRobot(text, end, primitive_visuals=prim, path_prefix=str(dirname)), text


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
    to_world = rigid_inverse(M)
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


# every joint type, rotated origins, unnormalised axes, links without visuals and a side branch; mesh visuals only by
# name (no OBJ file is written)
MIXED_URDF = """<robot name="mixed">
  <link name="base"><visual><origin xyz="0 0 0.1" rpy="0.1 -0.2 0.3"/><geometry><mesh filename="a.obj" scale="2 2 2"/></geometry></visual>
                    <visual><geometry><box size="0.1 0.1 0.1"/></geometry></visual></link>
  <link name="l1"/>
  <link name="l2"><visual><origin xyz="0.01 0 0" rpy="0 0 1.5"/><geometry><mesh filename="package://b.obj"/></geometry></visual></link>
  <link name="l3"><visual><geometry><mesh filename="c.obj"/></geometry></visual></link>
  <link name="tool"><visual><geometry><mesh filename="d.obj"/></geometry></visual></link>
  <link name="side"><visual><geometry><mesh filename="e.obj"/></geometry></visual></link>
  <joint name="j_fixed" type="fixed"><parent link="base"/><child link="l1"/><origin xyz="0 0 0.3" rpy="0 0.5 0"/></joint>
  <joint name="j_rev" type="revolute"><parent link="l1"/><child link="l2"/><origin xyz="0.1 0.2 0" rpy="0.3 0 -0.4"/>
         <axis xyz="1 1 0"/><limit lower="-3" upper="3"/></joint>
  <joint name="j_pris" type="prismatic"><parent link="l2"/><child link="l3"/><origin xyz="0 0 0.2"/><axis xyz="0 -1 0.5"/></joint>
  <joint name="j_cont" type="continuous"><parent link="l3"/><child link="tool"/><origin xyz="0.05 0 0" rpy="1.0 0 0"/><axis xyz="0 0 -1"/></joint>
  <joint name="j_side" type="revolute"><parent link="l1"/><child link="side"/><axis xyz="0 0 1"/></joint>
</robot>"""
