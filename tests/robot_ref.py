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
Test infrastructure only."""
import math
import os
import xml.etree.ElementTree as ET

import numpy as np

import primitive_ref as pr

EPS32 = float(np.finfo(np.float32).eps)
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
