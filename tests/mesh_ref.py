"""fp64 MeshSDF for the CPU and GPU tiers: ObjectFactory.object_frame_closest_point (reference sdf.py:122-172)
restated in fp64 over the structure the kernels read -- the fp32 vertices and the fp32 face normals
(`obj._face_normals`) -- by brute force over every triangle.  Numpy only; it uses neither the kernels nor
oracle/port.py's fp32 mesh.

Rules (the ones the package states):
  * closest point: Ericson's Voronoi regions (robot_ref.closest_on_triangles); the closest face is the lowest index
    among exact ties;
  * sign: closed meshes (parity) -- odd rounded generalized winding number (any ray gives that parity);
    open meshes (parity) -- crossings of the ray p + t dir, t >= 0, with dir = fmaf(1e-4, hash_normal(seed, i, k),
    ray_far[k]) in fp32 and i the point's index in the call; sign_mode "winding" -- |w| > 1/2;
  * gradient: (closest - p) / |d| inside, (p - closest) / |d| outside, the closest face's normal where |d| < 1e-3;
    the `normal` output is the closest face's normal.

Each point also carries what may legitimately make an fp32 answer differ (see `query`): a closest-feature tie (another
face within the fp32 slack gives another closest point, normal or face index), the edge of the 1e-3 shell, a small
sign margin, and the conditioning length of the gradient.  The bounds below are stated once and pinned against the
host build of the device code by tests/test_mesh_ref_cpu.py.  Test infrastructure only."""
import numpy as np

from helpers import hash_normal
from robot_ref import closest_on_triangles

U = 2.0 ** -24               # fp32 unit roundoff
SHELL = 1e-3                 # |d| below which the gradient is the closest face's normal (sdf.py:162)

# ---- error bounds of the fp32 kernels, in units of U times the point's coordinate scale s = max(|p|_inf, |v|_inf)
# times the shape factor k = max(1, longest edge / smallest altitude) of the closest triangle (the largest over the
# faces tied with it).  The closest point is a handful of fp32 dot products, one division and an affine combination
# of vertices: each coordinate carries O(10) roundings of terms of size s, and the barycentric weights of a sliver
# triangle amplify them by its shape factor.  Its distance inherits that error (1-Lipschitz), plus the rounding of
# the norm.  The gradient (closest - p) / d moves by the closest-point error over the conditioning length
# d, plus the few roundings of the normalisation.  test_mesh_ref_cpu measures the host build against these and
# requires at least a tenth of each bound to be used.
C_CLOSEST = 64               # |closest_fp32 - closest_ref|_inf   <= C_CLOSEST * U * s * k
C_VALUE = 32                 # | |d_fp32| - |d_ref| |              <= C_VALUE * U * s * k
C_GRAD = 128                 # |grad_fp32 - grad_ref|_inf          <= C_GRAD * U * s * k / cond + 8 U
C_TIE = 4 * C_VALUE           # faces whose fp64 distance is within this of the closest one may be the fp32 argmin
C_SIGN = 64                  # |d| below C_SIGN * U * s: the sign test's origin is on the surface up to rounding
C_RAY = 64                   # ray passing within C_RAY * U * (|p| + |v|) of a crossed triangle's edge
WINDING_MARGIN = 0.1         # the GPU's far field is a first-order expansion: ||w| - 1/2| below this is ambiguous


def coord_scale(pts, vscale):
    return np.maximum(np.abs(np.asarray(pts, np.float64)).max(axis=1), vscale)


def value_bound(s):
    return C_VALUE * U * s


def closest_bound(s):
    return C_CLOSEST * U * s


def grad_bound(s, cond):
    with np.errstate(divide="ignore"):
        return C_GRAD * U * s / cond + 8 * U


def _chunk(n_faces):
    return max(1, (1 << 19) // max(n_faces, 1))


class MeshRef:
    """The fp64 query of a pytorch_volumetric_b200 ObjectFactory `obj` (its fp32 vertices, fp32 face normals, ray
    seed, ray_far and closedness)."""

    def __init__(self, obj):
        v32 = obj._mesh.vertices.astype(np.float32).astype(np.float64)
        self.faces = np.asarray(obj._mesh.triangles)
        self.tri = v32[self.faces]                                        # [F, 3, 3]
        edges = np.linalg.norm(self.tri[:, [1, 2, 0]] - self.tri, axis=2)
        area2 = np.linalg.norm(np.cross(self.tri[:, 1] - self.tri[:, 0], self.tri[:, 2] - self.tri[:, 0]), axis=1)
        with np.errstate(divide="ignore"):
            self.shape = np.clip(edges.max(axis=1) ** 2 / area2, 1.0, 1e6)   # longest edge / smallest altitude
        self.fn32 = obj._face_normals.astype(np.float32)
        self.closed = bool(obj.is_closed)
        self.vscale = float(np.abs(v32).max())
        self.ray_far = obj.bounding_box(padding=1.0)[:, 1].astype(np.float32)
        self.ray_seed = obj.ray_seed & 0xFFFFFFFF

    # ---------------------------------------------------------------- unsigned part, once per distinct point
    def geometry(self, pts, winding=None):
        """dict of fp64 'dist', 'closest', 'face' and the tie flags 'tie_face', 'tie_closest', 'tie_normal' and the
        winding number 'w' for points [n, 3] (fp32 values).  Repeated points are evaluated once."""
        p = np.asarray(pts, dtype=np.float32).astype(np.float64)
        uniq, inv = np.unique(p, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        F = len(self.tri)
        out = {k: np.empty(len(uniq)) for k in ("dist", "w", "shape")}
        out["closest"] = np.empty((len(uniq), 3))
        out["face"] = np.empty(len(uniq), np.int64)
        for k in ("tie_face", "tie_closest", "tie_normal"):
            out[k] = np.zeros(len(uniq), bool)
        fn = self.fn32.astype(np.float64)
        m = _chunk(F)
        for s0 in range(0, len(uniq), m):
            q = uniq[s0:s0 + m]
            c, d = closest_on_triangles(q, self.tri)                       # [m, F, 3], [m, F]
            k = d.argmin(axis=1)                                           # first = lowest index on exact ties
            rows = np.arange(len(q))
            dmin, cbest = d[rows, k], c[rows, k]
            cs = coord_scale(q, self.vscale)
            # either face's fp32 distance may be off by its own bound
            near = d <= dmin[:, None] + C_TIE * U * cs[:, None] * (self.shape[None] + self.shape[k][:, None])
            s = cs * np.where(near, self.shape[None], 1.0).max(axis=1)
            near[rows, k] = False
            out["dist"][s0:s0 + m], out["closest"][s0:s0 + m], out["face"][s0:s0 + m] = dmin, cbest, k
            out["shape"][s0:s0 + m] = s / coord_scale(q, self.vscale)
            out["tie_face"][s0:s0 + m] = near.any(axis=1)
            moved = np.abs(c - cbest[:, None]).max(axis=2) > closest_bound(s)[:, None]
            out["tie_closest"][s0:s0 + m] = (near & moved).any(axis=1)
            out["tie_normal"][s0:s0 + m] = (near & (np.abs(fn[None] - fn[k][:, None]).max(axis=2) > 0)).any(axis=1)
            out["w"][s0:s0 + m] = self._winding(q) if (self.closed if winding is None else winding) else np.nan
        return {k: v[inv] for k, v in out.items()}

    def _winding(self, q):
        """Exact generalized winding number (sum of Van Oosterom-Strackee solid angles / 4 pi), fp64."""
        d = self.tri[None] - q[:, None, None, :]                           # [m, F, 3, 3]
        A, B, C = d[:, :, 0], d[:, :, 1], d[:, :, 2]
        la, lb, lc = (np.linalg.norm(x, axis=-1) for x in (A, B, C))
        num = np.einsum("mfi,mfi->mf", A, np.cross(B, C))
        den = la * lb * lc + (A * B).sum(-1) * lc + (B * C).sum(-1) * la + (C * A).sum(-1) * lb
        return (2.0 * np.arctan2(num, den)).sum(axis=1) / (4.0 * np.pi)

    # ---------------------------------------------------------------- the diagonal ray of open meshes
    def ray_dirs(self, idx):
        """The kernel's fp32 ray direction for call indices idx."""
        idx = np.asarray(idx, dtype=np.uint64)
        comp = [np.float32(1e-4) * hash_normal(self.ray_seed, idx, k).astype(np.float64) + float(self.ray_far[k])
                for k in range(3)]
        return np.stack(comp, axis=1).astype(np.float32).astype(np.float64)

    def ray_parity(self, pts, idx):
        """(parity [n] of the crossings of p + t dir_i, t >= 0, with the triangles, fp64 Moller-Trumbore;
        edge margin [n]: the smallest distance of the ray's crossing of a triangle's plane, t >= 0, to that
        triangle's boundary -- where the fp32 test may count a crossing the exact one does not, or miss one)."""
        p = np.asarray(pts, dtype=np.float32).astype(np.float64)
        dirs = self.ray_dirs(idx)
        a, b, c = self.tri[:, 0], self.tri[:, 1], self.tri[:, 2]
        e1, e2 = b - a, c - a
        n = len(p)
        par, margin = np.empty(n, np.int64), np.empty(n)
        m = _chunk(len(self.tri))
        dot = lambda x, y: np.einsum("...i,...i->...", x, y)
        for s0 in range(0, n, m):
            o, dr = p[s0:s0 + m, None, :], dirs[s0:s0 + m, None, :]
            h = np.cross(dr, e2[None])
            det = dot(e1[None], h)
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                sv = o - a[None]
                u = dot(sv, h) * inv
                qv = np.cross(sv, e1[None])
                v = dot(dr, qv) * inv
                t = dot(e2[None], qv) * inv
            hit = (det != 0) & (u >= 0) & (v >= 0) & (u + v <= 1) & (t >= 0)
            par[s0:s0 + m] = hit.sum(axis=1) & 1
            x = o + t[..., None] * dr                                       # the crossing of the plane
            dist_edge = np.full(det.shape, np.inf)
            for pa, pb in ((a, b), (b, c), (c, a)):
                ab = (pb - pa)[None]
                ap = x - pa[None]
                with np.errstate(invalid="ignore"):
                    tt = np.clip(dot(ap, ab) / dot(ab, ab), 0.0, 1.0)
                dist_edge = np.minimum(dist_edge, np.linalg.norm(ap - tt[..., None] * ab, axis=-1))
            dist_edge = np.where((det != 0) & (t >= 0) & np.isfinite(dist_edge), dist_edge, np.inf)
            margin[s0:s0 + m] = dist_edge.min(axis=1)
        return par, margin

    def ray_grazes(self, pts, idx):
        """bool [n]: the kernel's diagonal ray from each point passes within the fp32 slack of a crossed triangle's
        edge.  On a closed mesh the parity does not depend on the ray, and the watertight test counts a crossing at a
        shared edge once; this is the margin of that test's fp32 shear all the same, consulted only where the signs
        differ (it costs a brute-force ray cast per point)."""
        p = np.asarray(pts, dtype=np.float32).astype(np.float64)
        _, edge = self.ray_parity(p, idx)
        return edge <= C_RAY * U * (np.abs(p).max(axis=1) + self.vscale)

    # ---------------------------------------------------------------- the full query
    def query(self, pts, sign="parity", idx=None, geo=None):
        """fp64 outputs and classification for points [n, 3] passed to the kernel as one call (idx: the points'
        indices in that call, default 0..n-1).  sign: "parity" or "winding" (a closed mesh's parity does not depend
        on the ray, so axis_ray_when_closed does not change it; compare's sign_excuse adds the diagonal ray's margin);
        geo: geometry(pts) when already computed.  Returns a dict:
        value, grad, closest, normal, dist, face and the classes tie_face / tie_closest / tie_normal / shell_edge /
        sign_margin (bool: the sign may legitimately differ) and cond (gradient conditioning length)."""
        p = np.asarray(pts, dtype=np.float32).astype(np.float64)
        n = len(p)
        idx = np.arange(n) if idx is None else np.asarray(idx)
        g = self.geometry(p, winding=self.closed or sign == "winding") if geo is None else geo
        dist, cq, face = g["dist"], g["closest"], g["face"]
        s = coord_scale(p, self.vscale) * g["shape"]
        near_surface = dist <= C_SIGN * U * coord_scale(p, self.vscale)
        if sign == "winding":
            inside = np.abs(g["w"]) > 0.5
            sign_margin = (np.abs(np.abs(g["w"]) - 0.5) < WINDING_MARGIN) | near_surface
        elif self.closed:
            inside = (np.rint(g["w"]).astype(np.int64) & 1) == 1
            sign_margin = near_surface
        else:
            inside = self.ray_parity(p, idx)[0] == 1
            sign_margin = near_surface | self.ray_grazes(p, idx)
        with np.errstate(invalid="ignore", divide="ignore"):
            unit = np.where(dist[:, None] > 0, (cq - p) / dist[:, None], 0.0)
        grad = np.where(inside[:, None], unit, -unit)
        value = np.where(inside, -dist, dist)
        normal = self.fn32[face].astype(np.float64)
        shell = dist < SHELL
        grad = np.where(shell[:, None], normal, grad)
        return dict(value=value, grad=grad, closest=cq, normal=normal, dist=dist, face=face, inside=inside,
                    tie_face=g["tie_face"], tie_closest=g["tie_closest"], tie_normal=g["tie_normal"],
                    shell_edge=np.abs(dist - SHELL) <= value_bound(s), sign_margin=sign_margin,
                    cond=np.where(shell, np.inf, dist), scale=s, w=g["w"])


def point_kinds(v, f, n, seed):
    """fp32 point sets [n, 3] around the mesh (v, f): 'uniform' in its box padded by a tenth of the extent; 'shell':
    surface samples moved along the face normal by +-[1e-7, 2e-3], across the 1e-3 shell and the sign change; 'far':
    beyond the box padded by 0.55 extents, which the sort frame (padded by half the extent) clamps to border cells."""
    rng = np.random.default_rng(seed)
    v = np.asarray(v, np.float32).astype(np.float64)
    lo, hi = v.min(0), v.max(0)
    ext = hi - lo
    uniform = rng.uniform(lo - 0.1 * ext, hi + 0.1 * ext, (n, 3))
    tri = v[np.asarray(f)]
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    area = np.linalg.norm(nrm, axis=1)
    k = rng.choice(len(tri), n, p=area / area.sum())
    r1, r2 = np.sqrt(rng.random(n)), rng.random(n)
    x = ((1 - r1)[:, None] * tri[k, 0] + (r1 * (1 - r2))[:, None] * tri[k, 1] + (r1 * r2)[:, None] * tri[k, 2])
    off = 10.0 ** rng.uniform(-7, np.log10(2e-3), n) * rng.choice([-1.0, 1.0], n)
    shell = x + (nrm[k] / area[k, None]) * off[:, None]
    cand = rng.uniform(lo - 2 * ext, hi + 2 * ext, (8 * n, 3))
    cand = cand[((cand < lo - 0.55 * ext) | (cand > hi + 0.55 * ext)).any(axis=1)][:n]
    f32 = lambda a: a.astype(np.float32)
    return {"uniform": f32(uniform), "shell": f32(shell), "far": f32(cand)}


def mixed_points(v, f, n, seed, cluster=0.65, extra=None):
    """[n, 3] fp32: the three point_kinds (and the rows of `extra`) interleaved at random, and `cluster` of the rows
    copies of one shell point (most of the batch in one sort cell).  Returns (points, cluster row mask)."""
    rng = np.random.default_rng(seed + 1)
    m = n - int(cluster * n)
    kinds = point_kinds(v, f, m // 3 + 1, seed)
    extra = np.zeros((0, 3), np.float32) if extra is None else np.asarray(extra, np.float32)[:m // 4]
    rest = np.concatenate([extra, kinds["uniform"], kinds["shell"], kinds["far"]])[:m]
    rest = rest[rng.permutation(len(rest))]
    pts = np.empty((n, 3), np.float32)
    is_cluster = np.zeros(n, bool)
    is_cluster[rng.permutation(n)[:n - m]] = True
    pts[~is_cluster] = rest
    pts[is_cluster] = kinds["shell"][-1]
    return pts, is_cluster


def grazing_points(obj, n, seed, t_range=(0.03, 0.3)):
    """[n, 3] fp32 points whose unjittered ray (direction ray_far) passes exactly through a boundary edge of the open
    mesh of `obj`: whether the kernel's ray crosses the face at that edge is decided by the point's jitter, so an
    answer computed with another point's seed has the wrong sign half of the time."""
    rng = np.random.default_rng(seed)
    f = np.asarray(obj._mesh.triangles)
    v = obj._mesh.vertices.astype(np.float32).astype(np.float64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = np.sort(e, axis=1)
    _, first, count = np.unique(key, axis=0, return_index=True, return_counts=True)
    border = e[first[count == 1]]
    assert len(border), "the mesh is closed"
    k = rng.integers(0, len(border), n)
    b = v[border[k, 0]] + rng.uniform(0.1, 0.9, n)[:, None] * (v[border[k, 1]] - v[border[k, 0]])
    far = obj.bounding_box(padding=1.0)[:, 1].astype(np.float32).astype(np.float64)
    return (b - rng.uniform(*t_range, n)[:, None] * far).astype(np.float32)


def compare(ref, closest, value, grad, normal=None, sub=None, sign_excuse=None):
    """Per-output error / bound of fp32 outputs against `ref` (a MeshRef.query result) on the rows `sub` (default:
    all), and every exceedance sorted into the classes that may explain it.  sign_excuse(rows) -> bool [len(rows)]
    adds a sign margin for the rows whose sign differs (MeshRef.ray_grazes, for a closed mesh queried with the
    diagonal ray).  Returns (report, unexplained) where unexplained is a dict output -> indices (into the rows) that no
    class explains."""
    r = {k: (v[sub] if sub is not None else v) for k, v in ref.items()}
    f = lambda x: None if x is None else np.asarray(x, np.float64)
    closest, value, grad, normal = f(closest), f(value), f(grad), f(normal)
    s = r["scale"]
    tie_c, tie_n, tie_f = r["tie_closest"], r["tie_normal"], r["tie_face"]
    rep, bad = {}, {}
    classes = {"tie": 0, "shell_edge": 0, "sign_margin": 0}

    def account(name, err, bound, excuse_sets):
        over = err > bound
        ok = np.zeros_like(over)
        for cname, m in excuse_sets:
            classes[cname] += int((over & ~ok & m).sum())
            ok |= m
        # error / bound over the points no class covers (<= 1 where the test passes)
        fin = np.isfinite(bound) & (bound > 0) & ~ok
        rep[name] = float((err[fin] / bound[fin]).max()) if fin.any() else 0.0
        rep[name + "_exceed"] = int(over.sum())
        bad[name] = np.nonzero(over & ~ok)[0]

    sign_flip = (value < 0) != r["inside"]
    margin = r["sign_margin"].copy()
    if sign_excuse is not None and (sign_flip & ~margin).any():
        rows = np.nonzero(sign_flip & ~margin)[0]
        margin[rows] = sign_excuse(rows)
    # a point the reference puts on the surface (d = 0) has no sign: both are right
    sign_ok = ~sign_flip | margin | (r["dist"] == 0)
    classes["sign_margin"] += int((sign_flip & margin).sum())
    bad["sign"] = np.nonzero(~sign_ok)[0]
    account("value", np.abs(np.abs(value) - r["dist"]), value_bound(s), [])
    if closest is not None:
        account("closest", np.abs(closest - r["closest"]).max(axis=1), closest_bound(s), [("tie", tie_c)])
    # gradient: the fp32 sign is taken as given (a legitimately flipped sign flips the gradient off the shell)
    gref = np.where((sign_flip & (r["cond"] < np.inf))[:, None], -r["grad"], r["grad"])
    shell_rule = r["cond"] == np.inf
    gtie = np.where(shell_rule, tie_n, tie_c)
    account("grad", np.abs(grad - gref).max(axis=1), grad_bound(s, r["cond"]),
            [("tie", gtie), ("shell_edge", r["shell_edge"])])
    if normal is not None:
        account("normal", np.abs(normal - r["normal"]).max(axis=1), np.zeros(len(s)), [("tie", tie_n)])
    rep["classes"] = classes
    rep["n"] = int(len(s))
    return rep, bad
