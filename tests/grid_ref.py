"""fp64 reference of the voxel-grid lookups for the CPU and GPU tiers: CachedSDF (reference sdf.py:535-571) with the
nearest-voxel rule and with the trilinear extension, and the GridView index rule of the VoxelGrid containers.

Inputs are what the kernels read: the fp32 value / gradient tables, the ranges as given (their dtype decides the index
arithmetic) and fp32 points; fp64 points are rounded to fp32 first, as the library does.

Rules:
  * nearest key: round((p - lo) / res), half to even, in the dtype torch infers for the range -- fp64 for numpy
    ranges, fp32 for Python floats (TorchMultidimView.ensure_index_key); in range when all(lo <= p <= hi) against the
    range in that dtype; in-range value and gradient are the table entries at the key;
  * bounding-box rule outside the range (sdf.py:555-571): the signed per-axis overshoot of the fp32 box, its fp64
    norm and direction (a NaN coordinate overshoots by 0, like the reference's `below > 0` test);
  * trilinear: oracle.port.trilinear_lookup_port (the interpolant and its analytic gradient), evaluated at the point
    clamped into the range (the kernel clamps the cell fraction to [0, 1]);
  * VoxelGrid / GridView: the nearest key per axis, valid when every index lies in [0, n).

Error bounds of the fp32 kernels, stated once (U = 2^-24, fp32 unit roundoff) and pinned by tests/test_grid_ref_cpu.py,
which requires the host build of the device code to use at least a tenth of each:
  * in-range nearest value and gradient: exact (a gather at the exact key);
  * bounding-box value: C_BOX * U * |v|; gradient: C_BOX * U per component (one rounding per overshoot, three for
    the sum of squares, ~2 ulp for the reciprocal square root and its Newton step);
  * trilinear value: sum_a slope_a * e_a + C_INTERP * U * M, with slope_a the largest corner difference of the cell
    along axis a, M the largest |corner value| and e_a the fp32 error of the cell coordinate
    u_a = (p_a - lo_a) * inv_res_a in cells: C_U * U * (|lo_a| / res_a + |u_a|) (rounding lo to fp32, the
    subtraction, the rounding of 1 / res and the product);
  * trilinear gradient along a: (C_TGRAD * U * M + sum_{b != a} D_ab * e_b) / res_a + C_BOX * U * |g_a|, with D_ab
    the largest mixed second difference of the cell in (a, b).  Off cell faces only: within e_b of an interior face
    normal to b, the fp32 cell coordinate may land in either cell, and either cell's gradient is accepted there (the
    classes of `compare_trilinear`).
Test infrastructure only."""
import numpy as np
import torch

from oracle import port

U = 2.0 ** -24
C_BOX = 8
C_U = 4
C_INTERP = 16
C_TGRAD = 48


def _range_is_fp32(ranges):
    return torch.tensor([min(r) for r in ranges]).dtype == torch.float32


def as_points(p):
    """fp32 points as the kernels read them, widened to fp64."""
    p = p.detach().cpu().numpy() if torch.is_tensor(p) else np.asarray(p)
    return np.asarray(p, dtype=np.float32).reshape(-1, p.shape[-1]).astype(np.float64)


def index_rule(lo, hi, n, fp32, p):
    """Per-axis nearest index round((p - lo) / res) (half to even) in the range's dtype, unclamped, as fp64; NaN for
    NaN points.  lo, hi, n: per-axis arrays; p [m, d] fp64 holding fp32 values."""
    lo, hi, n = np.asarray(lo, np.float64), np.asarray(hi, np.float64), np.asarray(n)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if fp32:
            lo32, hi32 = lo.astype(np.float32), hi.astype(np.float32)
            res32 = ((hi32 - lo32) / (n - 1).astype(np.float32)).astype(np.float32)
            return np.rint(((p.astype(np.float32) - lo32).astype(np.float32) / res32).astype(np.float32)).astype(
                np.float64)
        return np.rint((p - lo) / ((hi - lo) / (n - 1)))


def voxel_index(ranges, shape, p):
    """GridView / VoxelGrid flat index of points p [m, d] (-1 where an index leaves [0, n)), d = 1..3."""
    lo = np.array([float(min(r)) for r in ranges]); hi = np.array([float(max(r)) for r in ranges])
    n = np.array(shape)
    k = index_rule(lo, hi, n, _range_is_fp32(ranges), as_points(p))
    ok = np.all((k >= 0) & (k < n), axis=1)
    flat = np.zeros(len(k), np.int64)
    for a in range(len(n)):
        flat = flat * n[a] + np.where(ok, k[:, a], 0).astype(np.int64)
    return np.where(ok, flat, -1)


def box_rule(bb32, p):
    """(value [m], gradient [m, 3]) of the bounding-box rule, fp64 over the fp32 box; 0 / NaN gradient at zero
    overshoot, like the reference."""
    with np.errstate(invalid="ignore"):
        below = bb32[:, 0] - p
        above = p - bb32[:, 1]
        below_on, above_on = below > 0, above > 0
        delta = np.where(below_on, below, 0.0) + np.where(above_on, above, 0.0)
        delta = np.where(below_on, -delta, delta)
        dist = np.sqrt((delta ** 2).sum(axis=1))
        with np.errstate(divide="ignore"):
            grad = delta / dist[:, None]
    return dist, grad


class Grid:
    """fp64 reference of one CachedSDF: table_val (nx, ny, nz), table_grad (nx*ny*nz, 3), ranges (as the CachedSDF
    holds them), bb (3, 2) box of the out-of-range rule."""

    def __init__(self, table_val, table_grad, ranges, bb):
        tv = table_val.detach().cpu().numpy() if torch.is_tensor(table_val) else np.asarray(table_val)
        tg = table_grad.detach().cpu().numpy() if torch.is_tensor(table_grad) else np.asarray(table_grad)
        self.val32 = np.asarray(tv, np.float32)
        self.shape = np.array(self.val32.shape)
        self.val = self.val32.astype(np.float64)
        self.grad = np.asarray(tg, np.float32).reshape(-1, 3).astype(np.float64)
        self.ranges = ranges
        self.fp32 = _range_is_fp32(ranges)
        self.lo64 = np.array([float(min(r)) for r in ranges]); self.hi64 = np.array([float(max(r)) for r in ranges])
        t = np.float32 if self.fp32 else np.float64
        self.lo = self.lo64.astype(t).astype(np.float64); self.hi = self.hi64.astype(t).astype(np.float64)
        self.res = (self.hi64 - self.lo64) / np.maximum(self.shape - 1, 1)
        bb = bb.detach().cpu().numpy() if torch.is_tensor(bb) else np.asarray(bb)
        self.bb32 = np.asarray(bb, np.float32).astype(np.float64)

    @classmethod
    def of(cls, cached):
        """The reference of a pytorch_volumetric_b200.CachedSDF (the tables the kernels read)."""
        return cls(cached.voxels.raw_data.reshape(tuple(cached.voxels.shape)), cached.voxels_grad, cached.ranges,
                   cached.bb)

    # ------------------------------------------------------------ nearest
    def in_range(self, p):
        with np.errstate(invalid="ignore"):
            return np.all((p >= self.lo) & (p <= self.hi), axis=1)

    def keys(self, p):
        """(ravelled key [m], -1 out of range; per-axis index [m, 3], clamped)."""
        p = as_points(p)
        inb = self.in_range(p)
        k = index_rule(self.lo64, self.hi64, self.shape, self.fp32, p)
        k = np.clip(np.where(inb[:, None], k, 0), 0, self.shape - 1).astype(np.int64)
        flat = (k[:, 0] * self.shape[1] + k[:, 1]) * self.shape[2] + k[:, 2]
        return np.where(inb, flat, -1), k

    def nearest(self, p):
        """dict of key, inb, value, grad (fp64) and the bounds vbound [m], gbound [m, 3] (0 in range)."""
        p = as_points(p)
        key, _ = self.keys(p)
        inb = key >= 0
        bv, bg = box_rule(self.bb32, p)
        safe = np.where(inb, key, 0)
        value = np.where(inb, self.val.reshape(-1)[safe], bv)
        grad = np.where(inb[:, None], self.grad[safe], bg)
        vb = np.where(inb, 0.0, C_BOX * U * np.abs(bv))
        gb = np.where(inb[:, None], 0.0, C_BOX * U)
        return dict(key=key, inb=inb, value=value, grad=grad, vbound=vb, gbound=gb * np.ones((1, 3)))

    # ------------------------------------------------------------ trilinear
    def _port(self, p):
        v, g, _ = port.trilinear_lookup_port(torch.from_numpy(self.val), self.ranges, self.bb32, torch.from_numpy(p))
        return v.numpy(), g.numpy()

    def trilinear(self, p, band=0.0):
        """dict of inb, value, grad, bounds vbound [m] / gbound [m, 3], the cell-coordinate error e [m, 3], the
        distance in cells to the nearest interior cell face per axis `face` [m, 3] (inf where there is none), and
        `alt` [8, m, 3]: the gradient of every cell touching the faces within max(2 e, band) of the point (NaN for
        points off every face)."""
        p = as_points(p)
        m = len(p)
        inb = self.in_range(p)
        pc = np.where(inb[:, None], np.clip(p, self.lo64, self.hi64), self.lo64)
        value, grad = self._port(pc)
        n = self.shape
        u = (pc - self.lo64) / self.res
        c0 = np.clip(np.floor(u).astype(np.int64), 0, np.maximum(n - 2, 0))
        step = (n > 1).astype(np.int64)
        corner = np.empty((m, 2, 2, 2))
        for i in range(2):
            for j in range(2):
                for k in range(2):
                    corner[:, i, j, k] = self.val[c0[:, 0] + i * step[0], c0[:, 1] + j * step[1], c0[:, 2] + k * step[2]]
        M = np.abs(corner).reshape(m, 8).max(axis=1)
        d1 = [np.abs(np.diff(corner, axis=1 + a)).reshape(m, -1).max(axis=1) for a in range(3)]
        mixed = {}
        for a in range(3):
            for b in range(a + 1, 3):
                dd = np.diff(np.diff(corner, axis=1 + a), axis=1 + b)
                mixed[(a, b)] = mixed[(b, a)] = np.abs(dd).reshape(m, -1).max(axis=1)
        e = C_U * U * (np.abs(self.lo64)[None] / self.res + np.abs(u))
        vb = sum(d1[a] * e[:, a] for a in range(3)) + C_INTERP * U * M
        gb = np.stack([(C_TGRAD * U * M + sum(mixed[(a, b)] * e[:, b] for b in range(3) if b != a)) / self.res[a]
                       for a in range(3)], axis=1) + C_BOX * U * np.abs(grad)
        r = np.rint(u)
        face = np.where((r >= 1) & (r <= n - 2), np.abs(u - r), np.inf)
        # the gradient in each cell around the faces the point lies on (a lattice edge or node touches 4 or 8 cells)
        on_face = face <= np.maximum(2 * e, band) + 1e-9
        near = np.nonzero(on_face.any(axis=1))[0]
        alt = np.full((8, m, 3), np.nan)
        for s in range(8):
            side = np.array([1e-9 if s >> b & 1 else -1e-9 for b in range(3)])
            uu = np.where(on_face[near], r[near] + side, u[near])
            alt[s, near] = self._port(self.lo64 + uu * self.res)[1]
        bv, bg = box_rule(self.bb32, p)
        value = np.where(inb, value, bv)
        grad = np.where(inb[:, None], grad, bg)
        vb = np.where(inb, vb, C_BOX * U * np.abs(bv))
        gb = np.where(inb[:, None], gb, C_BOX * U)
        return dict(inb=inb, value=value, grad=grad, vbound=vb, gbound=gb, e=e, face=face, alt=alt, u=u)


# ---------------------------------------------------------------- comparison
def _nan_equal(a, b):
    return (a == b) | (np.isnan(a) & np.isnan(b))


def compare_nearest(ref, val, grad, key=None):
    """Largest error / bound of value and gradient (in-range points: bit-exact; NaN where the reference is NaN) and the
    indices that break them.  Returns (report, bad)."""
    val = np.asarray(val, np.float64); grad = np.asarray(grad, np.float64).reshape(-1, 3)
    inb = ref["inb"]
    bad = {}
    bad["key"] = np.nonzero(key != ref["key"])[0] if key is not None else np.zeros(0, np.int64)
    bad["exact"] = np.nonzero(inb & ~(_nan_equal(val, ref["value"]) & _nan_equal(grad, ref["grad"]).all(1)))[0]
    rv, rg = ref["value"], ref["grad"]
    with np.errstate(invalid="ignore", divide="ignore"):
        ev = np.where(_nan_equal(val, rv), 0.0, np.abs(val - rv) / ref["vbound"])
        eg = np.where(_nan_equal(grad, rg), 0.0, np.abs(grad - rg) / ref["gbound"]).max(axis=1)
    ev, eg = np.where(inb, 0.0, ev), np.where(inb, 0.0, eg)
    bad["value"] = np.nonzero(~(ev <= 1))[0]
    bad["grad"] = np.nonzero(~(eg <= 1))[0]
    rep = dict(n=len(val), inb=int(inb.sum()), value=float(np.max(ev, initial=0)), grad=float(np.max(eg, initial=0)))
    return rep, bad


def compare_trilinear(ref, val, grad):
    """Value within vbound everywhere; each gradient component within gbound, or -- class 'face' -- within gbound of
    the gradient of another cell touching a cell face the point lies within the cell-coordinate error of.
    Returns (report, bad)."""
    val = np.asarray(val, np.float64); grad = np.asarray(grad, np.float64).reshape(-1, 3)
    rv, rg = ref["value"], ref["grad"]
    with np.errstate(invalid="ignore", divide="ignore"):
        ev = np.where(_nan_equal(val, rv), 0.0, np.abs(val - rv) / ref["vbound"])
        eg = np.where(_nan_equal(grad, rg), 0.0, np.abs(grad - rg) / ref["gbound"])
    ok = eg <= 1
    face = np.zeros(len(val), bool)
    for alt in ref["alt"]:
        with np.errstate(invalid="ignore"):
            e_alt = np.abs(grad - alt) / ref["gbound"]
        face |= ~ok.all(axis=1) & (e_alt <= 1).all(axis=1) & ref["inb"]
    on_face = (ref["face"] <= 2 * ref["e"] + 1e-9).any(axis=1) & ref["inb"]
    bad = {"value": np.nonzero(~(ev <= 1))[0], "grad": np.nonzero(~((eg.max(axis=1) <= 1) | face))[0]}
    # the reported ratio is that of the points off every cell face, where only rounding separates the two
    rep = dict(n=len(val), value=float(np.max(ev, initial=0)),
               grad=float(np.max(np.where(on_face, 0.0, eg.max(axis=1)), initial=0)), face=int(face.sum()))
    return rep, bad


# ---------------------------------------------------------------- a dyadic table
DYADIC_RES = 1.0 / 32
DYADIC_RANGE = [(-1.0, 1.0), (-0.5, 0.5), (-0.03125, 0.03125)]     # 65 x 33 x 3 nodes: a 2-cell z axis
DYADIC_RADIUS = 0.75                                                 # SphereSDF whose box the out-of-range rule uses


def dyadic_ranges(fp32_range):
    """The snapped ranges of the dyadic table: numpy scalars (fp64 index arithmetic) or Python floats (fp32)."""
    conv = float if fp32_range else np.float64
    return [(conv(a), conv(b)) for a, b in DYADIC_RANGE]


def dyadic_table():
    """(val [65, 33, 3] fp32, grad [N, 3] fp32) of a smooth function whose slope differs on every axis, on a range
    whose nodes and half-way points are exact in fp32."""
    ax = [np.arange(a, b + DYADIC_RES / 2, DYADIC_RES) for a, b in DYADIC_RANGE]
    x, y, z = np.meshgrid(*ax, indexing="ij")
    val = np.sin(3 * x) + 0.5 * y ** 2 - 2.5 * z + 3 * x * y * z
    grad = np.stack([3 * np.cos(3 * x) + 3 * y * z, y + 3 * x * z, -2.5 + 3 * x * y], axis=-1)
    return val.astype(np.float32), grad.reshape(-1, 3).astype(np.float32)


# ---------------------------------------------------------------- point sets
def _near(x, ulps):
    out = [x]
    up, down = x.copy(), x.copy()
    for _ in range(ulps):
        up = np.nextafter(up, np.float32(np.inf)); down = np.nextafter(down, np.float32(-np.inf))
        out += [up.copy(), down.copy()]
    return np.concatenate(out)


def point_sets(lo, hi, n, seed=0, n_uniform=20000, ulps=4):
    """dict name -> fp32 points [m, 3] for a grid over [lo, hi] with n nodes per axis:
    uniform, boundary (+-1..ulps ulps around every cell boundary on each axis, the other axes uniform), half (exact
    half-way points), ends (the fp32 neighbours of both range ends on each axis), nodes (lattice nodes, including the
    upper face), outside (10^-6 .. 10^3 beyond the range on one or more axes) and nan."""
    lo, hi, n = np.asarray(lo, np.float64), np.asarray(hi, np.float64), np.asarray(n)
    rng = np.random.default_rng(seed)
    res = (hi - lo) / (n - 1)

    def fill(axis_vals, a):
        q = rng.uniform(lo, hi, (len(axis_vals), 3))
        q[:, a] = axis_vals
        return q.astype(np.float32)

    out = {"uniform": rng.uniform(lo, hi, (n_uniform, 3)).astype(np.float32)}
    half = [(lo[a] + (np.arange(n[a] - 1) + 0.5) * res[a]).astype(np.float32) for a in range(3)]
    out["boundary"] = np.concatenate([fill(_near(half[a], ulps)[len(half[a]):], a) for a in range(3)])
    out["half"] = np.concatenate([fill(half[a], a) for a in range(3)])
    ends = [_near(np.array([lo[a], hi[a]], np.float32), 3) for a in range(3)]
    out["ends"] = np.concatenate([fill(np.repeat(ends[a], 40), a) for a in range(3)])
    k = [rng.integers(0, n[a], 4000) for a in range(3)]
    nodes = np.stack([lo[a] + k[a] * res[a] for a in range(3)], axis=1)
    face = nodes[:600].copy()
    face[:, 0] = hi[0]; face[200:, 1] = hi[1]; face[400:, 2] = hi[2]
    out["nodes"] = np.concatenate([nodes, face]).astype(np.float32)
    mag = 10.0 ** rng.uniform(-6, 3, 3000)
    q = rng.uniform(lo, hi, (3000, 3))
    axes = rng.integers(0, 3, 3000)
    sgn = rng.integers(0, 2, 3000)
    rows = np.arange(3000)
    q[rows, axes] = np.where(sgn == 1, hi[axes] + mag, lo[axes] - mag)
    both = rows[::3]
    q[both, (axes[both] + 1) % 3] = hi[(axes[both] + 1) % 3] + mag[both] * 0.5
    out["outside"] = q.astype(np.float32)
    nan = rng.uniform(lo, hi, (12, 3)).astype(np.float32)
    nan[np.arange(12), np.arange(12) % 3] = np.nan
    nan[9:, :] = np.float32(np.nan)
    out["nan"] = nan
    return out


def all_points(sets):
    return np.concatenate([sets[k] for k in sorted(sets)])
