"""CPU tier of the ray carve (ray_occupancy, OccupancySDF.from_rays, OccupancyMap.integrate_points, pvb_ray_carve,
pvb_occupancy_apply).

1. The host build of ray_walk (tests/hostsim/hostsim_rays.cpp) equals the fp64 traversal of tests/ray_ref.py up to
   classified near ties, on random rays with origins inside and outside the grid, axis-aligned rays, rays in lattice
   planes and through lattice edges and corners, rays that miss the grid or stay in one voxel, rays spanning a
   1024-long axis, free margins at and above the length, max_range at the length and one float below it, and invalid
   rays.  Unclassified differences: none.
2. Walk properties: a face-connected path, each voxel once, indices moving one way along the ray, at most
   nx + ny + nz voxels; the carve's marks are the union of the walks.
3. out_points is p for a valid ray and NaN otherwise, bit for bit; validity follows the rule.
4. The host build of occupancy_apply_kernel equals occupancy_map_ref.update, marks 1 -> hit, 2 -> free, 0 -> nothing.
5. The C entry points' refusals, and the Python ValueErrors, before any device work."""
import ctypes
import math

import numpy as np
import pytest
import torch

import occupancy_map_ref as omr
import ray_ref
import workloads
from hostsim_lib import PVB_ERR_INVALID

# (name, resolution, range): a generic grid, one whose lattice is exact in binary (ties are exact there), and a
# 1024-long axis
GRIDS = {"tabletop": (0.05, workloads.TABLETOP_RANGE),
         "binary": (0.125, ((-2.0, 1.875), (-1.0, 1.0), (-1.5, 2.0))),
         "long": (0.00176, ((-1.1, -1.1 + 1023 * 0.00176), (-0.55, -0.55 + 4 * 0.00176), (-0.3, -0.3 + 5 * 0.00176)))}


def _box(res, rng):
    lo, dims = ray_ref.lattice(res, rng)
    lo = lo - 0.5 * res                                  # the faces of the grid's first voxels
    return lo, lo + np.asarray(dims) * res, dims


def ray_cases(grid, seed=0):
    """[(name, points fp32 [V, N, 3], origins fp32 [V, 3], max_range, free_margin or None)] on one grid."""
    res, rng = GRIDS[grid]
    lo, hi, dims = _box(res, rng)
    g = np.random.default_rng(seed)
    size = hi - lo
    f32 = np.float32
    out = []

    def add(name, pts, org, max_range=math.inf, margin=None):
        out.append((name, np.asarray(pts, f32), np.asarray(org, f32), max_range, margin))

    org_in = lo + g.uniform(0.05, 0.95, (4, 3)) * size
    add("random inside", lo - 0.3 * size + g.uniform(0, 1.6, (4, 400, 3)) * size, org_in)
    far = g.normal(size=(4, 3))
    org_out = (lo + hi) / 2 + far / np.linalg.norm(far, axis=1, keepdims=True) * np.linalg.norm(size) * 0.9
    add("random outside", lo + g.uniform(0, 1, (4, 400, 3)) * size, org_out)
    add("random outside, beyond", lo - 0.5 * size + g.uniform(0, 2, (4, 400, 3)) * size, org_out, margin=0.0)
    axes = np.eye(3)[g.integers(0, 3, 300)] * g.choice([-1, 1], (300, 1)) * g.uniform(0, 1, (300, 1)) * size.max()
    add("axis-aligned", org_in[:, None] + axes[None], org_in)
    add("axis-aligned, outside", org_out[:, None] + axes[None] * 3, org_out)
    if grid == "binary":
        # lattice coordinates are exact here: a = (x - lo) / r + 0.5 with lo, r and x multiples of 1 / 64
        def world(cells):
            return lo + np.asarray(cells, np.float64) * res
        # in a lattice plane: one coordinate on a face for both ends
        pts, org = [], []
        for k in range(40):
            j = g.integers(0, 3)
            o = g.uniform(0.5, np.asarray(dims) - 0.5)
            p = g.uniform(-2, np.asarray(dims) + 2)
            o[j] = p[j] = g.integers(0, dims[j] + 1)
            org.append(world(np.round(o * 16) / 16)); pts.append(world(np.round(p * 16) / 16))
        add("lattice planes", np.array(pts)[:, None], np.array(org))
        # through edges and corners: from a lattice corner, along integer directions
        pts, org = [], []
        for k in range(60):
            o = g.integers(0, np.asarray(dims) + 1).astype(np.float64)
            d = g.integers(-3, 4, 3).astype(np.float64)
            if not d.any():
                d[0] = 1
            if k % 3 == 0:
                d[g.integers(0, 3)] = 0                  # through edges only
            org.append(world(o)); pts.append(world(o + d * g.integers(1, 6)))
        add("edges and corners", np.array(pts)[:, None], np.array(org), margin=0.0)
        add("edges and corners, margin", np.array(pts)[:, None], np.array(org))
        # one voxel: both ends in the same voxel, no margin
        c = g.integers(0, dims, (50, 3)).astype(np.float64)
        add("one voxel", world(c + g.uniform(0.05, 0.95, (50, 3)))[:, None], world(c + g.uniform(0.05, 0.95, (50, 3))),
            margin=0.0)
        # the free margin at and around the length, and max_range at the length and the next float above it
        o = world(np.array([4.25, 3.5, 7.0]))
        L = np.float32(1.5)
        ends = o + np.array([[L, 0, 0], [0, -L, 0], [0, 0, L]], np.float32)
        add("margin = l", ends, o, margin=float(L))
        add("margin above l", ends, o, margin=float(np.nextafter(L, np.float32(np.inf))))
        add("margin below l", ends, o, margin=float(np.nextafter(L, np.float32(0))))
        add("max_range = l", ends, o, max_range=float(L))
        add("l just above max_range", ends, o, max_range=float(np.nextafter(L, np.float32(0))))
    # rays that miss: both ends on one side outside the grid
    miss = lo - 0.2 * size + g.uniform(0, 0.1, (200, 3)) * size
    add("miss", miss[None], (lo - 0.3 * size)[None])
    add("miss, passing by", np.stack([np.stack([hi[0] + 0.1, lo[1] + 0.5 * size[1], lo[2] - 0.1 + t], 0)
                                       for t in np.linspace(-0.2, 0.0, 20)])[None], (lo - 0.1)[None])
    if grid == "long":
        # spanning the 1024-long axis, end to end, from both sides
        y = g.uniform(lo[1:], hi[1:], (200, 2))
        a = np.concatenate([np.full((200, 1), lo[0] - 0.01), y], 1)
        b = np.concatenate([np.full((200, 1), hi[0] + 0.01), g.uniform(lo[1:], hi[1:], (200, 2))], 1)
        add("spanning", b[None], a[:1])
        add("spanning back", a[None], b[:1])
        for k in range(4):
            add(f"spanning {k}", b[None, 50 * k:50 * (k + 1)], a[50 * k:50 * k + 1])
    # invalid rays: l = 0, NaN and inf in the point or in the origin, mixed with valid ones
    o = org_in[0]
    pts = lo + g.uniform(0, 1, (12, 3)) * size
    pts[0] = o
    pts[1, 0] = np.nan
    pts[2, 1] = np.inf
    pts[3, 2] = -np.inf
    add("invalid points", pts, o)
    add("invalid origin nan", pts, np.array([o[0], np.nan, o[2]]))
    add("invalid origin inf", pts, np.array([np.inf, o[1], o[2]]))
    return [(grid,) + c for c in out]


def all_cases():
    return [c for grid in GRIDS for c in ray_cases(grid)]


CASES = all_cases()


def _walk_and_ref(grid, pts, org, max_range, margin):
    res, rng = GRIDS[grid]
    V, N = pts.shape[0] if pts.ndim == 3 else 1, pts.shape[-2]
    pts = pts.reshape(V, N, 3)
    org = org.reshape(V, 3)
    walks, valid = ray_ref.host_walks(pts, org, N, res, rng, max_range, margin)
    lo, dims = ray_ref.lattice(res, rng)
    m = math.sqrt(3.0) * res / 2 if margin is None else margin
    return walks, valid, lo, dims, m, pts.reshape(-1, 3), np.repeat(org, N, 0)


# ---------------------------------------------------------------- 1. against the fp64 traversal
@pytest.mark.parametrize("grid", list(GRIDS))
def test_walk_equals_the_fp64_traversal_up_to_near_ties(grid):
    res, _ = GRIDS[grid]
    total = diffs = voxels = 0
    report = []
    for _, name, pts, org, max_range, margin in ray_cases(grid):
        walks, valid, lo, dims, m, P, O = _walk_and_ref(grid, pts, org, max_range, margin)
        n_diff, bad = 0, []
        for t, w in enumerate(walks):
            ok, a, u, t_end = ray_ref.segment(O[t], P[t], max_range, m, lo, res)
            assert ok == valid[t], (name, t)
            ref = ray_ref.voxels(a, u, t_end, dims) if ok else np.zeros((0, 3))
            dn, b = ray_ref.compare(w, ref, a, u, t_end) if ok else (len(w), [()] * len(w))
            n_diff += dn
            bad += [(t, v) for v in b]
            voxels += len(ref)
        total += len(walks)
        diffs += n_diff
        report.append((name, n_diff))
        assert not bad, (name, bad[:5])
    print(f"{grid}: {total} rays, {voxels} reference voxels, {diffs} classified differences: {report}")
    assert voxels > 1000


def test_cases_cover_what_they_name():
    by = {(c[0], c[1]): c for c in CASES}
    # ends on the margin: l <= margin carves nothing, just above carves
    for name, carves in (("margin = l", False), ("margin above l", False), ("margin below l", True),
                         ("max_range = l", True), ("l just above max_range", False)):
        walks, valid, *_ = _walk_and_ref("binary", *by[("binary", name)][2:])
        assert all((len(w) > 0) == carves for w in walks), name
    walks, valid, *_ = _walk_and_ref("binary", *by[("binary", "l just above max_range")][2:])
    assert not valid.any()
    for name in ("miss", "miss, passing by"):
        for grid in GRIDS:
            walks, valid, *_ = _walk_and_ref(grid, *by[(grid, name)][2:])
            assert valid.all() and not any(len(w) for w in walks), (grid, name)
    walks, valid, *_ = _walk_and_ref("binary", *by[("binary", "one voxel")][2:])
    assert all(len(w) == 1 for w in walks)
    walks, valid, *_ = _walk_and_ref("long", *by[("long", "spanning")][2:])
    assert all(len(w) >= 1024 for w in walks) and valid.all()
    walks, valid, *_ = _walk_and_ref("tabletop", *by[("tabletop", "invalid points")][2:])
    assert valid.tolist() == [False] * 4 + [True] * 8
    for name in ("invalid origin nan", "invalid origin inf"):
        walks, valid, *_ = _walk_and_ref("tabletop", *by[("tabletop", name)][2:])
        assert not valid.any() and not any(len(w) for w in walks)


# ---------------------------------------------------------------- 2. walk properties
@pytest.mark.parametrize("grid", list(GRIDS))
def test_walk_properties_and_the_carve(grid):
    res, rng = GRIDS[grid]
    for _, name, pts, org, max_range, margin in ray_cases(grid):
        walks, valid, lo, dims, m, P, O = _walk_and_ref(grid, pts, org, max_range, margin)
        union = np.zeros(dims, np.uint8)
        for t, w in enumerate(walks):
            assert len(w) <= sum(dims)
            if len(w) == 0:
                continue
            assert (w >= 0).all() and (w < np.asarray(dims)).all()
            step = np.diff(w.astype(np.int64), axis=0)
            assert (np.abs(step).sum(1) == 1).all(), (name, t)               # face-connected
            assert len({tuple(v) for v in w.tolist()}) == len(w)            # each voxel once
            u = P[t].astype(np.float64) - O[t].astype(np.float64)
            assert ((step * np.sign(u)[None]) >= 0).all(), (name, t)         # in order along the ray
            union[tuple(w.T)] = 2
        marks, _ = ray_ref.host_carve(pts.reshape(-1, 3), org.reshape(-1, 3), pts.shape[-2], res, rng, max_range,
                                      margin)
        assert np.array_equal(marks, union), name


def test_walk_bound_on_the_long_diagonals():
    res, rng = GRIDS["long"]
    lo, hi, dims = _box(res, rng)
    e = 0.01 * res
    a = np.float32([lo + e, [lo[0] + e, hi[1] - e, lo[2] + e]])
    b = np.float32([hi - e, [hi[0] - e, lo[1] + e, hi[2] - e]])
    walks, valid = ray_ref.host_walks(b, a, 1, res, rng, margin=0.0)
    assert [len(w) for w in walks] == [sum(dims) - 2] * 2


# ---------------------------------------------------------------- 3. out_points
def test_out_points_are_the_valid_returns_bit_for_bit():
    for grid, name, pts, org, max_range, margin in CASES:
        res, rng = GRIDS[grid]
        V, N = (pts.shape[0], pts.shape[1]) if pts.ndim == 3 else (1, pts.shape[0])
        P = pts.reshape(-1, 3)
        O = np.repeat(org.reshape(-1, 3), N, 0)
        _, out = ray_ref.host_carve(P, O[::N], N, res, rng, max_range, margin)
        d = P.astype(np.float64) - O.astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            ln = np.sqrt((d * d).sum(1))
            valid = np.isfinite(P).all(1) & np.isfinite(O).all(1) & (ln > 0) & (ln <= max_range)
        got = ~np.isnan(out).any(1)
        assert np.isnan(out[~got]).all()
        assert np.array_equal(out[got].view(np.uint32), P[got].view(np.uint32)), (grid, name)
        # validity follows the fp64 rule wherever l is not within rounding of max_range
        with np.errstate(invalid="ignore"):
            near = np.abs(ln - max_range) <= 1e-6 * ln
        assert np.array_equal(got[~near], valid[~near]), (grid, name)


# ---------------------------------------------------------------- 4. the apply
@pytest.mark.parametrize("q", [omr.quantize(**omr.DEFAULTS), (2048, -256, -1024, 4096, 1024),
                               (32767, -32767, -32767, 32767, 0)])
def test_apply_equals_the_reference_update(q):
    L = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    for m in (0, 1, 2):
        marks = np.full(L.shape, m, np.uint8)
        got_marks, got = ray_ref.host_apply(marks, L, q)
        want = omr.update(L, np.full(L.shape, {0: 2, 1: 1, 2: 0}[m], np.uint8), q)
        assert np.array_equal(got, want), m
        assert not got_marks.any()


# ---------------------------------------------------------------- 5. refusals
def test_abi_refuses_invalid_inputs(built_lib):
    L = built_lib
    fake = ctypes.c_void_p(1 << 12)            # never dereferenced: every call below fails its argument checks
    lo = (ctypes.c_float * 3)(0, 0, 0)
    dims = (ctypes.c_int32 * 3)(10, 20, 30)
    good = (ctypes.c_int32 * 4)(870, -410, -2048, 3584)

    def carve(points=fake, n=1000, per=10, origins=fake, max_range=math.inf, margin=0.01, lo=lo, r=0.01, dims=dims,
              marks=fake, out=fake):
        return L.pvb_ray_carve(points, n, per, origins, max_range, margin, lo, r, dims, marks, out, None)

    def apply(marks=fake, log_odds=fake, dims=dims, params=good):
        return L.pvb_occupancy_apply(marks, log_odds, dims, params, None)

    def params(*p):
        return (ctypes.c_int32 * 4)(*p)

    bad = [dict(points=None), dict(origins=None), dict(lo=None), dict(marks=None), dict(out=None), dict(n=0),
           dict(n=-10), dict(n=1 << 31, per=1), dict(n=(1 << 31) + 10, per=2), dict(per=0), dict(per=-1), dict(per=7),
           dict(per=1001), dict(max_range=0.0), dict(max_range=-1.0), dict(max_range=math.nan), dict(dims=None),
           dict(dims=(ctypes.c_int32 * 3)(1, 20, 30)), dict(dims=(ctypes.c_int32 * 3)(10, 1025, 30)), dict(r=0.0),
           dict(r=-0.01), dict(r=math.inf), dict(r=math.nan), dict(margin=-0.01), dict(margin=math.nan),
           dict(margin=math.inf), dict(lo=(ctypes.c_float * 3)(0, math.inf, 0)),
           dict(lo=(ctypes.c_float * 3)(math.nan, 0, 0))]
    for kw in bad:
        assert carve(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_ray_carve"), kw
    assert b"2..1024" in (carve(dims=(ctypes.c_int32 * 3)(1, 20, 30)), L.pvb_last_error())[1]
    assert b"null" in (carve(marks=None), L.pvb_last_error())[1]
    assert b"max_range" in (carve(max_range=math.nan), L.pvb_last_error())[1]
    assert b"free_margin" in (carve(margin=-1.0), L.pvb_last_error())[1]
    assert b"rays_per_origin" in (carve(per=7), L.pvb_last_error())[1]
    bad = [dict(marks=None), dict(log_odds=None), dict(params=None), dict(dims=None),
           dict(dims=(ctypes.c_int32 * 3)(10, 20, 1025)), dict(params=params(0, -410, -2048, 3584)),
           dict(params=params(870, 0, -2048, 3584)), dict(params=params(870, -410, -409, 3584)),
           dict(params=params(870, -410, -2048, 869)), dict(params=params(870, -410, -32768, 3584)),
           dict(params=params(870, -410, -2048, 32768))]
    for kw in bad:
        assert apply(**kw) == PVB_ERR_INVALID, kw
        assert L.pvb_last_error().startswith(b"pvb_occupancy_apply"), kw
    assert b"clamp_lo <= miss" in (apply(params=params(870, -410, -409, 3584)), L.pvb_last_error())[1]


def test_python_value_errors_before_device_work():
    import pytorch_volumetric_b200 as pv
    rng = workloads.TABLETOP_RANGE
    pts = torch.zeros(10, 3)
    o = torch.zeros(3)
    bad_rays = [(pts.double(), o), (pts.half(), o), (pts.int(), o), (pts, o.double()), (np.zeros((10, 3)), o),
                (torch.zeros(10, 2), o), (torch.zeros(10, 4), o), (torch.zeros(10), o), (torch.zeros(0, 3), o),
                (pts, torch.zeros(1, 3)), (pts, torch.zeros(2)), (torch.zeros(2, 10, 3), torch.zeros(3)),
                (torch.zeros(2, 10, 3), torch.zeros(3, 3)), (torch.zeros(0, 10, 3), torch.zeros(0, 3)),
                (torch.zeros(2, 0, 3), torch.zeros(2, 3)), (torch.zeros(2, 2, 10, 3), torch.zeros(2, 3))]
    for p, org in bad_rays:
        with pytest.raises(ValueError):
            pv.ray_occupancy(p, org, 0.05, rng)
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_rays(p, org, 0.05, rng)
    for kw in (dict(max_range=0.0), dict(max_range=-1.0), dict(max_range=math.nan), dict(resolution=0.0),
               dict(resolution=math.nan), dict(resolution=0.001), dict(range_per_dim=[(0, 1), (0, 1), (0, 0)]),
               dict(free_margin=-0.01), dict(free_margin=math.inf), dict(free_margin=math.nan)):
        args = dict(resolution=0.05, range_per_dim=rng) | kw
        with pytest.raises(ValueError):
            pv.ray_occupancy(pts, o, **args)
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_rays(pts, o, **args)
    for kw in (dict(unknown="seen"), dict(interpolation="cubic")):
        with pytest.raises(ValueError):
            pv.OccupancySDF.from_rays(pts, o, 0.05, rng, **kw)
    m = pv.OccupancyMap.__new__(pv.OccupancyMap)      # the argument checks run before the map's buffers are touched
    for p, org in bad_rays[:6]:
        with pytest.raises(ValueError):
            m.integrate_points(p, org)
    for mr in (0.0, math.nan):
        with pytest.raises(ValueError):
            m.integrate_points(pts, o, max_range=mr)
