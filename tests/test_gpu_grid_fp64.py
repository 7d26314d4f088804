"""GPU: the voxel-grid lookups against the fp64 grid reference (tests/grid_ref.py) on every launch route.

  * CachedSDF nearest lookup: grid_lookup_tma_kernel (one tile, a partial last tile, the tile loop wrapping once and
    twice over the resident CTAs), grid_lookup_vec4_kernel<false> (below the TMA threshold and with the
    outside_surface / voxel_keys outputs) and grid_lookup_scalar_kernel<false> (n = 1..3 mod 4, a view offset by one
    point); in-range outputs and keys bit-exact; the pinned-host pipeline and a process without the TMA kernel give
    the same bits;
  * trilinear CachedSDF: grid_trilinear_kernel within the trilinear bounds, lattice nodes bit-exact;
  * trilinear links in the fused kernels (point-major PTS 1 / 2, composed_cfgmajor_kernel, robot_serial_kernel) and
    LOOKUP_GT_SDF grids in composed_query_kernel<true, ...> and the paired kernel against the fp64 composition;
  * the voxel containers: nonempty_indices past 2^20 cells (the scan's carry across chunks) and VoxelGrid reads and
    writes in 1-3 dimensions.
Point sets: grid_ref.point_sets -- uniform, +-1..4 ulps around every cell boundary, exact half-way points, the fp32
neighbours of both range ends, lattice nodes and the upper face, 10^-6 .. 10^3 outside the range, NaN.  A
torch.profiler session over the module asserts that every kernel named above was launched."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import composed_ref as cr
import grid_ref as gr
import mesh_ref as mr
import workloads
from helpers import golden
from test_gpu_cached import _cached_from_golden
from test_gpu_clearance import _reduce as _clearance_reduce
from test_gpu_composed_counts import _assert_fp64
from test_gpu_swept import _reduce as _swept_reduce
from test_gpu_trilinear_composed import _arm, _arm_points

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES = [("probe", False), ("probe", True), ("drill", False), ("dyadic", False), ("dyadic", True)]
_CACHE = {}


# ---------------------------------------------------------------- kernel coverage
@pytest.fixture(scope="module", autouse=True)
def kernels():
    """Every kernel this module exists to exercise must appear in one torch.profiler session spanning it."""
    from torch.profiler import ProfilerActivity, profile
    want = {"grid_lookup_tma_kernel", "grid_lookup_vec4_kernel<false>", "grid_lookup_scalar_kernel<false>",
            "grid_trilinear_kernel", "compact_scan_kernel", "composed_query_kernel<false, 1,",
            "composed_query_kernel<false, 2,", "composed_query_kernel<true,", "composed_cfgmajor_kernel<",
            "robot_serial_kernel<", "composed_paired_kernel<true,", "voxel_gather_kernel", "voxel_scatter_kernel"}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    missing = [w for w in sorted(want) if not any(w in n for n in names)]
    assert not missing, (missing, sorted(n for n in names if "kernel" in n)[:60])


# ---------------------------------------------------------------- tables
def make_cached(name, fp32_range, tmp, **kw):
    import pytorch_volumetric_b200 as pv
    if name != "dyadic":
        z = golden(f"ref_cachedsdf_{name}")
        if fp32_range:
            rng32 = [(float(a), float(b)) for a, b in z["range_in"]]
            return _cached_from_golden(z, name + "32", tmp, "table_val_f32range", "table_grad_f32range",
                                       range_in=rng32, **kw)
        return _cached_from_golden(z, name, tmp, **kw)
    val, grad = gr.dyadic_table()
    rin = gr.dyadic_ranges(fp32_range)
    ranges = pv.get_divisible_range_by_resolution(gr.DYADIC_RES, rin)
    nm = "dyadic32" if fp32_range else "dyadic"
    path = str(tmp / f"{nm}.pkl")
    torch.save({f"{nm} {gr.DYADIC_RES} {tuple(ranges)}": (torch.from_numpy(val), torch.from_numpy(grad))}, path)
    c = pv.CachedSDF(nm, gr.DYADIC_RES, rin, pv.SphereSDF(gr.DYADIC_RADIUS), device=kw.pop("device", "cuda"),
                     cache_path=path, **kw)
    assert tuple(c.voxels.shape) == val.shape
    return c


def table_points(ref):
    key = ("pts", tuple(ref.lo64), tuple(ref.shape))
    if key not in _CACHE:
        _CACHE[key] = gr.all_points(gr.point_sets(ref.lo64, ref.hi64, ref.shape, seed=3))
    return _CACHE[key]


def tiled(p, n, seed):
    """n points: the set repeated and shuffled (every point of the set appears in every size >= its length)."""
    reps = np.concatenate([p] * (n // len(p) + 1))
    rest = np.random.default_rng(seed).permutation(len(reps) - len(p)) + len(p)
    return np.ascontiguousarray(np.concatenate([reps[:len(p)], reps[rest]])[:n])


def sizes():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    wave = 1024 * 3 * sm                                    # points one pass of the resident TMA CTAs covers
    return [1, 3, 16383, 16384, 16387, 16384 + 516] + [k * wave + d for k in (1, 2) for d in (-1024, 1024)]


def _same(a, b):
    """Bit for bit, NaN where the other is NaN (the bounding-box rule's gradient at zero overshoot, NaN points)."""
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))


def _check_nearest(ref, p, val, grad, key=None, what=""):
    rep, bad = gr.compare_nearest(ref.nearest(p), val.cpu().numpy(), grad.cpu().numpy(),
                                  key=None if key is None else key.cpu().numpy())
    assert all(len(b) == 0 for b in bad.values()), (what, rep, {k: p[v[:5]] for k, v in bad.items()})
    return rep


# ---------------------------------------------------------------- standalone nearest
@pytest.mark.parametrize("name,fp32_range", TABLES)
def test_nearest_every_route_vs_fp64(name, fp32_range, tmp_path):
    c = make_cached(name, fp32_range, tmp_path)
    ref = gr.Grid.of(c)
    base = table_points(ref)
    worst = {}
    for n in sizes():
        p = tiled(base, n, seed=n)
        q = torch.from_numpy(p).cuda()
        val, grad = c(q)
        keys = c.voxel_keys(q)
        rep = _check_nearest(ref, p, val, grad, keys, (name, n))
        want = ref.nearest(p)
        out = c.outside_surface(q).cpu().numpy()
        assert np.array_equal(out, np.where(want["inb"], want["value"] > 0, True)), n
        if n % 4 == 0 and n >= 16384:                       # the scalar kernel on a view one point into a buffer
            buf = torch.zeros(n + 1, 3, device="cuda")
            buf[1:] = q
            v1, g1 = c(buf[1:])
            assert buf[1:].data_ptr() % 16 != 0
            assert _same(v1, val) and _same(g1, grad)
        worst[n] = (rep["value"], rep["grad"])
    print(name, fp32_range, "err/bound (value, grad) per size:", {k: tuple(round(x, 3) for x in v)
                                                                   for k, v in worst.items()})


def test_host_pipeline_equals_device_call(tmp_path):
    """A pinned host batch through the chunked pipeline at 40 000-point chunks equals the device call."""
    c = make_cached("dyadic", False, tmp_path)
    ch = make_cached("dyadic", False, tmp_path, device="cpu")
    ch.host_pipeline_min_points = 1000
    ch.host_pipeline_chunk = 40000
    p = tiled(table_points(gr.Grid.of(c)), 200_003, seed=1)
    v, g = c(torch.from_numpy(p).cuda())
    vh, gh = ch(torch.from_numpy(p).pin_memory())
    assert vh.is_pinned()
    assert _same(vh, v.cpu()) and _same(gh, g.cpu())


_CHILD = """
import sys, numpy as np, torch, pathlib
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_grid_fp64 as t, grid_ref as gr
out = {{}}
for name, f32 in t.TABLES:
    c = t.make_cached(name, f32, pathlib.Path({tmp!r}))
    base = t.table_points(gr.Grid.of(c))
    for n in t.sizes()[2:]:
        v, g = c(torch.from_numpy(t.tiled(base, n, seed=n)).cuda())
        out[(name, f32, n)] = (v.cpu(), g.cpu())
torch.save(out, {out!r})
"""


def test_tma_equals_vec4_bit_for_bit(tmp_path):
    """Every table and size from 16 383 points up in a process with PVB_GRID_TMA=0 (the knob is read once per
    process): the vector kernel gives the TMA kernel's bits."""
    res = str(tmp_path / "out.pt")
    flags = ["-s"] if sys.flags.no_user_site else []
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), tmp=str(tmp_path), out=res)
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, PVB_GRID_TMA="0"),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    other = torch.load(res)
    for (name, f32, n), (v0, g0) in other.items():
        c = make_cached(name, f32, tmp_path)
        v, g = c(torch.from_numpy(tiled(table_points(gr.Grid.of(c)), n, seed=n)).cuda())
        assert _same(v.cpu(), v0) and _same(g.cpu(), g0), (name, f32, n)


# ---------------------------------------------------------------- standalone trilinear
@pytest.mark.parametrize("name,fp32_range", TABLES)
def test_trilinear_kernel_vs_fp64(name, fp32_range, tmp_path):
    from test_grid_ref_cpu import exact_nodes
    c = make_cached(name, fp32_range, tmp_path, interpolation="trilinear")
    ref = gr.Grid.of(c)
    p = table_points(ref)
    v, g = (t.cpu().numpy() for t in c(torch.from_numpy(p).cuda()))
    rep, bad = gr.compare_trilinear(ref.trilinear(p), v, g)
    assert all(len(b) == 0 for b in bad.values()), (rep, {k: p[x[:5]] for k, x in bad.items()})
    node, key = exact_nodes(ref, p)
    assert np.array_equal(v[node], ref.val32.reshape(-1)[key[node]])
    print(name, fp32_range, "trilinear err/bound", rep, "exact nodes", int(node.sum()))


# ---------------------------------------------------------------- fused kernels, trilinear links
def _arm_case(tmp_path, n_cfg, S=8):
    from pytorch_volumetric_b200.transforms import matrix_of
    s = _arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
    M = matrix_of(s.sdf.obj_frame_to_link_frame).detach().reshape(8, n_cfg, 4, 4)
    links = list(s.sdf.sdfs)
    if S > 8:
        links += links[:S - 8]
        M = torch.cat([M, M[:S - 8].flip(1)])
    members = [(l, cr.trilinear_spec(l), None) for l in links]
    return s, members, M


@pytest.mark.parametrize("n_cfg,S,n_pts,offset", [(5, 8, 4096, 0), (5, 8, 1001, 1), (64, 12, 4096, 0),
                                                   (8, 8, 3001, 0)])
def test_trilinear_links_vs_fp64_composition(tmp_path, n_cfg, S, n_pts, offset):
    """Point-major (aligned: PTS 2, offset view: PTS 1), configuration-major (12 links, 64 configurations) and the
    serial robot kernel (8 links, 8 configurations): values, gradients and argmin against the fp64 composition, every
    exceedance a classified cell-face flip, boundary flip or tie; swept and clearance forms equal the reductions."""
    import pytorch_volumetric_b200 as pv
    s, members, M = _arm_case(tmp_path, n_cfg, S)
    base = _arm_points(n_pts + 1, seed=31)
    pts = base.reshape(-1)[3 * offset:3 * (offset + n_pts)].view(n_pts, 3)
    comp = s.sdf if S == 8 else pv.ComposedSDF([m[0] for m in members],
                                               pv.Transform3d(matrix=M.reshape(S * n_cfg, 4, 4)))
    v, g, w = comp.query(pts, return_which=True)
    _assert_fp64(members, M.cpu().numpy(), pts.cpu().numpy(), v, g, w, (n_cfg, S, n_pts))
    sw = comp.query_swept(pts, return_which=True)
    for a, b in zip(sw, _swept_reduce(v, g, w, n_cfg)):
        assert torch.equal(a, b)
    seg = pts[:n_pts - n_pts % 7].reshape(7, -1, 3)
    cl = comp.query_clearance(seg, return_which=True)
    vs, gs, ws = comp.query(seg.reshape(-1, 3), return_which=True)
    for a, b in zip(cl, _clearance_reduce(vs, gs, ws, n_cfg, 7)):
        assert torch.equal(a, b)


# ---------------------------------------------------------------- fused kernels, LOOKUP_GT_SDF grids
def test_lookup_gt_grids_in_composed_kernels_vs_fp64(tmp_path):
    """Three LOOKUP_GT_SDF probe grids under 4 configurations (composed_query_kernel<true, ...>) and the paired form,
    points in and out of the range of several grids: in range the exact gather (up to boundary flips of the fp32
    transform), out of range the signed fp64 mesh."""
    import pytorch_volumetric_b200 as pv
    c = make_cached("probe", False, tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    assert c.native_desc("cuda").flags & 2
    spec = cr.grid_gt_spec(c, mr.MeshRef(c.gt_sdf.obj_factory))
    S, A, P = 3, 4, 3000
    tm = workloads.random_rigid(S * A, seed=7, t_range=0.01).numpy().reshape(S, A, 4, 4)
    pts = np.random.default_rng(2).uniform(-0.04, 0.04, (P, 3)).astype(np.float32)
    members = [(c, spec, None)] * S
    comp = pv.ComposedSDF([c] * S, pv.Transform3d(matrix=torch.from_numpy(tm).reshape(S * A, 4, 4).cuda()))
    q = torch.from_numpy(pts).cuda()
    v, g, w = comp.query(q, return_which=True)
    inb = np.stack([spec["ref"].in_range(np.einsum("aij,pj->api", tm[s, :, :3, :3], pts.astype(np.float64)).reshape(-1, 3)
                                         + np.repeat(tm[s, :, :3, 3], P, axis=0)) for s in range(S)])
    assert 0.1 < inb.mean() < 0.9 and (inb.sum(0) >= 2).any() and (inb.sum(0) == 0).any()
    _assert_fp64(members, tm, pts, v, g, w, "gt grids")
    own = q[None].expand(A, P, 3).contiguous()
    vp, gp, wp = comp.query_paired(own, return_which=True)
    assert torch.equal(vp, v) and torch.equal(gp, g) and torch.equal(wp, w)


# ---------------------------------------------------------------- voxel containers
@pytest.mark.parametrize("n", [(1 << 20) + 1000, 5 * (1 << 20) + 3, 1 << 26])
def test_nonempty_indices_past_one_scan_chunk(n):
    """The ordered compaction over more than 1 024 blocks of 1 024 cells (the scan carries its total across chunks of
    block counts): equal to torch.nonzero, with a cell set in every block and sparse runs between."""
    from pytorch_volumetric_b200.voxel import nonempty_indices
    gen = torch.Generator(device="cuda").manual_seed(n % 1000)
    flat = (torch.rand(n, device="cuda", generator=gen) < 0.01).float()
    flat[::1024] = 2.0
    flat[-1] = 3.0
    assert torch.equal(nonempty_indices(flat), torch.nonzero(flat).reshape(-1))
    b = flat.bool()
    assert torch.equal(nonempty_indices(b), torch.nonzero(b).reshape(-1))


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("fp32_range", [False, True])
def test_voxel_grid_reads_and_writes_vs_index_rule(d, fp32_range):
    """VoxelGrid on the GPU at boundary-dense points: a write of each point's id lands in the reference's cell
    (one writer per cell kept), and a read returns that cell's content, 0 outside."""
    import pytorch_volumetric_b200 as pv
    from test_grid_ref_cpu import voxel_case
    box = [(-0.37, 0.41), (0.1, 0.9), (-2.0, -1.3)][:d]
    box = [(float(a), float(b)) for a, b in box] if fp32_range else np.array(box)
    vg = pv.VoxelGrid(0.02, box, device="cuda")
    p, want = voxel_case(vg, box)
    ncell = vg.get_voxel_values().numel()
    vg.get_voxel_values().reshape(-1).copy_(torch.arange(1, ncell + 1, dtype=torch.float32, device="cuda"))
    got = vg[torch.from_numpy(p).cuda()].cpu().numpy()
    assert np.array_equal(got, np.where(want >= 0, want + 1, 0).astype(np.float32))
    first = np.unique(want[want >= 0], return_index=True)[1]
    rows = np.nonzero(want >= 0)[0][first]                  # one point per reachable cell
    vg.get_voxel_values().zero_()
    vg[torch.from_numpy(p[rows]).cuda()] = torch.from_numpy(rows.astype(np.float32) + 1).cuda()
    data = vg.get_voxel_values().reshape(-1).cpu().numpy()
    expect = np.zeros(ncell, np.float32)
    expect[want[rows]] = rows + 1
    assert np.array_equal(data, expect)
