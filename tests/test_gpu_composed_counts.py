"""GPU: compositions of 9-200 sub-SDFs on the kernels their count selects, against the fp64 composition of
tests/composed_ref.py and bit for bit against each other.

Every case names the kernel instantiations it exists to exercise, and a torch.profiler session over the module asserts
that each of them was launched, so that a routing change fails here instead of silently testing another kernel:
  * composed_query_kernel<kMesh, PTS, 16 | 128, kMulti, kExt> (9-16 / 17-128 sub-SDFs; vector, scalar, mesh and
    multi-destination forms), composed_paired_kernel, composed_swept_kernel, composed_clearance_kernel and
    clearance_finish_kernel at MAXS = 128;
  * transforms read from global memory past 64 sub-SDFs, the mesh nearest-bound-first loop up to 32 and the
    bit-reversed order past it (boundary invariance: one far sub-SDF appended across 16->17, 32->33 and 64->65 changes
    no bit), the first-index rule over identical copies;
  * robot_query_kernel<16, false, *> for 9-16 nearest-voxel grid links with well-filled configuration tiles;
  * more than 128 sub-SDFs: the generic per-sub-SDF path of ComposedSDF."""
import numpy as np
import pytest
import torch

import composed_ref as cr
import workloads
from helpers import classify_composed, golden, grid_spec
from oracle import port
from test_gpu_cached import _cached_from_golden
from test_gpu_clearance import _reduce as _clearance_reduce
from test_gpu_swept import _reduce as _swept_reduce

pytestmark = pytest.mark.gpu
TOL = 1e-5
COUNTS = [9, 16, 17, 31, 32, 33, 64, 65, 127, 128]


# ---------------------------------------------------------------- kernel coverage
@pytest.fixture(scope="module")
def kernels():
    """The kernel instantiations this module's tests exist to exercise: tests add their names (see _k), and one
    torch.profiler session (CUDA activity only) spanning the module must have seen every one of them launched.  (One
    session for the module: in a process that had run for minutes, sessions of a few milliseconds lost their kernel
    records.)"""
    from torch.profiler import ProfilerActivity, profile
    want = set()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield want
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    missing = [w for w in sorted(want) if not any(w in n for n in names)]
    assert not missing, (missing, sorted(n for n in names if "<" in n))


def _k(kernel, *args):
    """The demangled name of a kernel instantiation: _k("robot_query_kernel", 16, False, 0)."""
    return f"{kernel}<{', '.join(str(a).lower() for a in args)}>"


# ---------------------------------------------------------------- sets
@pytest.fixture(scope="module")
def parts(tmp_path_factory):
    """(sdf, fp64 spec, interior point in its frame) of every sub-SDF kind."""
    import pytorch_volumetric_b200 as pv
    z = golden("ref_cachedsdf_probe")
    cached = _cached_from_golden(z, "probe", tmp_path_factory.mktemp("counts"))
    gs = grid_spec(cached)
    k = np.unravel_index(np.argmin(gs["val"]), gs["val"].shape)
    g_inside = gs["lo"] + np.array(k) * (gs["hi"] - gs["lo"]) / (np.array(gs["val"].shape) - 1)
    prims = [pv.SphereSDF(0.012), pv.BoxSDF([0.03, 0.012, 0.02]), pv.CylinderSDF(0.01, 0.035)]
    v, f = workloads.bumpy_sphere(16, 9, radius=0.02)
    mesh = pv.MeshSDF(pv.MeshObjectFactory("bumpy", mesh=(v, f)))
    assert mesh.obj_factory.is_closed
    return {"grid": [(cached, gs, g_inside)],
            "prims": [(p, cr.primitive_spec(p.native_desc("cuda")), np.array(c)) for p, c in
                      zip(prims, [(0.004, 0.002, 0.001), (0.002, 0.003, 0.001), (0.004, 0.002, 0.003)])],
            "mesh": [(mesh, cr.mesh_spec(port.MeshPort(vertices=v, faces=f)), np.array([0.003, 0.002, 0.001]))]}


def _members(parts, kind, S):
    """S sub-SDFs: 'grid' (the golden probe table), 'mixed' (the probe, a sphere, a box and a cylinder in turn: the
    kExt instantiations) or 'mesh' (a closed bumpy sphere)."""
    cycle = {"grid": parts["grid"], "mixed": parts["grid"] + parts["prims"], "mesh": parts["mesh"]}[kind]
    return [cycle[s % len(cycle)] for s in range(S)]


def _composed(members, tm):
    """ComposedSDF of the members under tm (S, A, 4, 4): a configuration batch of A (none for A = 1)."""
    import pytorch_volumetric_b200 as pv
    S, A = tm.shape[:2]
    return pv.ComposedSDF([m[0] for m in members], pv.Transform3d(matrix=torch.as_tensor(tm).reshape(S * A, 4, 4).cuda()))


def _points(members, tm, P, seed):
    """P points: a uniform cloud around the set whose first min(S, P) points are replaced by each sub-SDF's interior
    point under configuration 0's transform, so that many sub-SDFs win somewhere."""
    pts = np.random.default_rng(seed).uniform(-0.1, 0.1, (P, 3))
    for s, m in enumerate(members[:P]):
        pts[s] = np.linalg.solve(tm[s, 0].astype(np.float64), np.append(m[2], 1.0))[:3]
    return pts.astype(np.float32)


def _setup(parts, kind, S, A, P, seed=0):
    members = _members(parts, kind, S)
    tm = workloads.random_rigid(S * A, seed=1000 * S + A, t_range=0.06).numpy().reshape(S, A, 4, 4)
    pts = _points(members, tm, P, seed)
    return members, tm, pts


def _which_values(specs, tm, pts, w):
    """fp64 value of the reported sub-SDF w (A, P) at every pair."""
    out = np.full(w.shape, np.nan)
    for s, spec in enumerate(specs):
        a, i = np.nonzero(w == s)
        if len(a):
            q = np.einsum("nij,nj->ni", tm[s, a, :3, :3], pts[i].astype(np.float64)) + tm[s, a, :3, 3]
            out[a, i] = cr.evaluate(spec, q)[0]
    return out


def _assert_fp64(members, tm, pts, v, g, w, what):
    """query(..., return_which=True) against the fp64 composition: grids and primitives through
    helpers.classify_composed (every exceedance a classified flip or tie), meshes through composed_ref.mesh_mismatch;
    `which` names a sub-SDF whose fp64 value is the result's within the tolerance.  Returns the exceedance mask."""
    S, A = tm.shape[:2]
    P = len(pts)
    v, g, w = (t.cpu().numpy() for t in (v, g, w))
    v, g, w = v.reshape(A, P), g.reshape(A, P, 3), w.reshape(A, P)
    specs = [m[1] for m in members]
    assert ((w >= 0) & (w < S)).all(), what
    if specs[0]["kind"] == "mesh":
        ref = cr.compose(specs, tm, pts, per_sub=True)
        bad_v, bad_g, bad_w, rep = cr.mesh_mismatch(v, g, w, ref, TOL, coord_scale=0.2)
        assert bad_v == 0 and bad_g == 0 and bad_w == 0, (what, rep)
        return np.zeros((A, P), bool)
    rv, rg, _rw = cr.compose(specs, tm, pts)
    n_ex, n_un, rep = classify_composed(v, g, rv, rg, specs, tm, pts, TOL)
    assert n_un == 0, (what, rep)
    assert n_ex <= 2e-3 * A * P, (what, rep)
    exceed = (np.abs(v - rv) > TOL) | (np.abs(g - rg).max(-1) > TOL)
    assert ((np.abs(_which_values(specs, tm, pts, w) - rv) <= TOL) | exceed).all(), what
    return exceed


def _same(got, ref, what):
    for k, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), (what, k, int((a != b).reshape(len(a), -1).any(-1).sum()))


# ---------------------------------------------------------------- counts
def _query_args(kind, S, P, multi=False):
    mesh = kind == "mesh"
    return (mesh, 1 if mesh or P % 4 else 2, 16 if S <= 16 else 128, multi, kind == "mixed")


def _case(kernels, parts, kind, S, A, P):
    members, tm, pts_np = _setup(parts, kind, S, A, P)
    comp = _composed(members, tm)
    pts = torch.from_numpy(pts_np).cuda()
    what = (kind, S, A, P)
    kmesh, _pts, maxs, _m, kext = _query_args(kind, S, P)

    v, g, w = comp.query(pts, return_which=True)
    kernels.add(_k("composed_query_kernel", *_query_args(kind, S, P)))
    _assert_fp64(members, tm, pts_np, v, g, w, what)

    # the paired kernel on the same points for every configuration is the cross product itself
    kernels.add(_k("composed_paired_kernel", kmesh, kext, maxs))
    _same(comp.query_paired(pts.expand(A, P, 3).contiguous(), return_which=True), (v, g, w), what + ("paired",))

    kernels.add(_k("composed_swept_kernel", kmesh, kext, maxs))
    _same(comp.query_swept(pts, return_which=True), _swept_reduce(v, g, w, A), what + ("swept",))

    n_seg = 4 if P % 4 == 0 else 1
    kernels |= {_k("composed_clearance_kernel", kmesh, kext, maxs), _k("clearance_finish_kernel", kmesh, kext, maxs)}
    _same(comp.query_clearance(pts.reshape(n_seg, P // n_seg, 3), return_which=True),
          _clearance_reduce(v, g, w, A, n_seg), what + ("clearance",))

    targets = [(torch.full((A * P,), float("nan"), device="cuda"), torch.full((A * P, 3), float("nan"), device="cuda"))
               for _ in range(2)]
    comp.query_into(pts, targets)
    if kind == "mesh" or S > 16 or A < 8 or P % 4:       # otherwise the robot / configuration-major kernels take it
        kernels.add(_k("composed_query_kernel", *_query_args(kind, S, P, multi=True)))
    for tv, tg in targets:
        _same((tv, tg), (v, g), what + ("query_into",))

    if A > 1:
        b, c = A // 5, A // 3
        got = comp.query(pts, cfg_begin=b, cfg_count=c, return_which=True)
        _same(got, (v[b * P:(b + c) * P], g[b * P:(b + c) * P], w[b * P:(b + c) * P]), what + ("slab",))


@pytest.mark.parametrize("S", COUNTS)
@pytest.mark.parametrize("kind", ["grid", "mixed"])
def test_counts(kernels, parts, kind, S):
    for A in (1, 40):
        for P in (4096, 4093):
            _case(kernels, parts, kind, S, A, P)


@pytest.mark.parametrize("S", [31, 32, 33, 128])
def test_counts_mesh(kernels, parts, S):
    for A in (1, 4):
        _case(kernels, parts, "mesh", S, A, 2000)


# ---------------------------------------------------------------- boundary invariance
def _far(tm_row_count):
    """Transforms that put every point ~100 m from the appended sub-SDF: it never wins."""
    m = np.repeat(np.eye(4, dtype=np.float32)[None], tm_row_count, axis=0)
    m[:, :3, 3] = 100.0
    return m


@pytest.mark.parametrize("kind,S", [("grid", 16), ("mixed", 16), ("mesh", 32), ("grid", 64), ("mixed", 64)])
def test_a_far_sub_sdf_changes_nothing(kernels, parts, kind, S):
    A = 1 if kind == "mesh" else 24
    P = 2000 if kind == "mesh" else 4096
    members, tm, pts_np = _setup(parts, kind, S, A, P, seed=3)
    tm_more = np.concatenate([tm, _far(A)[None]])
    pts = torch.from_numpy(pts_np).cuda()
    base, more = _composed(members, tm), _composed(members + members[:1], tm_more)
    ref = base.query(pts, return_which=True)
    got = more.query(pts, return_which=True)
    kernels |= {_k("composed_query_kernel", *_query_args(kind, n, P)) for n in (S, S + 1)}
    assert (ref[2] < S).all()
    _same(got, ref, (kind, S, "query"))
    _same(more.query_paired(pts.expand(A, P, 3).contiguous(), return_which=True), ref, (kind, S, "paired"))
    _same(more.query_swept(pts, return_which=True), base.query_swept(pts, return_which=True), (kind, S, "swept"))


@pytest.mark.parametrize("S", [17, 65, 128])
@pytest.mark.parametrize("kind", ["grid", "mixed", "mesh"])
def test_identical_copies_report_the_first(kernels, parts, kind, S):
    """S copies of one sub-SDF at one pose: sub-SDF 0 everywhere, with the single sub-SDF's bits."""
    member = _members(parts, kind, 2)[-1]           # the probe for grids and meshes' only kind, the sphere for mixed
    tm = np.repeat(workloads.random_rigid(1, seed=5, t_range=0.06).numpy()[:, None], S, axis=0)
    P = 2000 if kind == "mesh" else 4096
    pts = torch.from_numpy(_points([member], tm, P, seed=4)).cuda()
    one = _composed([member], tm[:1]).query(pts, return_which=True)
    copies = _composed([member] * S, tm)
    got = copies.query(pts, return_which=True)
    kernels.add(_k("composed_query_kernel", *_query_args(kind, S, P)))
    assert (got[2] == 0).all() and (one[2] == 0).all()
    _same(got, one, (kind, S))
    _same(copies.query_paired(pts[None], return_which=True), one, (kind, S, "paired"))


# ---------------------------------------------------------------- robot_query_kernel<16, false>
@pytest.mark.parametrize("S", [12, 16])
@pytest.mark.parametrize("A", [64, 28])
def test_robot_kernel_16_links(kernels, parts, S, A):
    members = _members(parts, "grid", S)
    tm = workloads.random_rigid(S * A, seed=S + A, t_range=0.06).numpy().reshape(S, A, 4, 4)
    comp = _composed(members, tm)
    for P, aligned in ((4096, True), (4096, False), (4093, False)):
        _robot_case(kernels, comp, members, tm, P, aligned)


def _robot_case(kernels, comp, members, tm, P, aligned):
    """One point set of test_robot_kernel_16_links."""
    S, A = tm.shape[:2]
    pts_np = _points(members, tm, P, seed=P)
    if aligned:
        pts = torch.from_numpy(pts_np).cuda()
    else:       # a point buffer 4 bytes past a 16-byte boundary
        buf = torch.empty(3 * P + 1, device="cuda")
        pts = buf[1:].view(P, 3)
        pts.copy_(torch.from_numpy(pts_np))
        assert pts.data_ptr() % 16 != 0
    what = (S, A, P, aligned)
    v, g, w = comp.query(pts, return_which=True)
    kernels.add(_k("robot_query_kernel", 16, False, 0))
    _assert_fp64(members, tm, pts_np, v, g, w, what)
    # per-configuration slabs take the point-major kernel
    slabs = [comp.query(pts, cfg_begin=a, cfg_count=1, return_which=True) for a in range(A)]
    kernels.add(_k("composed_query_kernel", False, 2 if aligned and P % 4 == 0 else 1, 16, False, False))
    _same(tuple(torch.cat([s[k] for s in slabs]) for k in range(3)), (v, g, w), what + ("slabs",))
    targets = [(torch.full((A * P,), float("nan"), device="cuda"),
                torch.full((A * P, 3), float("nan"), device="cuda")) for _ in range(2)]
    comp.query_into(pts, targets)
    kernels.add(_k("robot_query_kernel", 16, False, 1))
    for tv, tg in targets:
        _same((tv, tg), (v, g), what + ("query_into",))


# ---------------------------------------------------------------- more than 128 sub-SDFs
@pytest.mark.parametrize("S", [129, 200])
def test_more_than_128_sub_sdfs(kernels, parts, S):
    """__call__, swept, clearance and paired through the generic per-sub-SDF path, against the fp64 composition."""
    A, P = 4, 1000
    members, tm, pts_np = _setup(parts, "mixed", S, A, P)
    comp = _composed(members, tm)
    pts = torch.from_numpy(pts_np).cuda()
    specs = [m[1] for m in members]
    assert comp._native_descs(pts.device)[0] is None          # no fused kernel takes the set
    v, g = comp(pts)
    kernels.add("transform_points_kernel")
    assert v.shape == (A, P) and g.shape == (A, P, 3)
    vw, gw, w = comp.query(pts, return_which=True)
    _same((vw, gw), (v.reshape(-1), g.reshape(-1, 3)), S)
    exceed = _assert_fp64(members, tm, pts_np, v, g, w, (S, "call"))
    rv = cr.compose(specs, tm, pts_np)[0]

    sv, sg, sc, sw = comp.swept(pts, return_argmin=True)
    _same(comp.query_swept(pts, return_which=True), _swept_reduce(vw, gw, w, A), (S, "swept"))
    clean = ~exceed.any(0)
    assert clean.mean() > 0.99
    assert (np.abs(sv.cpu().numpy() - rv.min(0))[clean] <= TOL).all(), S

    seg = pts.reshape(4, P // 4, 3)
    cv, cg, ci, cw = comp.clearance(seg, return_argmin=True)
    assert cv.shape == (A, 4)
    _same(comp.query_clearance(seg, return_which=True), _clearance_reduce(vw, gw, w, A, 4), (S, "clearance"))
    clean = ~exceed.reshape(A, 4, P // 4).any(-1)
    assert (np.abs(cv.cpu().numpy() - rv.reshape(A, 4, P // 4).min(-1))[clean] <= TOL).all(), S

    own = np.stack([_points(members, tm, P, seed=10 + a) for a in range(A)])
    pv_, pg = comp.paired(torch.from_numpy(own).cuda())
    assert pv_.shape == (A, P)
    prv, prg, _ = cr.compose(specs, tm, own)
    for a in range(A):
        n_ex, n_un, rep = classify_composed(pv_[a:a + 1].cpu().numpy(), pg[a:a + 1].cpu().numpy(), prv[a:a + 1],
                                            prg[a:a + 1], specs, tm[:, a:a + 1], own[a], TOL)
        assert n_un == 0 and n_ex <= 2e-3 * P, (S, "paired", a, rep)
