"""GPU: the unfused ("generic") route of ComposedSDF against the fp64 composition and against the fused route.

Sets the fused kernels do not take -- sub-SDFs without a native descriptor, nested compositions, more than 128
sub-SDFs -- run `ComposedSDF._generic_query`: for every sub-SDF, pvb_transform_points (transform_points_kernel) or,
for the paired forms, pvb_transform_points_paired (transform_points_paired_kernel), then the sub-SDF's own __call__
and a running minimum in torch, over chunks of at most `generic_chunk_pairs` (configuration, point) pairs.  The
swept, clearance and collision-cost forms fold chunks of 64 configurations of it.

  * Both transform kernels against an fp64 affine product, within the roundoff of their three chained FMAs, and bit
    for bit against a numpy emulation of that chain (each step a * b + c in fp64, rounded to fp32; the elements where
    rounding twice can differ from the single rounding of fmaf are detected and counted): point counts around the
    block size and past the grid-stride cap, transform counts past 65535, a point view that is not 16-byte aligned.
  * Every public form on unfused sets -- the golden mixed+sphere set and the 8-link arm with nearest, trilinear and
    primitive links, wrapped in an opaque ObjectFrameSDF (helpers.opaque_sdfs) -- at 1, 63, 64, 65 and 129
    configurations and on slabs that start and end inside a chunk: against tests/composed_ref.py
    (helpers.assert_fp64), and against the fused route on the same sub-SDFs: values and configuration, point and
    sub-SDF indices bit for bit, gradients within 1e-6 (the rotation back to the object frame is a torch matmul here,
    FMAs there).  Collision costs are sums, compared within the fp32 rounding of their terms.
  * __call__, query and query_paired at 65535, 65536 and 70 000 configurations of 32 points: more transforms than a
    grid dimension holds, and more than one chunk.
  * 129 sub-SDFs at 65 configurations.

A torch.profiler session spanning the module asserts that both transform kernels were launched."""
import time

import numpy as np
import pytest
import torch

import composed_ref as cr
import workloads
from helpers import (arm_points, arm_robot, assert_fp64, clearance_reduce, golden_sets, grid_spec, opaque_sdfs,
                     own_points, swept_reduce)

pytestmark = pytest.mark.gpu
TOL = 1e-5
GRAD_ROT = 1e-6                 # gradients: torch matmul (unfused) against FMAs (fused) for the rotation back
U32 = 2.0 ** -24                # unit roundoff of fp32
GRID_STRIDE_CAP = 132 * 8 * 256  # threads of a grid_for(n, 256, 8) launch on a 132-SM H100
CFG_COUNTS = [1, 63, 64, 65, 129]


# ---------------------------------------------------------------- kernel coverage
@pytest.fixture(scope="module")
def kernels():
    """One torch.profiler session (CUDA activity only) spanning the module: both transform kernels must have been
    launched, so that a routing change fails here instead of silently testing another path."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield
        torch.cuda.synchronize()
    names = {e.name.split("(")[0].split("::")[-1] for e in prof.events()}
    missing = [k for k in ("transform_points_kernel", "transform_points_paired_kernel") if k not in names]
    assert not missing, (missing, sorted(n for n in names if "transform" in n))


# ---------------------------------------------------------------- the transform kernels
def _transform(paired, xf, pts, n_pts):
    """pvb_transform_points(_paired) of xf [n_tf, 4, 4] at pts (device, fp32); [n_tf, n_pts, 3]."""
    from pytorch_volumetric_b200 import _native as nat
    out = torch.empty(xf.shape[0], n_pts, 3, dtype=torch.float32, device="cuda")
    entry = nat.lib().pvb_transform_points_paired if paired else nat.lib().pvb_transform_points
    nat.check(entry(nat.ptr(xf), xf.shape[0], nat.ptr(pts), n_pts, nat.ptr(out), nat.stream_ptr(out.device)),
              entry.__name__)
    return out


def _fma_chain(xf, p):
    """Both kernels' out_k = fmaf(M[k,0], x, fmaf(M[k,1], y, fmaf(M[k,2], z, M[k,3]))) emulated in numpy: xf [n, 4, 4]
    and p [n, 3] fp32, every step a * b + c in fp64 (the product is exact), then rounded to fp32.  Returns (out [n, 3]
    fp32, double [n, 3] bool): double marks the coordinates where some step's fp64 sum was inexact and fell exactly
    on the midpoint of two fp32 values -- the only case where rounding twice can differ from fmaf's one rounding."""
    out = np.empty(p.shape, np.float32)
    double = np.zeros(p.shape, bool)
    for k in range(3):
        acc = xf[:, k, 3]
        for j in (2, 1, 0):
            ab = xf[:, k, j].astype(np.float64) * p[:, j].astype(np.float64)
            c = acc.astype(np.float64)
            s = ab + c
            bp = s - ab
            inexact = ((ab - (s - bp)) + (c - bp)) != 0                    # TwoSum: the error of the fp64 sum
            acc = s.astype(np.float32)
            nb = np.nextafter(acc, np.where(s > acc, np.inf, -np.inf).astype(np.float32))
            mid = (acc.astype(np.float64) + nb.astype(np.float64)) * 0.5
            double[:, k] |= inexact & (s != acc) & (s == mid)
        out[:, k] = acc
    return out, double


def _check_transform(paired, n_tf, n_pts, aligned, seed):
    xf = workloads.random_rigid(n_tf, seed=seed, t_range=0.5).cuda().contiguous()
    n_in = n_tf * n_pts if paired else n_pts
    g = torch.Generator().manual_seed(seed + 1)
    src = ((torch.rand(n_in, 3, generator=g, dtype=torch.float64) * 2 - 1)
           * torch.logspace(-3, 1, n_in, dtype=torch.float64)[:, None]).float()   # magnitudes 1e-3 .. 10
    if aligned:
        pts = src.cuda()
    else:                               # a view one point (12 bytes) into its buffer: not 16-byte aligned
        buf = torch.empty(n_in + 1, 3, device="cuda")
        pts = buf[1:]
        pts.copy_(src)
        assert pts.data_ptr() % 16 != 0
    out = _transform(paired, xf, pts, n_pts).cpu().numpy()
    what = (paired, n_tf, n_pts, aligned)

    x = xf.cpu().numpy()
    p = src.numpy().reshape(n_tf, n_pts, 3) if paired else np.broadcast_to(src.numpy()[None], (n_tf, n_pts, 3))
    R, t = x[:, :3, :3].astype(np.float64), x[:, :3, 3].astype(np.float64)
    terms = np.abs(R[:, None]) * np.abs(p.astype(np.float64))[:, :, None, :]       # [n_tf, n_pts, 3, 3]
    ref = np.einsum("bij,bpj->bpi", R, p.astype(np.float64)) + t[:, None]
    bound = 3 * U32 * (1 + 4 * U32) * (terms.sum(-1) + np.abs(t)[:, None])
    err = np.abs(out - ref)
    assert (err <= bound).all(), (what, "fp64", float((err - bound).max()))

    emu, double = _fma_chain(np.repeat(x, n_pts, axis=0), np.ascontiguousarray(p).reshape(-1, 3))
    emu, double = emu.reshape(out.shape), double.reshape(out.shape)
    differ = out.view(np.uint32) != emu.view(np.uint32)
    print(f"transform {what}: {int(double.sum())} double-rounding cases of {double.size}, "
          f"{int((differ & double).sum())} of them differ")
    assert not (differ & ~double).any(), (what, "fma chain", int((differ & ~double).sum()))
    assert double.sum() <= max(4, 1e-4 * double.size), (what, int(double.sum()))


TRANSFORM_CASES = ([(1, n, True) for n in (1, 255, 256, 257, GRID_STRIDE_CAP + 1001)]
                   + [(7, n, a) for n in (1, 257, GRID_STRIDE_CAP + 1001) for a in (True, False)]
                   + [(n, 5, a) for n in (65535, 65536, 70_000) for a in (True, False)])


@pytest.mark.parametrize("n_tf,n_pts,aligned", TRANSFORM_CASES)
def test_transform_points_kernel(kernels, n_tf, n_pts, aligned):
    """Every transform at every point; 70 000 x 5 pairs also run the grid-stride loop more than once."""
    _check_transform(False, n_tf, n_pts, aligned, seed=n_tf + n_pts)


@pytest.mark.parametrize("n_tf,n_pts,aligned", [(1, 1, True), (1, 257, False), (7, 37, True), (7, 300, False),
                                                (3, GRID_STRIDE_CAP // 3 + 77, True), (65535, 7, False),
                                                (65536, 37, True), (70_000, 37, False)])
def test_transform_points_paired_kernel(kernels, n_tf, n_pts, aligned):
    """Every transform at its own block of n_pts points, blocks not a multiple of the 256-thread block."""
    _check_transform(True, n_tf, n_pts, aligned, seed=3 * n_tf + n_pts)


def test_transform_points_refuses_an_overflowing_size(kernels):
    """n_tf * n_pts * 3 beyond int64 is refused before any launch, by both entry points."""
    from pytorch_volumetric_b200 import _native as nat
    n_tf = 70_000
    xf = torch.eye(4, device="cuda").repeat(n_tf, 1, 1)
    buf = torch.zeros(3, device="cuda")
    for entry in (nat.lib().pvb_transform_points, nat.lib().pvb_transform_points_paired):
        for n_pts, ok in (((2 ** 63 - 1) // 3 // n_tf + 1, False), (0, True)):
            rc = entry(nat.ptr(xf), n_tf, nat.ptr(buf), n_pts, nat.ptr(buf), nat.stream_ptr(buf.device))
            assert (rc == 0) == ok, (entry.__name__, n_pts)
            if not ok:
                assert b"invalid argument" in nat.lib().pvb_last_error()


# ---------------------------------------------------------------- sets
@pytest.fixture(scope="module")
def golden(tmp_path_factory):
    """(sub-SDF, fp64 spec) of the golden mixed+sphere set: trilinear probe, nearest probe, sphere, trilinear probe;
    and the golden query points."""
    z, sets = golden_sets(tmp_path_factory.mktemp("generic"))
    return [(s, _spec(s)) for s in sets["mixed+sphere"]], z["q"]


def _spec(sdf):
    import pytorch_volumetric_b200 as pv
    if isinstance(sdf, pv.CachedSDF):
        return cr.trilinear_spec(sdf) if sdf.interpolation == "trilinear" else grid_spec(sdf)
    return cr.primitive_spec(sdf.native_desc("cuda"))


def _routes(sdfs, tm, opaque=True):
    """(unfused, fused) ComposedSDF of sdfs under tm (S, A, 4, 4), a configuration batch of A: the unfused one over
    the sub-SDFs wrapped in opaque ObjectFrameSDFs (or over sdfs themselves when opaque is False, fused then None)."""
    import pytorch_volumetric_b200 as pv
    S, A = tm.shape[:2]
    tsf = pv.Transform3d(matrix=torch.as_tensor(tm, dtype=torch.float32).reshape(S * A, 4, 4).cuda())
    unfused = pv.ComposedSDF(opaque_sdfs(pv, sdfs) if opaque else sdfs, tsf)
    unfused.set_transforms(tsf, batch_dim=(A,))
    assert unfused._native_descs(torch.device("cuda", torch.cuda.current_device()))[0] is None
    if not opaque:
        return unfused, None
    fused = pv.ComposedSDF(sdfs, tsf)
    fused.set_transforms(tsf, batch_dim=(A,))
    return unfused, fused


def _same(got, ref, what):
    for k, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape and torch.equal(a, b), (what, k, int((a != b).sum()))


def _grad(a, b, what):
    assert a.shape == b.shape, what
    if a.numel():
        assert float((a - b).abs().max()) < GRAD_ROT, (what, float((a - b).abs().max()))


def _matches_fused(got, ref, grad_at, what):
    """Bit for bit but for the gradients, the tuple entries at grad_at."""
    for k, (a, b) in enumerate(zip(got, ref)):
        if k in grad_at:
            _grad(a, b, (what, k))
        else:
            _same((a,), (b,), (what, k))


def _cost_rows(v, g, w, p, m, S, ev=0.0, eg=0.0):
    """fp64 collision-cost rows of per-pair results v [A, n_seg, L], g [.., 3], w [..] at points p [.., n_seg, L, 3]
    (broadcast over A when shared): (cost [A * n_seg], twist [A * n_seg, S, 6], sum|twist term|, slack).  The slack
    bounds how far the rows can move when every value moves by at most ev and every gradient component by at most
    eg: (cost slack [A * n_seg], twist slack [A * n_seg, S, 6])."""
    v, g, p = v.double(), g.double(), p.double().expand_as(g)
    h = (m - v).clamp_min(0.0)
    terms = torch.cat([g, torch.linalg.cross(p, g, dim=-1)], -1) * (2 * h)[..., None]
    hp = (m - v + ev).clamp_min(0.0)
    live = hp > 0
    lin = (2 * ev * (g.abs().amax(-1) + eg) + 2 * hp * eg) * live
    slack = torch.cat([lin[..., None].expand(*lin.shape, 3), (lin * p.abs().sum(-1))[..., None].expand(*lin.shape, 3)],
                      -1)
    cslack = (ev * (2 * hp + ev) * live).sum(-1).reshape(-1)
    A, n_seg = v.shape[:2]
    twist, abs_tw, tslack = (torch.zeros(A, n_seg, S, 6, dtype=torch.float64, device=v.device) for _ in range(3))
    for s in range(S):
        mask = (w == s)[..., None]
        twist[:, :, s] = (terms * mask).sum(-2)
        abs_tw[:, :, s] = (terms.abs() * mask).sum(-2)
        tslack[:, :, s] = (slack * mask).sum(-2)
    return ((h * h).sum(-1).reshape(-1), twist.reshape(-1, S, 6), abs_tw.reshape(-1, S, 6),
            (cslack, tslack.reshape(-1, S, 6)))


def _assert_cost(got, ref, what):
    """got (cost, twist) within the fp32 rounding of ref's terms plus ref's slack."""
    rc, rt, at, (cs, ts) = ref
    cost, twist = got[0].reshape(-1).double(), got[1].reshape(rt.shape).double()
    ec = (cost - rc).abs() - 1e-5 * rc - cs
    et = (twist - rt).abs() - 1e-5 * at - ts
    assert float(ec.max()) <= 1e-30, (what, "cost", float((cost - rc).abs().max()))
    assert float(et.max()) <= 1e-30, (what, "twist", float((twist - rt).abs().max()))


def _cost_slab(ref, rows):
    """The rows of a _cost_rows result."""
    rc, rt, at, (cs, ts) = ref
    return rc[rows], rt[rows], at[rows], (cs[rows], ts[rows])


def _fp64_per_pair(members, tm, pts, v, g, exceed):
    """fp64 (value, gradient) of the composition at every pair, the route's own output at its classified exceedances
    (voxel-boundary flips and ties, which assert_fp64 admits); [A, P] / [A, P, 3] torch fp64 on the GPU."""
    rv, rg, _ = cr.compose([m[1] for m in members], tm, pts)
    A, P = rv.shape
    v, g = v.reshape(A, P).double().cpu().numpy(), g.reshape(A, P, 3).double().cpu().numpy()
    rv, rg = np.where(exceed, v, rv), np.where(exceed[..., None], g, rg)
    return torch.from_numpy(rv).cuda(), torch.from_numpy(rg).cuda()


# ---------------------------------------------------------------- every form
def _every_form(members, tm, pts_np, own_np, slabs, opaque=True, what=""):
    """Every public form of the unfused route against the fp64 composition, and against the fused route on the
    same sub-SDFs when opaque.  pts_np [P, 3] shared points, own_np [A, P, 3] every configuration's own points; P a
    multiple of 4 (4 clearance segments)."""
    S, A = tm.shape[:2]
    P = len(pts_np)
    sdfs = [m[0] for m in members]
    unfused, fused = _routes(sdfs, tm, opaque)
    pts, own = torch.from_numpy(pts_np).cuda(), torch.from_numpy(own_np).cuda()
    seg, own_seg = pts.reshape(4, P // 4, 3), own.reshape(A, 4, P // 4, 3)

    # query: fp64, fused, slabs
    v, g, w = unfused.query(pts, return_which=True)
    exceed = assert_fp64(members, tm, pts_np, v, g, w, (what, "query"))
    if fused:
        _matches_fused((v, g, w), fused.query(pts, return_which=True), (1,), (what, "query"))
    for b, c in slabs:
        rows = slice(b * P, (b + c) * P)
        _same(unfused.query(pts, b, c, return_which=True), (v[rows], g[rows], w[rows]), (what, "query slab", b, c))
    # __call__: the query, shaped [A, P]
    cv, cg = unfused(pts)
    _same((cv, cg), (v.reshape(A, P), g.reshape(A, P, 3)), (what, "call"))
    if fused:
        _matches_fused((cv, cg), fused(pts), (1,), (what, "call"))

    # query_paired / paired
    pv_, pg, pw = unfused.query_paired(own, return_which=True)
    pexceed = assert_fp64(members, tm, own_np, pv_, pg, pw, (what, "paired"))
    if fused:
        _matches_fused((pv_, pg, pw), fused.query_paired(own, return_which=True), (1,), (what, "paired"))
    _same(unfused.paired(own), (pv_.reshape(A, P), pg.reshape(A, P, 3)), (what, "paired()"))
    for b, c in slabs:
        rows = slice(b * P, (b + c) * P)
        _same(unfused.query_paired(own[b:b + c], b, c, return_which=True), (pv_[rows], pg[rows], pw[rows]),
              (what, "paired slab", b, c))

    # swept: the (value, configuration, sub-SDF) minimum of the query
    rv = cr.compose([m[1] for m in members], tm, pts_np)[0]
    got = unfused.swept(pts, return_argmin=True)
    red = swept_reduce(v, g, w, A)
    _same(unfused.query_swept(pts, return_which=True), red, (what, "swept"))
    _same(got, (red[0], red[1], red[2].long(), red[3].long()), (what, "swept()"))
    if fused:
        _matches_fused(got, fused.swept(pts, return_argmin=True), (1,), (what, "swept"))
    clean = ~exceed.any(0)
    assert (np.abs(got[0].cpu().numpy() - rv.min(0))[clean] <= TOL).all(), (what, "swept fp64")
    for b, c in slabs:
        rows = slice(b * P, (b + c) * P)
        _same(unfused.query_swept(pts, b, c, return_which=True), swept_reduce(v[rows], g[rows], w[rows], c, b),
              (what, "swept slab", b, c))

    # clearance: the first-point minimum over each of 4 segments, every configuration
    got = unfused.clearance(seg, return_argmin=True)
    red = clearance_reduce(v, g, w, A, 4)
    _same(unfused.query_clearance(seg, return_which=True), red, (what, "clearance"))
    _same(got, (red[0].reshape(A, 4), red[1].reshape(A, 4, 3), red[2].reshape(A, 4).long(),
                red[3].reshape(A, 4).long()), (what, "clearance()"))
    if fused:
        _matches_fused(got, fused.clearance(seg, return_argmin=True), (1,), (what, "clearance"))
    clean = ~exceed.reshape(A, 4, P // 4).any(-1)
    assert (np.abs(got[0].cpu().numpy() - rv.reshape(A, 4, P // 4).min(-1))[clean] <= TOL).all(), \
        (what, "clearance fp64")
    for b, c in slabs:
        rows = slice(b * P, (b + c) * P)
        _same(unfused.query_clearance(seg, b, c, return_which=True), clearance_reduce(v[rows], g[rows], w[rows], c, 4),
              (what, "clearance slab", b, c))

    # paired clearance
    got = unfused.paired_clearance(own_seg, return_argmin=True)
    red = clearance_reduce(pv_, pg, pw, A, 4)
    _same(unfused.query_paired_clearance(own_seg, return_which=True), red, (what, "paired clearance"))
    _same(got, (red[0].reshape(A, 4), red[1].reshape(A, 4, 3), red[2].reshape(A, 4).long(),
                red[3].reshape(A, 4).long()), (what, "paired_clearance()"))
    if fused:
        _matches_fused(got, fused.paired_clearance(own_seg, return_argmin=True), (1,), (what, "paired clearance"))
    prv = cr.compose([m[1] for m in members], tm, own_np)[0]
    clean = ~pexceed.reshape(A, 4, P // 4).any(-1)
    assert (np.abs(got[0].cpu().numpy() - prv.reshape(A, 4, P // 4).min(-1))[clean] <= TOL).all(), \
        (what, "paired clearance fp64")
    for b, c in slabs:
        rows = slice(b * 4, (b + c) * 4)
        _same(unfused.query_paired_clearance(own_seg[b:b + c], b, c, return_which=True),
              tuple(t[rows] for t in red), (what, "paired clearance slab", b, c))

    # collision costs: fp64 sums of the route's own per-pair results (the definition), of the fp64 composition within
    # what the per-pair tolerance moves them, and the fused route's rows within what its gradients move them
    m = float(np.float32(torch.quantile(v.float(), 0.25).item()))
    shape = (A, 4, P // 4)
    for paired_form in (False, True):
        vv, gg, ww, ex = (pv_, pg, pw, pexceed) if paired_form else (v, g, w, exceed)
        p = own_seg if paired_form else seg
        call = (lambda c: c.paired_collision_cost(own_seg, m)) if paired_form else (lambda c: c.collision_cost(seg, m))
        got = call(unfused)
        assert got[0].shape == (A, 4) and got[1].shape == (A, 4, S, 6)
        tag = (what, "paired collision cost" if paired_form else "collision cost")
        own_ref = _cost_rows(vv.reshape(shape), gg.reshape(*shape, 3), ww.reshape(shape), p, m, S)
        _assert_cost(got, own_ref, tag)
        fv, fg = _fp64_per_pair(members, tm, own_np if paired_form else pts_np, vv, gg, ex)
        _assert_cost(got, _cost_rows(fv.reshape(shape), fg.reshape(*shape, 3), ww.reshape(shape), p, m, S, TOL, TOL),
                     tag + ("fp64",))
        if fused:
            _assert_cost(call(fused), _cost_rows(vv.reshape(shape), gg.reshape(*shape, 3), ww.reshape(shape), p, m,
                                                 S, 0.0, GRAD_ROT), tag + ("fused",))
        b, c = slabs[-1]
        rows = slice(b * 4, (b + c) * 4)
        if paired_form:
            sc, st = unfused.query_paired_collision_cost(own_seg[b:b + c], m, b, c)
        else:
            sc, st = unfused.query_collision_cost(seg, m, b, c)
        _assert_cost((sc, st), _cost_slab(own_ref, rows), tag + ("slab", b, c))
    return unfused


def _slabs(A):
    """Slabs [b, b + c) that start and end inside a 64-configuration chunk, one of them crossing chunks."""
    out = [(0, A)] if A == 1 else [(1, A - 2), (A // 3, 1)]
    if A > 64:
        out.append((5, A - 10))
    return out


@pytest.mark.parametrize("A", CFG_COUNTS)
def test_golden_set_every_form(kernels, golden, A):
    members, q = golden
    S, P = len(members), 512
    tm = workloads.random_rigid(S * A, seed=100 + A, t_range=0.03).numpy().reshape(S, A, 4, 4)
    pts = q[:P]
    own = own_points(torch.from_numpy(pts), A, seed=A).cpu().numpy()
    _every_form(members, tm, pts, own, _slabs(A), what=("golden", A))


def test_golden_set_small_query_chunks(kernels, golden):
    """`_generic_query` in chunks of 64 configurations of 512 points: its chunk seams do not show in any output."""
    members, q = golden
    S, A, P = len(members), 129, 512
    tm = workloads.random_rigid(S * A, seed=7, t_range=0.03).numpy().reshape(S, A, 4, 4)
    pts = torch.from_numpy(q[:P]).cuda()
    own = own_points(pts, A, seed=8)
    small, fused = _routes([m[0] for m in members], tm)
    small.generic_chunk_pairs = 64 * P
    whole, _ = _routes([m[0] for m in members], tm)
    assert A * P <= whole.generic_chunk_pairs
    for b, c in ((0, A), (3, 100), (60, 8), (64, 65)):
        _same(small.query(pts, b, c, return_which=True), whole.query(pts, b, c, return_which=True), ("query", b, c))
        _same(small.query_paired(own[b:b + c], b, c, return_which=True),
              whole.query_paired(own[b:b + c], b, c, return_which=True), ("paired", b, c))
    _matches_fused(small.query(pts, return_which=True), fused.query(pts, return_which=True), (1,), "fused")


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_opaque_arm_every_form(kernels, tmp_path, kind):
    s = arm_robot(tmp_path, kind)
    A, P = 65, 1000
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    sdfs = s.sdf.sdfs
    members = [(l, _spec(l)) for l in sdfs]
    tm = s.sdf.obj_frame_to_link_frame.get_matrix().detach().cpu().numpy().reshape(len(sdfs), A, 4, 4)
    pts = arm_points(P, seed=31)
    own = torch.stack([arm_points(P, seed=300 + a) for a in range(A)])
    _every_form(members, tm, pts.cpu().numpy(), own.cpu().numpy(), _slabs(A), what=("arm", kind))


def test_more_than_128_sub_sdfs_every_form(kernels, golden):
    """129 sub-SDFs take the unfused route without a wrapper; no fused route to compare with."""
    members, q = golden
    S, A, P = 129, 65, 512
    members = [members[s % len(members)] for s in range(S)]
    tm = workloads.random_rigid(S * A, seed=129, t_range=0.03).numpy().reshape(S, A, 4, 4)
    pts = q[:P]
    own = own_points(torch.from_numpy(pts), A, seed=9).cpu().numpy()
    _every_form(members, tm, pts, own, _slabs(A), opaque=False, what=("129 sub-SDFs",))


# ---------------------------------------------------------------- past 65535 configurations
def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


@pytest.mark.parametrize("A", [65535, 65536, 70_000])
def test_past_65535_configurations(kernels, golden, A):
    """__call__, query and query_paired at A configurations of 32 points: bit for bit (gradients within 1e-6) with
    the fused route everywhere, and against the fp64 composition on the configurations around 65535 and a sample of
    the others."""
    members, q = golden
    S, P = len(members), 32
    sdfs = [m[0] for m in members]
    tm = workloads.random_rigid(S * A, seed=A, t_range=0.03).numpy().reshape(S, A, 4, 4)
    unfused, fused = _routes(sdfs, tm)
    pts_np = q[:P]
    pts = torch.from_numpy(pts_np).cuda()
    own = own_points(pts, A, seed=A)
    rng = np.random.default_rng(A)
    sample = np.unique(np.concatenate([[0, 1, 32767, 32768, 65534, 65535, A - 2, A - 1],
                                       rng.integers(0, A, 250)]))
    sample = sample[sample < A]

    (cv, cg), t_call = _timed(lambda: unfused(pts))
    assert cv.shape == (A, P) and cg.shape == (A, P, 3)
    _matches_fused((cv, cg), fused(pts), (1,), (A, "call"))
    del cv, cg
    (v, g, w), t_query = _timed(lambda: unfused.query(pts, return_which=True))
    _matches_fused((v, g, w), fused.query(pts, return_which=True), (1,), (A, "query"))
    v, g, w = (t.reshape(A, P, *t.shape[1:])[sample].reshape(len(sample) * P, *t.shape[1:]) for t in (v, g, w))
    assert_fp64(members, tm[:, sample], pts_np, v, g, w, (A, "query"))
    del v, g, w
    (v, g, w), t_paired = _timed(lambda: unfused.query_paired(own, return_which=True))
    _matches_fused((v, g, w), fused.query_paired(own, return_which=True), (1,), (A, "paired"))
    v, g, w = (t.reshape(A, P, *t.shape[1:])[sample].reshape(len(sample) * P, *t.shape[1:]) for t in (v, g, w))
    assert_fp64(members, tm[:, sample], own[sample].cpu().numpy(), v, g, w, (A, "paired"))
    print(f"unfused route, {A} configurations x {P} points, {S} sub-SDFs: __call__ {t_call * 1e3:.1f} ms, "
          f"query {t_query * 1e3:.1f} ms, query_paired {t_paired * 1e3:.1f} ms")
