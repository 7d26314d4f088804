"""GPU: batch_chamfer_dist, pairwise_distance_chamfer and PlausibleDiversity against the fp64 restatement
(tests/chamfer_ref.py) on every route of chamfer_partial_kernel, one value per (transform, point) pair where that is
possible, across the 65 535-transform launch split, the grid-stride and binning edges, and bit for bit on an exact
cloud.  Tolerances are derived from fp32 unit roundoff (chamfer_ref: transform_error, square_bound, sum_bound)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import chamfer_ref as cr
import workloads
from helpers import golden, pv_factory

pytestmark = pytest.mark.gpu

U = cr.U32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MESH_EVAL = 2e-6          # fp32 closest point at unit coordinate scale (tests/test_hostsim.py)
PRIM_EVAL = 1e-6          # fp32 primitive evaluation (tests/primitive_ref.py)


def n_blk(n):
    """pvb_chamfer_workspace: blocks per transform."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return min(-(-n // 256), 4 * sms)


@pytest.fixture(scope="module")
def objects(tmp_path_factory):
    """A 64-triangle closed bumpy sphere (radius 0.1 m) as a mesh, nearest-voxel grids with both out-of-range
    strategies, a trilinear grid, and the three primitives, with their fp64 specs."""
    import pytorch_volumetric_b200 as pv
    v, f = workloads.bumpy_sphere(8, 5)
    obj = pv.MeshObjectFactory("bumpy64", mesh=(v, f))
    msdf = pv.MeshSDF(obj)
    d = tmp_path_factory.mktemp("chamfer_fp64")
    rng = obj.bounding_box(padding=0.05)
    grid = pv.CachedSDF("bumpy64", 0.01, rng, msdf, device="cuda", cache_path=str(d / "g.pkl"), clean_cache=True)
    grid_gt = pv.CachedSDF("bumpy64", 0.01, rng, msdf, device="cuda", cache_path=str(d / "g.pkl"),
                           out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    tri = pv.CachedSDF("bumpy64", 0.01, rng, msdf, device="cuda", cache_path=str(d / "g.pkl"),
                       interpolation="trilinear")
    assert grid_gt.native_desc("cuda").flags & 2            # PVB_GRID_OOB_GT: the tree walk runs in the kernel
    sphere, box, cyl = pv.SphereSDF(0.07), pv.BoxSDF([0.12, 0.08, 0.1]), pv.CylinderSDF(0.05, 0.14)
    return {
        "mesh": (dict(obj_factory=obj), cr.mesh_spec(v, f)),
        "grid": (dict(obj_sdf=grid), cr.grid_spec(grid)),
        "grid_gt": (dict(obj_sdf=grid_gt), cr.grid_spec(grid_gt, gt_mesh=(v, f))),
        "trilinear": (dict(obj_sdf=tri), cr.trilinear_spec(tri)),
        "sphere": (dict(obj_sdf=sphere), cr.primitive_spec(sphere.native_desc("cuda"))),
        "box": (dict(obj_sdf=box), cr.primitive_spec(box.native_desc("cuda"))),
        "cylinder": (dict(obj_sdf=cyl), cr.primitive_spec(cyl.native_desc("cuda"))),
        "_mesh": (v, f, obj),
    }


def eval_error(route, spec, q):
    """Bound on the fp32 evaluation error of the unsigned distance at object-frame points q [m, 3]."""
    if route in ("mesh", "grid_gt"):
        return np.full(len(q), MESH_EVAL)
    if route in ("sphere", "box", "cylinder"):
        return np.full(len(q), PRIM_EVAL)
    if route == "trilinear":
        return np.full(len(q), PRIM_EVAL)
    # nearest voxel: table entries are exact; the bounding-box rule is a few fp32 operations on |q| and the box
    return 8 * U * (np.linalg.norm(q, axis=1) + np.abs(spec["bb"]).max())


def lipschitz(route):
    """1 for distances; the trilinear interpolant of a distance table has slope at most 1 per axis."""
    return math.sqrt(3) if route == "trilinear" else 1.0


def check_pairs(route, spec, out, w2o, pts, scale):
    """out (B,) for a one-point cloud: every (transform, point) value against fp64, nearest-voxel mismatches only
    as classified voxel-boundary flips.  Returns the number of flips."""
    q = cr.object_points(w2o, pts)[:, 0]
    d = cr.distance(spec, q)
    ref = (scale * d) ** 2
    dd = lipschitz(route) * cr.transform_error(w2o, pts)[:, 0] + eval_error(route, spec, q)
    tol = cr.square_bound(d, dd, scale) + 4 * U * ref
    bad = np.nonzero(np.abs(out - ref) > tol)[0]
    if route not in ("grid", "grid_gt"):
        assert len(bad) == 0, (route, bad[:5], out[bad[:5]], ref[bad[:5]])
        return 0
    for b in bad:
        alts = cr.grid_alternatives(spec, q[b])
        ok = any(abs(out[b] - (scale * a) ** 2) <= tol[b] + 4 * U * (scale * a) ** 2 for a in alts)
        assert ok, (route, int(b), float(out[b]), float(ref[b]), q[b])
    return len(bad)


def transforms_near_and_far(n, seed):
    """Random rigid transforms; a third of them put the point far outside the object's box (up to 2 m)."""
    near = workloads.random_rigid(n - n // 3, seed=seed, t_range=0.12, dtype=torch.float64)
    far = workloads.random_rigid(n // 3, seed=seed + 1, t_range=2.0, dtype=torch.float64)
    return torch.cat([near, far]).float()


@pytest.mark.parametrize("route", ["mesh", "grid", "grid_gt", "trilinear", "sphere", "box", "cylinder"])
def test_one_point_per_transform_across_the_launch_split(objects, route):
    """A one-point cloud under B = 70 000 transforms: B separate values of (scale d)^2, checked at every index
    (the kernel takes 65 535 transforms per launch; chamfer.py splits the rest)."""
    import pytorch_volumetric_b200 as pv
    kw, spec = objects[route]
    B = 70_000
    w2o = transforms_near_and_far(B, seed=11)
    pts = torch.tensor([[0.031, -0.022, 0.047]])
    out = pv.batch_chamfer_dist(w2o.cuda(), pts.cuda(), scale=1000.0, **kw)
    assert out.shape == (B,) and out.dtype == torch.float32 and out.device.type == "cuda"
    flips = check_pairs(route, spec, out.cpu().numpy().astype(np.float64), w2o.numpy(), pts.numpy(), 1000.0)
    assert flips <= B // 1000, flips
    # the far third really is outside the box (the bounding-box / tree-walk side of the grid routes)
    q = cr.object_points(w2o[-10:].numpy(), pts.numpy())[:, 0]
    if route.startswith("grid"):
        assert not np.all((q >= spec["lo"]) & (q <= spec["hi"]), axis=1).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 32_767, 32_768, 100_000])
def test_sizes_and_accumulation(objects, n, B):
    """Means over n points at the grid-stride and binning edges (binned from 32 768 points, in the frame of the first
    transform; the second and third transforms are far from it, so their points land in clamped border cells).
    fp64 and host inputs give the same bits as fp32 CUDA inputs, returned as fp64 on the host."""
    import pytorch_volumetric_b200 as pv
    v, f, obj = objects["_mesh"]
    spec = objects["mesh"][1]
    g = torch.Generator().manual_seed(n + B)
    pts = ((torch.rand(n, 3, generator=g, dtype=torch.float64) - 0.5) * 0.3).float()
    w2o = workloads.random_rigid(3, seed=n, t_range=0.02)
    w2o[1:, :3, 3] += torch.tensor([[0.9, -0.4, 0.3], [-0.5, 1.1, -0.7]])
    w2o = w2o[:B].contiguous()
    out = pv.batch_chamfer_dist(w2o.cuda(), pts.cuda(), obj, scale=1000.0)
    assert out.shape == (B,) and out.dtype == torch.float32
    d = cr.per_pair(spec, w2o.numpy(), pts.numpy())
    ref = ((1000.0 * d) ** 2).mean(axis=1)
    dd = cr.transform_error(w2o.numpy(), pts.numpy()) + MESH_EVAL
    tol = cr.square_bound(d, dd, 1000.0).mean(axis=1) + cr.sum_bound(n, n_blk(n)) * ref
    err = np.abs(out.cpu().numpy().astype(np.float64) - ref)
    assert (err <= tol).all(), (err, tol)
    out64 = pv.batch_chamfer_dist(w2o.double(), pts.double(), obj, scale=1000.0)
    assert out64.dtype == torch.float64 and out64.device.type == "cpu"
    assert torch.equal(out64, out.cpu().double())


def exact_cloud(n, B, seed):
    """World points and transforms for which every object-frame point lies straight above a face interior of the
    12-triangle box mesh at height 2^-6 or 2^-5 (tests/test_chamfer_ref_cpu.py confirms the premise on the host
    build): transform 0 is a signed permutation plus a dyadic translation, transform b > 0 a box symmetry after it.
    Returns (box mesh, world points fp32, transforms fp32, the exact mean of d^2 as fp64)."""
    rng = np.random.default_rng(seed)
    half = 0.25
    v, f = cr.box_mesh(half)
    q, h = cr.exact_box_cloud(n, half, [2.0 ** -6, 2.0 ** -5], rng)
    P0 = cr.signed_permutations(1, rng)[0]
    t0 = rng.integers(-16, 17, 3) / 16.0
    world = (q - t0) @ P0                                  # P0^T (q - t0), exact
    W = np.zeros((B, 4, 4))
    W[:, 3, 3] = 1.0
    S = np.concatenate([np.eye(3)[None], cr.signed_permutations(B - 1, rng)])
    W[:, :3, :3] = S @ P0
    W[:, :3, 3] = t0 @ np.swapaxes(S, 1, 2)                # S t0
    assert np.array_equal(world.astype(np.float32).astype(np.float64), world)
    total = float((h * h).sum())                           # a sum of 2^-12 and 2^-10 terms: exact in fp64
    return (v, f), torch.from_numpy(world.astype(np.float32)), torch.from_numpy(W.astype(np.float32)), total / n


def test_exact_cloud_binned_path_is_exact():
    """n = 10^6 (binned), B = 5 (two passes of the binned scratch): every d^2 and every partial sum is exact, so the
    result must EQUAL float32(exact_sum / n) for every transform: a dropped or doubled point changes the bits."""
    import pytorch_volumetric_b200 as pv
    n, B = 1_000_000, 5
    (v, f), world, w2o, mean = exact_cloud(n, B, seed=3)
    obj = pv.MeshObjectFactory("box12", mesh=(v, f))
    out = pv.batch_chamfer_dist(w2o.cuda(), world.cuda(), obj, scale=1.0).cpu().numpy()
    assert np.array_equal(out, np.full(B, np.float32(mean))), (out, np.float32(mean))
    # the same through the unbinned path (first 32 767 points)
    m = 32_767
    out_u = pv.batch_chamfer_dist(w2o.cuda(), world[:m].cuda(), obj, scale=1.0).cpu().numpy()
    q =cr.object_points(w2o[:1].numpy(), world[:m].numpy())[0]
    h = np.abs(q).max(axis=1) - 0.25
    assert np.array_equal(out_u, np.full(B, np.float32(float((h * h).sum()) / m)))


def _random_cloud(n, seed):
    """n points around the 64-triangle bumpy sphere and 5 transforms near identity."""
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(n, 3, generator=g, dtype=torch.float64) - 0.5) * 0.3).float()
    w2o = workloads.random_rigid(5, seed=seed, t_range=0.01)
    return pts, w2o


_CHILD = """
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import workloads, pytorch_volumetric_b200 as pv
v, f = workloads.bumpy_sphere(8, 5)
obj = pv.MeshObjectFactory("bumpy64", mesh=(v, f))
pts, w2o = torch.load({inp!r})
torch.save(pv.batch_chamfer_dist(w2o.cuda(), pts.cuda(), obj).cpu(), {out!r})
"""


def test_binned_sum_is_reproducible_and_equals_unbinned(objects, tmp_path):
    """Three calls on the same random 10^6-point cloud return the same bits, and they equal, bit for bit, the
    unbinned kernel's result (a process started with PVB_SORT_QUERIES=0, read once per process)."""
    import pytorch_volumetric_b200 as pv
    obj = objects["_mesh"][2]
    pts, w2o = _random_cloud(1_000_000, seed=9)
    outs = [pv.batch_chamfer_dist(w2o.cuda(), pts.cuda(), obj).cpu() for _ in range(3)]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), torch.stack(outs)
    inp, res = str(tmp_path / "in.pt"), str(tmp_path / "out.pt")
    torch.save((pts, w2o), inp)
    env = dict(os.environ, PVB_SORT_QUERIES="0")
    flags = ["-s"] if sys.flags.no_user_site else []
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), inp=inp, out=res)
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    unbinned = torch.load(res)
    assert torch.equal(outs[0], unbinned), (outs[0], unbinned)


# ------------------------------------------------------------------ pose-set metrics
def _pose_bound(spec, left, right, pts, scale=1000.0):
    """fp64 values and bound of the GPU path: the fp32 einsum of the composites, the kernel's transform, evaluation
    and sum."""
    comp = np.einsum("bij,pjk->bpik", np.asarray(left, np.float64), np.asarray(right, np.float64)).reshape(-1, 4, 4)
    d = cr.per_pair(spec, comp, pts)
    dd = cr.transform_error(comp, pts) + cr.composite_error(left, right, pts) + (
        MESH_EVAL if spec["kind"] == "mesh" else PRIM_EVAL)
    val = ((scale * d) ** 2).mean(axis=1)
    return val, cr.square_bound(d, dd, scale).mean(axis=1) + cr.sum_bound(len(pts), n_blk(len(pts))) * val


def _golden_bound(z, left, right, spec):
    """The reference's own fp32 error (tests/test_chamfer_ref_cpu.py) plus the GPU path's."""
    val, tol = _pose_bound(spec, left, right, z["pts"])
    return val, 2 * tol + (len(z["pts"]) + 4) * U * val


def test_pairwise_distance_chamfer_vs_reference_and_fp64():
    import pytorch_volumetric_b200 as pv
    z = golden("ref_chamfer_pairwise")
    obj = pv_factory("probe")
    spec = cr.mesh_spec(*workloads.fixture_mesh("probe"))
    pts = torch.from_numpy(z["pts"]).cuda()
    A, Bw = torch.from_numpy(z["A"]).cuda(), torch.from_numpy(z["B_w2l"]).cuda()
    # given B_world_to_link_tfs, |A| = 5 != |B| = 3
    e = pv.pairwise_distance_chamfer(A, Bw, obj_factory=obj, model_points_eval=pts)
    assert e.shape == (5, 3)
    val, tol = _pose_bound(spec, z["B_w2l"], z["A"], z["pts"])
    e = e.cpu().numpy().astype(np.float64).reshape(-1)
    assert (np.abs(e - val) <= tol).all(), (e, val)
    assert np.array_equal(val.reshape(5, 3), cr.pairwise_distance_chamfer(spec, z["pts"], z["A"], z["B_w2l"]))
    _, gtol = _golden_bound(z, z["B_w2l"], z["A"], spec)
    assert (np.abs(e - z["err_given"].reshape(-1)) <= gtol).all()
    # None: the inverses of A
    e0 = pv.pairwise_distance_chamfer(A, None, obj_factory=obj, model_points_eval=pts)
    assert e0.shape == (5, 5)
    inv = cr.rigid_inverse(z["A"])
    val0, tol0 = _pose_bound(spec, inv, z["A"], z["pts"])
    e0 = e0.cpu().numpy().astype(np.float64).reshape(-1)
    # invert_rigid runs in fp32: 3u of the inverse's translation on top
    tol0 = tol0 + cr.square_bound(np.sqrt(val0) / 1000.0, 3 * U * np.abs(z["A"][:, :3, 3]).sum(), 1000.0).max()
    assert (np.abs(e0 - val0) <= tol0).all(), (e0, val0)
    assert (np.abs(e0 - z["err_none"].reshape(-1)) <= 2 * tol0 + (len(z["pts"]) + 4) * U * val0).all()
    # obj_sdf given (a box), unequal sizes
    box = pv.BoxSDF([0.05, 0.03, 0.2])
    bspec = cr.primitive_spec(box.native_desc("cuda"))
    eb = pv.pairwise_distance_chamfer(A[:4], Bw[:2], obj_sdf=box, model_points_eval=pts)
    assert eb.shape == (4, 2)
    valb, tolb = _pose_bound(bspec, z["B_w2l"][:2], z["A"][:4], z["pts"])
    assert np.array_equal(valb.reshape(4, 2), cr.pairwise_distance_chamfer(bspec, z["pts"], z["A"][:4], z["B_w2l"][:2]))
    assert (np.abs(eb.cpu().numpy().astype(np.float64).reshape(-1) - valb) <= tolb).all()


@pytest.mark.parametrize("with_sdf", [False, True])
def test_plausible_diversity_vs_reference_and_fp64(with_sdf):
    import pytorch_volumetric_b200 as pv
    z = golden("ref_chamfer_pairwise")
    obj = pv_factory("probe")
    box = pv.BoxSDF([0.05, 0.03, 0.2])
    spec = cr.primitive_spec(box.native_desc("cuda")) if with_sdf else cr.mesh_spec(*workloads.fixture_mesh("probe"))
    Te, Tp = z["T_est_inv"], z["T_p"]
    pd = pv.PlausibleDiversity(obj, model_points_eval=torch.from_numpy(z["pts"]).cuda(),
                               obj_sdf=box if with_sdf else None)
    r1 = pd(torch.from_numpy(Te).cuda(), torch.from_numpy(Tp).cuda())
    r2 = pd(torch.from_numpy(Te).cuda(), torch.from_numpy(Tp).cuda(), bidirectional=True)
    pl, cov, best_est, best_pl = cr.plausible_diversity(spec, z["pts"], Te, Tp)
    pl2, cov2, _, _ = cr.plausible_diversity(spec, z["pts"], Te, Tp, bidirectional=True)
    _, t1 = _pose_bound(spec, Te, Tp, z["pts"])
    _, t2 = _pose_bound(spec, Tp, Te, z["pts"])
    t = max(t1.max(), t2.max())
    assert abs(float(r1.plausibility) - pl) <= t and abs(float(r1.coverage) - cov) <= t
    assert abs(float(r2.plausibility) - pl2) <= t and abs(float(r2.coverage) - cov2) <= t
    assert np.array_equal(r1.most_plausible_per_estimated.indices.cpu().numpy(), best_est)
    assert np.array_equal(r1.most_covered_per_plausible.indices.cpu().numpy(), best_pl)
    assert r1.most_plausible_per_estimated.values.shape == (4,) and r1.most_covered_per_plausible.values.shape == (6,)
    if not with_sdf:
        g = 2 * t + (len(z["pts"]) + 4) * U * max(pl, cov, pl2, cov2)
        assert abs(float(r1.plausibility) - z["pd_plausibility"]) <= g
        assert abs(float(r1.coverage) - z["pd_coverage"]) <= g
        assert abs(float(r2.plausibility) - z["pd2_plausibility"]) <= g
        assert abs(float(r2.coverage) - z["pd2_coverage"]) <= g
        assert np.array_equal(best_est, z["pd_best_est"]) and np.array_equal(best_pl, z["pd_best_pl"])
