"""GPU: paired clearance queries (ComposedSDF.paired_clearance / query_paired_clearance, RobotSDF.paired_clearance,
pvb_composed_query_paired_clearance).

Every configuration against its own cloud: for every segment of its points, the result at the first point attaining
the minimum value.  Every result is compared bit for bit -- values, gradients, point index and sub-SDF -- with the
first-point reduction of query_paired(..., return_which=True) over each segment, and where it matters with the
per-configuration query_clearance."""
import pytest
import torch

import workloads
from helpers import (arm_points, arm_robot, cached_arm, cached_from_golden, clearance_reduce, golden, golden_sets,
                     no_generic, opaque_sdfs, own_points, pv_factory)

pytestmark = pytest.mark.gpu


def _reference(comp, own, cfg_begin=0, cfg_count=None):
    """own [cfg_count, *B, N, 3]: the first-point reduction of the paired query over every segment."""
    cfg_count = own.shape[0] if cfg_count is None else cfg_count
    N = own.shape[-2]
    n_seg = own.numel() // (3 * N * cfg_count)
    v, g, w = comp.query_paired(own, cfg_begin, cfg_count, return_which=True)
    return clearance_reduce(v, g, w, cfg_count, n_seg)


def _assert_pc(comp, own, cfg_begin=0, cfg_count=None, what=""):
    got = comp.query_paired_clearance(own, cfg_begin, cfg_count, return_which=True)
    ref = _reference(comp, own, cfg_begin, cfg_count)
    for a, b, name in zip(got, ref, ("val", "grad", "point", "which")):
        assert torch.equal(a, b), (what, name, int((a != b).reshape(len(a), -1).any(-1).sum()))
    return got


def _assert_equals_per_configuration(comp, own, cfg_begin, configs, got, what=""):
    """Entry c * n_seg + b == query_clearance(own[c], cfg_begin + c, 1)[b] (mesh jitter included)."""
    n_seg = len(got[0]) // own.shape[0]
    for c in configs:
        one = comp.query_clearance(own[c], cfg_begin + c, 1, return_which=True)
        for a, b, name in zip(got, one, ("val", "grad", "point", "which")):
            assert torch.equal(a[c * n_seg:(c + 1) * n_seg], b), (what, c, name)


def test_golden_sets_fused(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    own = own_points(torch.from_numpy(z["q"]), A, 0)
    own = own[:, :(own.shape[1] // 6) * 6]
    for name, sdfs in sets.items():
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        no_generic(monkeypatch, comp)
        got = _assert_pc(comp, own, what=name)
        _assert_equals_per_configuration(comp, own, 0, range(A), got, what=name)
        seg = own.reshape(A, 6, -1, 3)
        _assert_pc(comp, seg[1:3], cfg_begin=1, cfg_count=2, what=name)
        v, g = comp.paired_clearance(seg)
        pv_, _ = comp.paired(seg)
        assert torch.equal(v, pv_.amin(-1)) and v.shape == (A, 6) and g.shape == (A, 6, 3), name


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_arm_fused(tmp_path, monkeypatch, kind):
    s = arm_robot(tmp_path, kind)
    s.set_joint_configuration(workloads.arm_configurations(1000).cuda())
    no_generic(monkeypatch, s.sdf)
    pts = arm_points(1000 * 600, seed=31).reshape(1000, 600, 3)
    for count in (1, 7, 31, 32, 33, 200, 1000):
        _assert_pc(s.sdf, pts[:count], 0, count, what=(kind, count))
    for begin, count in ((3, 200), (500, 33), (999, 1)):
        got = _assert_pc(s.sdf, pts[begin:begin + count].reshape(count, 3, 200, 3), begin, count,
                         what=(kind, begin, count))
        _assert_equals_per_configuration(s.sdf, pts[begin:begin + count].reshape(count, 3, 200, 3), begin,
                                         (0, count - 1), got, what=(kind, begin))
    # segment shapes: N = 6000, B = (2, 3), N = 5 and N = 1
    big = arm_points(20 * 6000, seed=32).reshape(20, 6000, 3)
    _assert_pc(s.sdf, big, 0, 20, what=(kind, "N=6000"))
    _assert_pc(s.sdf, pts[:200].reshape(200, 2, 3, 100, 3), 0, 200, what=(kind, "B=(2,3)"))
    _assert_pc(s.sdf, pts[:33].reshape(33, 120, 5, 3), 0, 33, what=(kind, "N=5"))
    _assert_pc(s.sdf, pts[:40].reshape(40, 600, 1, 3), 0, 40, what=(kind, "N=1"))
    # RobotSDF delegates; the link index is a position in sdf_to_link_name
    v, g, i, w = s.paired_clearance(pts, return_argmin=True)
    rv, rg, ri, rw = _reference(s.sdf, pts)
    assert v.shape == (1000,) and g.shape == (1000, 3) and i.dtype == torch.int64 and w.dtype == torch.int64
    assert torch.equal(v, rv) and torch.equal(g, rg) and torch.equal(i, ri.long()) and torch.equal(w, rw.long())
    assert 0 <= int(w.min()) and int(w.max()) < len(s.sdf_to_link_name)


def test_seventy_thousand_configurations(tmp_path, monkeypatch):
    """70 000 configurations x 16 points: more configuration tiles than a grid row can hold, on the fused route."""
    s = cached_arm(tmp_path, "nearest")
    A = 70_000
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    no_generic(monkeypatch, s.sdf)
    pts = arm_points(A * 16, seed=33).reshape(A, 16, 3)
    got = _assert_pc(s.sdf, pts, what="70000")
    _assert_equals_per_configuration(s.sdf, pts, 0, (0, 65_535, 65_536, A - 1), got, what="70000")


def test_generic_route(tmp_path, monkeypatch):
    """Meshes (closed and open: ray jitter), 12 grid links, a LOOKUP_GT_SDF grid, 129 sub-SDFs and an opaque Python
    sub-SDF."""
    import pytorch_volumetric_b200 as pv
    v_, f_ = workloads.fixture_mesh("probe")
    open_probe = pv.MeshObjectFactory("probe_open", mesh=(v_, f_[: len(f_) - len(f_) // 5]))
    drill = pv_factory("drill")
    A, P = 40, 600
    own = (torch.rand(A, P, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda() * 0.15
    for obj in (drill, open_probe):
        tm = torch.eye(4).repeat(2 * A, 1, 1)
        tm[:, :3, 3] = 0.05 * torch.randn(2 * A, 3, generator=torch.Generator().manual_seed(2))
        comp = pv.ComposedSDF([pv.MeshSDF(obj), pv.MeshSDF(obj)], pv.Transform3d(matrix=tm.cuda()))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        no_generic(monkeypatch, comp)
        got = _assert_pc(comp, own, what=obj.name)
        _assert_equals_per_configuration(comp, own, 0, range(A), got, what=obj.name)
        sub = own[7:27].reshape(20, 6, 100, 3)
        got = _assert_pc(comp, sub, 7, 20, what=obj.name)
        _assert_equals_per_configuration(comp, sub, 7, (0, 19), got, what=obj.name)
    z, sets = golden_sets(tmp_path)
    near = sets["nearest"][0]
    zc = golden("ref_cachedsdf_probe")
    gt = cached_from_golden(zc, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    gown = own_points(torch.from_numpy(z["q"]), A, 1)
    gown = gown[:, :(gown.shape[1] // 10) * 10]
    for name, sdfs in (("12 links", [near] * 12), ("lookup-gt", [near, gt, near])):
        tm = workloads.random_rigid(len(sdfs) * A, seed=4, t_range=0.03).cuda()
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        no_generic(monkeypatch, comp)
        _assert_pc(comp, gown, what=name)
        _assert_pc(comp, gown[5:38].reshape(33, 10, -1, 3), 5, 33, what=name)
    # more than 128 sub-SDFs and opaque sub-SDFs: the Python reduction over _generic_query chunks
    tm = workloads.random_rigid(129 * 4, seed=5, t_range=0.03).cuda()
    many = pv.ComposedSDF([near] * 129, pv.Transform3d(matrix=tm))
    many.set_transforms(many.obj_frame_to_link_frame, batch_dim=(4,))
    _assert_pc(many, gown[:4].reshape(4, 2, -1, 3), what="129")
    s = cached_arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(150).cuda())
    opaque = pv.ComposedSDF(opaque_sdfs(pv, s.sdf.sdfs), s.sdf.obj_frame_to_link_frame)
    apts = arm_points(150 * 400, seed=34).reshape(150, 400, 3)
    got = _assert_pc(opaque, apts, what="opaque")
    _assert_pc(opaque, apts[10:110].reshape(100, 4, 100, 3), 10, 100, what="opaque slab")
    # the opaque path names the fused route's points, values and links (its gradient is rotated back by a torch
    # matmul instead of the kernels' composed_rotate_back, as in test_gpu_trilinear_composed)
    fused = s.sdf.query_paired_clearance(apts, return_which=True)
    assert torch.equal(got[0], fused[0]) and torch.equal(got[2], fused[2]) and torch.equal(got[3], fused[3])
    assert float((got[1] - fused[1]).abs().max()) < 1e-6


def test_semantics(tmp_path):
    s = cached_arm(tmp_path, "nearest")
    pts = arm_points(200 * 3 * 500, seed=35)
    # no configuration batch: clearance()
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    assert s.sdf.tsf_batch is None
    one = pts[:1500].reshape(3, 500, 3)
    for a, b in zip(s.paired_clearance(one, return_argmin=True), s.clearance(one, return_argmin=True)):
        assert torch.equal(a, b)
    # a 2-D configuration batch A = (4, 50): against paired() followed by amin, and per-configuration query_clearance
    s.set_joint_configuration(workloads.arm_configurations(200).cuda().reshape(4, 50, -1))
    own = pts.reshape(4, 50, 3, 500, 3)
    v, g, i, w = s.paired_clearance(own, return_argmin=True)
    assert v.shape == (4, 50, 3) and g.shape == (4, 50, 3, 3) and i.shape == v.shape and w.shape == v.shape
    pv_, pg = s.paired(own)                                         # [4, 50, 3, 500]
    assert torch.equal(v, pv_.amin(-1))
    assert torch.equal(g, pg.gather(-2, i[..., None, None].expand(4, 50, 3, 1, 3))[..., 0, :])
    flat = own.reshape(200, 3, 500, 3)
    got = (v.reshape(-1), g.reshape(-1, 3), i.reshape(-1).int(), w.reshape(-1).int())
    _assert_equals_per_configuration(s.sdf, flat, 0, (0, 1, 77, 199), got, what="2-D batch")
    # host in, host out; fp64 in, fp64 out
    vh, gh = s.paired_clearance(own.cpu())
    assert vh.device.type == "cpu" and torch.equal(vh, v.cpu()) and torch.equal(gh, g.cpu())
    v64, g64 = s.paired_clearance(own.cpu().double())
    assert v64.dtype == torch.float64 and torch.equal(v64, v.cpu().double()) and torch.equal(g64, g.cpu().double())
    # repeated calls: identical bits
    for _ in range(3):
        again = s.paired_clearance(own, return_argmin=True)
        assert all(torch.equal(a, b) for a, b in zip(again, (v, g, i, w)))
    # no segments; empty segments raise before any device work
    v0, g0 = s.paired_clearance(torch.empty(4, 50, 0, 7, 3, device="cuda"))
    assert v0.shape == (4, 50, 0) and g0.shape == (4, 50, 0, 3)
    with pytest.raises(ValueError, match="empty segment"):
        s.paired_clearance(torch.empty(4, 50, 2, 0, 3, device="cuda"))
    with pytest.raises(ValueError, match="leading"):
        s.paired_clearance(own.reshape(200, 3, 500, 3))
