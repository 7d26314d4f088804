"""GPU: clearance queries (ComposedSDF.clearance / query_clearance, RobotSDF.clearance, pvb_composed_query_clearance).

For every configuration and every segment of points, the result at the first point attaining the minimum value.
Every result is compared bit for bit -- values, gradients, point index and sub-SDF -- with the reduction written here
from the per-configuration query(..., return_which=True)."""
import pytest
import torch

import workloads
from helpers import (arm_points, arm_robot, cached_arm, cached_from_golden, clearance_reduce, golden, golden_sets,
                     no_generic, opaque_sdfs, pv_factory)

pytestmark = pytest.mark.gpu


def _reference(comp, pts, cfg_begin=0, cfg_count=None):
    n_cfg = 1 if comp.tsf_batch is None else int(torch.tensor(comp.tsf_batch).prod())
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    n_seg = pts.reshape(-1, pts.shape[-2], 3).shape[0]
    v, g, w = comp.query(pts.reshape(-1, 3), cfg_begin, cfg_count, return_which=True)
    return clearance_reduce(v, g, w, cfg_count, n_seg)


def _assert_clearance(comp, pts, cfg_begin=0, cfg_count=None, what=""):
    got = comp.query_clearance(pts, cfg_begin, cfg_count, return_which=True)
    ref = _reference(comp, pts, cfg_begin, cfg_count)
    for a, b, name in zip(got, ref, ("val", "grad", "point", "which")):
        assert torch.equal(a, b), (what, name, int((a != b).reshape(len(a), -1).any(-1).sum()))
    return got


def test_golden_sets_fused(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    q = torch.from_numpy(z["q"]).cuda()
    for name, sdfs in sets.items():
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        no_generic(monkeypatch, comp)
        _assert_clearance(comp, q, what=name)
        _assert_clearance(comp, q.reshape(6, 500, 3), cfg_begin=1, cfg_count=2, what=name)
        v, g = comp.clearance(q.reshape(2, 3, 500, 3))
        cv, cg = comp(q.reshape(2, 3, 500, 3))
        assert torch.equal(v, cv.amin(-1)) and v.shape == (A, 2, 3) and g.shape == (A, 2, 3, 3), name


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_arm_fused(tmp_path, monkeypatch, kind):
    s = arm_robot(tmp_path, kind)
    s.set_joint_configuration(workloads.arm_configurations(1000).cuda())
    no_generic(monkeypatch, s.sdf)
    pts = arm_points(6000, seed=21)
    for count in (1, 7, 31, 32, 33, 200, 1000):
        _assert_clearance(s.sdf, pts, 0, count, what=(kind, count))
    for begin, count in ((3, 200), (500, 33), (999, 1)):
        _assert_clearance(s.sdf, pts.reshape(3, 2000, 3), begin, count, what=(kind, begin, count))
    # B = (2, 3) segments, and tiny segments (N = 1 and 5) with many of them
    _assert_clearance(s.sdf, pts.reshape(2, 3, 1000, 3), 0, 200, what=(kind, "B=(2,3)"))
    _assert_clearance(s.sdf, pts.reshape(1200, 5, 3), 0, 33, what=(kind, "N=5"))
    _assert_clearance(s.sdf, pts[:1500].reshape(1500, 1, 3), 0, 40, what=(kind, "N=1"))
    # a 2-D configuration batch A = (4, 50)
    s.set_joint_configuration(workloads.arm_configurations(200).cuda().reshape(4, 50, -1))
    bp = pts.reshape(2, 3, 1000, 3)
    v, g, i, w = s.clearance(bp, return_argmin=True)
    assert v.shape == (4, 50, 2, 3) and g.shape == (4, 50, 2, 3, 3) and i.dtype == torch.int64 and w.shape == v.shape
    rv, rg, ri, rw = _reference(s.sdf, bp)
    assert torch.equal(v.reshape(-1), rv) and torch.equal(g.reshape(-1, 3), rg)
    assert torch.equal(i.reshape(-1), ri.long()) and torch.equal(w.reshape(-1), rw.long())
    cv, _ = s(bp)                                          # [4, 50, 2, 3, 1000]
    assert torch.equal(v, cv.amin(-1))
    assert 0 <= int(w.min()) and int(w.max()) < len(s.sdf_to_link_name)


def test_generic_route(tmp_path, monkeypatch):
    """Meshes (closed and open), 12 grid links, a LOOKUP_GT_SDF grid and an opaque Python sub-SDF."""
    import pytorch_volumetric_b200 as pv
    v_, f_ = workloads.fixture_mesh("probe")
    open_probe = pv.MeshObjectFactory("probe_open", mesh=(v_, f_[: len(f_) - len(f_) // 5]))
    drill = pv_factory("drill")
    A, P = 40, 3000
    pts = (torch.rand(P, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda() * 0.15
    for obj in (drill, open_probe):
        tm = torch.eye(4).repeat(2 * A, 1, 1)
        tm[:, :3, 3] = 0.05 * torch.randn(2 * A, 3, generator=torch.Generator().manual_seed(2))
        comp = pv.ComposedSDF([pv.MeshSDF(obj), pv.MeshSDF(obj)], pv.Transform3d(matrix=tm.cuda()))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        no_generic(monkeypatch, comp)
        _assert_clearance(comp, pts, what=obj.name)
        _assert_clearance(comp, pts.reshape(6, 500, 3), 7, 20, what=obj.name)
    z, sets = golden_sets(tmp_path)
    near = sets["nearest"][0]
    zc = golden("ref_cachedsdf_probe")
    gt = cached_from_golden(zc, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    q = torch.from_numpy(z["q"]).cuda()
    for name, sdfs in (("12 links", [near] * 12), ("lookup-gt", [near, gt, near])):
        tm = workloads.random_rigid(len(sdfs) * A, seed=4, t_range=0.03).cuda()
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        no_generic(monkeypatch, comp)
        _assert_clearance(comp, q, what=name)
        _assert_clearance(comp, q.reshape(10, 300, 3), 5, 33, what=name)
    # opaque sub-SDFs: the Python reduction over _generic_query chunks
    s = cached_arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(150).cuda())
    opaque = pv.ComposedSDF(opaque_sdfs(pv, s.sdf.sdfs), s.sdf.obj_frame_to_link_frame)
    apts = arm_points(2000, seed=23)
    _assert_clearance(opaque, apts, what="opaque")
    _assert_clearance(opaque, apts.reshape(4, 500, 3), 10, 100, what="opaque slab")


def test_semantics(tmp_path):
    from pytorch_volumetric_b200 import distributed as pd
    s = cached_arm(tmp_path, "nearest")
    pts = arm_points(3000, seed=24)
    # no configuration batch: [*B]
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    assert s.sdf.tsf_batch is None
    v, g, i, w = s.clearance(pts.reshape(3, 1000, 3), return_argmin=True)
    cv, cg = s(pts.reshape(3, 1000, 3))
    cv, cg = cv.reshape(3, 1000), cg.reshape(3, 1000, 3)         # __call__ without a batch: flat results
    assert v.shape == (3,) and g.shape == (3, 3) and torch.equal(v, cv.amin(-1))
    assert torch.equal(g, cg.gather(-2, i[:, None, None].expand(3, 1, 3))[:, 0])
    s.set_joint_configuration(workloads.arm_configurations(64).cuda())
    # host in, host out; fp64 in, fp64 out
    vd, gd = s.clearance(pts.reshape(3, 1000, 3))
    vh, gh = s.clearance(pts.reshape(3, 1000, 3).cpu())
    assert vh.device.type == "cpu" and torch.equal(vh, vd.cpu()) and torch.equal(gh, gd.cpu())
    v64, g64 = s.clearance(pts.reshape(3, 1000, 3).cpu().double())
    assert v64.dtype == torch.float64 and torch.equal(v64, vd.cpu().double()) and torch.equal(g64, gd.cpu().double())
    # clearance == robot(points).amin(-1)
    cv, _ = s(pts.reshape(3, 1000, 3))
    assert vd.shape == (64, 3) and torch.equal(vd, cv.amin(-1))
    # no segments; empty segments raise before any device work
    v0, g0 = s.clearance(torch.empty(0, 7, 3, device="cuda"))
    assert v0.shape == (64, 0) and g0.shape == (64, 0, 3)
    with pytest.raises(ValueError, match="empty segment"):
        s.clearance(torch.empty(4, 0, 3, device="cuda"))
    # configuration slabs over one rank
    pb = pts.reshape(3, 1000, 3)
    vs, gs = pd.sharded_robot_query(s, pb, clearance=True)
    assert torch.equal(vs, vd) and torch.equal(gs, gd)
    lv, lg, rng = pd.sharded_robot_query(s, pb, gather=False, clearance=True)
    assert rng == (0, 64) and torch.equal(lv.reshape(-1), vd.reshape(-1)) and lg.shape == (64, 3, 3)


def test_capability_4096_by_a_million(tmp_path):
    """A = 4096, N = 10^6 on the 8-link arm: the cross product (65.5 GB) does not fit beside anything else; the
    clearance query needs the points, the |A|-sized outputs and keys only.  Compared with the reduction of
    256-configuration query slabs."""
    s = cached_arm(tmp_path, "nearest")
    A, N = 4096, 1_000_000
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    pts = arm_points(N, seed=25)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = s.sdf.query_clearance(pts, return_which=True)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    outputs = A * (4 + 12 + 4 + 4 + 8)                     # value, gradient, point, link, key
    assert extra < outputs + (4 << 20), extra
    ref = [[] for _ in range(4)]
    for b in range(0, A, 256):
        v, g, w = s.sdf.query(pts, b, 256, return_which=True)
        for k, t in enumerate(clearance_reduce(v, g, w, 256, 1)):
            ref[k].append(t)
        del v, g, w
    for a, b, name in zip(got, [torch.cat(r) for r in ref], ("val", "grad", "point", "which")):
        assert torch.equal(a, b), name
