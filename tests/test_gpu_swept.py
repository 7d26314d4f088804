"""GPU: swept composed queries (ComposedSDF.swept / query_swept, RobotSDF.swept, pvb_composed_query_swept).

At every point, the result of the first configuration attaining the minimum value over the slab.  Every result is
compared bit for bit -- values, gradients, configuration and sub-SDF -- with the reduction written here from the
per-configuration query(..., return_which=True)."""
import pytest
import torch

import workloads
from helpers import golden, pv_factory
from test_gpu_cached import _cached_from_golden
from test_gpu_paired import _golden_sets, _no_generic
from test_gpu_trilinear_composed import _arm, _arm_points, _opaque

pytestmark = pytest.mark.gpu


def _reduce(v, g, w, cfg_count, cfg_begin=0):
    """Lexicographic (value, configuration, sub-SDF) minimum of flat per-configuration results [cfg_count * P]."""
    P = v.numel() // cfg_count
    v, g, w = v.reshape(cfg_count, P), g.reshape(cfg_count, P, 3), w.reshape(cfg_count, P)
    c = (v == v.amin(dim=0)).int().argmax(dim=0)          # the first configuration attaining the minimum
    return (v.gather(0, c[None])[0], g.gather(0, c[None, :, None].expand(1, P, 3))[0],
            (c + cfg_begin).to(torch.int32), w.gather(0, c[None])[0])


def _reference(comp, pts, cfg_begin=0, cfg_count=None):
    n_cfg = 1 if comp.tsf_batch is None else int(torch.tensor(comp.tsf_batch).prod())
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    v, g, w = comp.query(pts, cfg_begin, cfg_count, return_which=True)
    return _reduce(v, g, w, cfg_count, cfg_begin)


def _assert_swept(comp, pts, cfg_begin=0, cfg_count=None, what=""):
    got = comp.query_swept(pts, cfg_begin, cfg_count, return_which=True)
    ref = _reference(comp, pts, cfg_begin, cfg_count)
    for a, b, name in zip(got, ref, ("val", "grad", "cfg", "which")):
        assert torch.equal(a, b), (what, name, int((a != b).reshape(len(a), -1).any(-1).sum()))
    return got


def test_golden_sets_fused(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = _golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    q = torch.from_numpy(z["q"]).cuda()
    for name, sdfs in sets.items():
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        _no_generic(monkeypatch, comp)
        _assert_swept(comp, q, what=name)
        _assert_swept(comp, q, cfg_begin=1, cfg_count=2, what=name)
        v, g = comp.swept(q)
        cv, cg = comp(q)
        assert torch.equal(v, cv.amin(0)) and v.shape == (len(q),) and g.shape == (len(q), 3), name


def _arm_robot(tmp_path, kind):
    import pytorch_volumetric_b200 as pv
    if kind == "primitive":
        urdf, end = workloads.write_primitive_arm(str(tmp_path / "prim"))
        return pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"),
                           primitive_visuals=True)
    return _arm(tmp_path, kind)


@pytest.mark.parametrize("kind", ["nearest", "trilinear", "primitive"])
def test_arm_fused(tmp_path, monkeypatch, kind):
    s = _arm_robot(tmp_path, kind)
    s.set_joint_configuration(workloads.arm_configurations(1000).cuda())
    _no_generic(monkeypatch, s.sdf)
    pts = _arm_points(5000, seed=11)
    for count in (1, 7, 31, 32, 33, 200, 1000):
        _assert_swept(s.sdf, pts, 0, count, what=(kind, count))
    for begin, count in ((3, 200), (500, 33), (999, 1)):
        got = _assert_swept(s.sdf, pts, begin, count, what=(kind, begin, count))
        assert int(got[2].min()) >= begin and int(got[2].max()) < begin + count
    # a 2-D configuration batch A = (4, 50): the flat row-major configuration index
    s.set_joint_configuration(workloads.arm_configurations(200).cuda().reshape(4, 50, -1))
    bp = _arm_points(2 * 3 * 700, seed=12).reshape(2, 3, 700, 3)
    v, g, c, w = s.swept(bp, return_argmin=True)
    assert v.shape == (2, 3, 700) and g.shape == (2, 3, 700, 3) and c.dtype == torch.int64 and w.shape == v.shape
    rv, rg, rc, rw = _reference(s.sdf, bp.reshape(-1, 3))
    assert torch.equal(v.reshape(-1), rv) and torch.equal(g.reshape(-1, 3), rg)
    assert torch.equal(c.reshape(-1), rc.long()) and torch.equal(w.reshape(-1), rw.long())
    cv, _ = s(bp)                                          # [4, 50, 2, 3, 700]
    assert torch.equal(v, cv.reshape(200, 2, 3, 700).amin(0))
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
        _no_generic(monkeypatch, comp)
        _assert_swept(comp, pts, what=obj.name)
        _assert_swept(comp, pts, 7, 20, what=obj.name)
    # 12 grid links (beyond the fused kernel's 8), and a grid with the LOOKUP_GT_SDF rule
    z, sets = _golden_sets(tmp_path)
    near = sets["nearest"][0]
    zc = golden("ref_cachedsdf_probe")
    gt = _cached_from_golden(zc, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    q = torch.from_numpy(z["q"]).cuda()
    for name, sdfs in (("12 links", [near] * 12), ("lookup-gt", [near, gt, near])):
        tm = workloads.random_rigid(len(sdfs) * A, seed=4, t_range=0.03).cuda()
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm))
        comp.set_transforms(comp.obj_frame_to_link_frame, batch_dim=(A,))
        _no_generic(monkeypatch, comp)
        _assert_swept(comp, q, what=name)
        _assert_swept(comp, q, 5, 33, what=name)
    # opaque sub-SDFs: the Python fold over _generic_query chunks
    s = _arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(150).cuda())
    opaque = pv.ComposedSDF(_opaque(pv, s.sdf.sdfs), s.sdf.obj_frame_to_link_frame)
    apts = _arm_points(2000, seed=13)
    _assert_swept(opaque, apts, what="opaque")
    _assert_swept(opaque, apts, 10, 100, what="opaque slab")


def test_semantics(tmp_path):
    from pytorch_volumetric_b200 import distributed as pd
    s = _arm(tmp_path, "nearest")
    # no configuration batch: swept == __call__, configuration 0
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    assert s.sdf.tsf_batch is None
    pts = _arm_points(3000, seed=14)
    v, g, c, w = s.swept(pts, return_argmin=True)
    cv, cg = s(pts)
    assert torch.equal(v, cv) and torch.equal(g, cg) and int(c.abs().max()) == 0
    s.set_joint_configuration(workloads.arm_configurations(64).cuda())
    # host in, host out; fp64 in, fp64 out
    vd, gd = s.swept(pts)
    vh, gh = s.swept(pts.cpu())
    assert vh.device.type == "cpu" and torch.equal(vh, vd.cpu()) and torch.equal(gh, gd.cpu())
    v64, g64 = s.swept(pts.cpu().double())
    assert v64.dtype == torch.float64 and torch.equal(v64, vd.cpu().double()) and torch.equal(g64, gd.cpu().double())
    # no points
    v0, g0 = s.swept(torch.empty(0, 3, device="cuda"))
    assert v0.shape == (0,) and g0.shape == (0, 3)
    # sharding the points over one rank
    pb = pts.reshape(3, 1000, 3)
    vs, gs = pd.sharded_query(s.swept, pb)
    vr, gr = s.swept(pb)
    assert torch.equal(vs, vr) and torch.equal(gs, gr)


def test_capability_4096_by_a_million(tmp_path):
    """A = 4096, N = 10^6 on the 8-link arm: the cross product (65.5 GB) does not fit beside anything else; the swept
    query needs the points and the N-sized outputs only.  Compared with the fold of 256-configuration query slabs."""
    s = _arm(tmp_path, "nearest")
    A, N = 4096, 1_000_000
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    pts = _arm_points(N, seed=15)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = s.sdf.query_swept(pts, return_which=True)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 40 << 20, extra                          # the outputs are 24 MB
    best = None
    for b in range(0, A, 256):
        v, g, w = s.sdf.query(pts, b, 256, return_which=True)
        cand = _reduce(v, g, w, 256, b)
        del v, g, w
        if best is None:
            best = list(cand)
        else:
            better = cand[0] < best[0]
            for k in range(4):
                best[k] = torch.where(better[:, None] if k == 1 else better, cand[k], best[k])
    for a, b, name in zip(got, best, ("val", "grad", "cfg", "which")):
        assert torch.equal(a, b), name
