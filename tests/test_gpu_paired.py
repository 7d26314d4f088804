"""GPU: paired composed queries (ComposedSDF.paired / query_paired, RobotSDF.paired, pvb_composed_query_paired).

Configuration a is evaluated at its own points only.  The results are bit-identical to what the library already
answers: the diagonal of __call__ for grid and sphere sets, and the per-configuration slab query
query(points[a], cfg_begin=a, cfg_count=1) for every set, mesh ray jitter included."""
import pytest
import torch

import workloads
from helpers import golden, pv_factory
from test_gpu_cached import _cached_from_golden
from test_gpu_trilinear_composed import _arm, _arm_points, _opaque

pytestmark = pytest.mark.gpu


def _no_generic(monkeypatch, comp):
    def boom(*a, **k):
        raise AssertionError("generic path taken")
    monkeypatch.setattr(comp, "_generic_query", boom)


def _assert_equals_slab_queries(comp, own, which=True):
    """query_paired(own [A, P, 3]) == query(own[a], cfg_begin=a, cfg_count=1) for every a, bit for bit."""
    A, P = own.shape[0], own.shape[1]
    v, g, w = comp.query_paired(own, return_which=True)
    for a in range(A):
        v1, g1, w1 = comp.query(own[a], cfg_begin=a, cfg_count=1, return_which=True)
        sl = slice(a * P, (a + 1) * P)
        assert torch.equal(v[sl], v1) and torch.equal(g[sl], g1), a
        if which:
            assert torch.equal(w[sl], w1), a
    return v, g, w


def _own_points(q, A, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = q.cpu()
    return torch.stack([q[torch.randperm(len(q), generator=g)] + 0.01 * torch.randn(3, generator=g)
                        for _ in range(A)]).cuda()


def _golden_sets(tmp_path):
    import pytorch_volumetric_b200 as pv
    zc = golden("ref_cachedsdf_probe")
    near = _cached_from_golden(zc, "probe", tmp_path)
    tri = _cached_from_golden(zc, "probe", tmp_path, interpolation="trilinear")
    z = golden("ref_composed")
    sph = pv.SphereSDF(float(z["sphere_radius"]))
    return z, {"nearest": [near, near, near, near], "trilinear": [tri, tri, tri], "mixed": [near, tri, near],
               "nearest+sphere": [near, near, sph, near], "mixed+sphere": [tri, near, sph, tri]}


def test_golden_paired_equals_the_call_diagonal(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    z, sets = _golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    own = _own_points(torch.from_numpy(z["q"]), A, 0)
    P = own.shape[1]
    for name, sdfs in sets.items():
        S = len(sdfs)
        comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tm[[s % S0 for s in range(S)]].reshape(S * A, 4, 4)))
        _no_generic(monkeypatch, comp)
        v, g = comp.paired(own)
        assert v.shape == (A, P) and g.shape == (A, P, 3)
        cv, cg = comp(own)                                     # [A, A, P]: every configuration at every block
        idx = torch.arange(A)
        assert torch.equal(v, cv[idx, idx]) and torch.equal(g, cg[idx, idx]), name
        _, _, w = comp.query_paired(own, return_which=True)
        _, _, cw = comp.query(own.reshape(-1, 3), return_which=True)
        assert torch.equal(w.reshape(A, P), cw.reshape(A, A, P)[idx, idx]), name
        _assert_equals_slab_queries(comp, own)


def test_mesh_paired_equals_slab_queries(monkeypatch):
    """Closed drill (the exact axis parity walk) and an open mesh (the reference's jittered diagonal ray, seeded by
    the absolute configuration index)."""
    import pytorch_volumetric_b200 as pv
    v_, f_ = workloads.fixture_mesh("probe")
    open_probe = pv.MeshObjectFactory("probe_open", mesh=(v_, f_[: len(f_) - len(f_) // 5]))
    drill = pv_factory("drill")
    assert drill.is_closed and not open_probe.is_closed
    A, P = 5, 700
    for obj, span in ((drill, 0.15), (open_probe, 0.05)):
        tm = torch.eye(4).repeat(2 * A, 1, 1)
        tm[:, :3, 3] = 0.3 * span * torch.randn(2 * A, 3, generator=torch.Generator().manual_seed(2))
        comp = pv.ComposedSDF([pv.MeshSDF(obj), pv.MeshSDF(obj)], pv.Transform3d(matrix=tm.cuda()))
        _no_generic(monkeypatch, comp)
        own = (torch.rand(A, P, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).cuda() * span
        _assert_equals_slab_queries(comp, own)
        # a slab of configurations keeps the absolute jitter index
        v, g = comp.query_paired(own[2:4], cfg_begin=2, cfg_count=2)
        v_all, g_all = comp.query_paired(own)
        assert torch.equal(v, v_all[2 * P:4 * P]) and torch.equal(g, g_all[2 * P:4 * P])


@pytest.mark.parametrize("scaled", [False, True])
def test_arm_paired_equals_slab_queries(tmp_path, monkeypatch, scaled):
    """8-link arm at A = 200, P = 4096 (the point-serial robot kernel answers the slab queries' cross product, the
    point-major kernel the single-configuration ones), and with non-rigid (scaled) transforms."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.transforms import matrix_of
    s = _arm(tmp_path, "nearest")
    A, P = 200, 4096
    s.set_joint_configuration(workloads.arm_configurations(A).cuda())
    comp = s.sdf
    if scaled:
        S = len(comp.sdfs)
        M = matrix_of(comp.obj_frame_to_link_frame).detach().clone().reshape(S, A, 4, 4)
        M[:, 5:13, :3, :3] *= 1.03
        M[3, 20:26, :3, :3] *= 0.97
        M[0, 150:, :3, :3] *= 1.02
        comp = pv.ComposedSDF(comp.sdfs, pv.Transform3d(matrix=M.reshape(S * A, 4, 4)))
    _no_generic(monkeypatch, comp)
    own = torch.stack([_arm_points(P, seed=100 + a) for a in range(A)])
    _assert_equals_slab_queries(comp, own)
    if not scaled:
        v, g = s.paired(own)                                   # RobotSDF delegates to its ComposedSDF
        v2, g2 = comp.query_paired(own)
        assert v.shape == (A, P) and torch.equal(v.reshape(-1), v2) and torch.equal(g.reshape(-1, 3), g2)


def test_edge_shapes(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    s = _arm(tmp_path, "nearest")
    _no_generic(monkeypatch, s.sdf)
    s.set_joint_configuration(workloads.arm_configurations(7).cuda())
    base = _arm_points(7 * 3 * 5 + 1, seed=5)
    for P in (1, 3):
        _assert_equals_slab_queries(s.sdf, base[:7 * P].reshape(7, P, 3))
    # a misaligned view: points start 4 bytes into the buffer
    mis = base.reshape(-1)[1:1 + 7 * 5 * 3].view(7, 5, 3)
    assert mis.data_ptr() % 16 != 0
    v, g = s.paired(mis)
    v_ref, g_ref = s.paired(mis.clone())
    assert torch.equal(v, v_ref) and torch.equal(g, g_ref)
    _assert_equals_slab_queries(s.sdf, mis)
    # P = 0
    v, g = s.paired(torch.empty(7, 0, 3, device="cuda"))
    assert v.shape == (7, 0) and g.shape == (7, 0, 3)
    # host tensors in, host tensors out, equal to the device result
    hp = base[:7 * 5].reshape(7, 5, 3)
    vd, gd = s.paired(hp)
    vh, gh = s.paired(hp.cpu())
    assert vh.device.type == "cpu" and torch.equal(vh, vd.cpu()) and torch.equal(gh, gd.cpu())
    vh64, _ = s.paired(hp.cpu().double())
    assert vh64.dtype == torch.float64 and torch.equal(vh64, vd.cpu().double())
    # a 2-D configuration batch [2, 3] with extra *B dimensions: points [2, 3, 4, 5, 3] -> [2, 3, 4, 5]
    s.set_joint_configuration(workloads.arm_configurations(6).cuda().reshape(2, 3, -1))
    pts = _arm_points(6 * 20, seed=6).reshape(2, 3, 4, 5, 3)
    v, g = s.paired(pts)
    assert v.shape == (2, 3, 4, 5) and g.shape == (2, 3, 4, 5, 3)
    flat_v, flat_g = s.sdf.query_paired(pts.reshape(6, 20, 3))
    assert torch.equal(v.reshape(-1), flat_v) and torch.equal(g.reshape(-1, 3), flat_g)
    with pytest.raises(ValueError):
        s.paired(pts.reshape(3, 2, 4, 5, 3))
    # A = 1, and no configuration batch at all: paired == __call__
    s.set_joint_configuration(workloads.arm_configurations(1).cuda())
    pts = _arm_points(300, seed=7).reshape(1, 300, 3)
    v, g = s.paired(pts)
    cv, cg = s(pts)
    assert torch.equal(v, cv[0]) and torch.equal(g, cg[0])
    s.set_joint_configuration(workloads.arm_configurations(1)[0].cuda())
    assert s.sdf.tsf_batch is None
    pts = _arm_points(300, seed=8)
    v, g = s.paired(pts)
    cv, cg = s(pts)
    assert torch.equal(v, cv) and torch.equal(g, cg)


def test_generic_route_equals_fused(tmp_path):
    """Opaque sub-SDFs (no native descriptor) take the unfused paired path: values and argmin equal the fused path
    exactly, gradients within 1e-6 (torch matmul instead of FMAs for the rotation back)."""
    import pytorch_volumetric_b200 as pv
    z, sets = _golden_sets(tmp_path)
    S0, A = int(z["S"]), int(z["A"])
    tm = torch.from_numpy(z["tmat"]).cuda().reshape(S0, A, 4, 4)
    own = _own_points(torch.from_numpy(z["q"]), A, 1)
    for name in ("nearest+sphere", "mixed+sphere"):
        sdfs = sets[name]
        tsf = pv.Transform3d(matrix=tm.reshape(S0 * A, 4, 4))
        vf, gf, wf = pv.ComposedSDF(sdfs, tsf).query_paired(own, return_which=True)
        vg, gg, wg = pv.ComposedSDF(_opaque(pv, sdfs), tsf).query_paired(own, return_which=True)
        assert torch.equal(vf, vg) and torch.equal(wf, wg), name
        assert float((gf - gg).abs().max()) < 1e-6, name
    s = _arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(40).cuda())
    own = torch.stack([_arm_points(1000, seed=200 + a) for a in range(40)])
    tsf = s.sdf.obj_frame_to_link_frame
    vf, gf, wf = pv.ComposedSDF(s.sdf.sdfs, tsf).query_paired(own, return_which=True)
    vg, gg, wg = pv.ComposedSDF(_opaque(pv, s.sdf.sdfs), tsf).query_paired(own, return_which=True)
    assert torch.equal(vf, vg) and torch.equal(wf, wg)
    assert float((gf - gg).abs().max()) < 1e-6


def test_trilinear_with_lookup_gt_is_refused(tmp_path):
    """CachedSDF refuses the combination at construction; a descriptor that carries it anyway is refused by the
    paired entry point as by the composed one."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import _native as nat
    zc = golden("ref_cachedsdf_probe")
    tri = _cached_from_golden(zc, "probe", tmp_path, interpolation="trilinear")

    class TriGt(pv.ObjectFrameSDF):
        def __call__(self, p):
            return tri(p)

        def surface_bounding_box(self, **kw):
            return tri.surface_bounding_box(**kw)

        def native_desc(self, device):
            d = tri.native_desc(device).copy()
            d.flags |= nat.PVB_GRID_OOB_GT
            return d

    comp = pv.ComposedSDF([TriGt(), TriGt()], pv.Transform3d(matrix=torch.eye(4, device="cuda").repeat(4, 1, 1)))
    NativeLibraryError = nat.NativeLibraryError
    pts = torch.zeros(2, 10, 3, device="cuda")
    with pytest.raises(NativeLibraryError, match="bounding-box"):
        comp.query(pts[0])
    with pytest.raises(NativeLibraryError, match="bounding-box"):
        comp.paired(pts)


def test_sharded_paired_single_rank(tmp_path):
    from pytorch_volumetric_b200 import distributed as pd
    s = _arm(tmp_path, "nearest")
    s.set_joint_configuration(workloads.arm_configurations(12).cuda().reshape(3, 4, -1))
    pts = _arm_points(12 * 50, seed=9).reshape(3, 4, 5, 10, 3)
    v_ref, g_ref = s.paired(pts)
    v, g = pd.sharded_robot_query(s, pts, gather=True, paired=True)
    assert torch.equal(v, v_ref) and torch.equal(g, g_ref)
    v, g, (b, e) = pd.sharded_robot_query(s, pts, gather=False, paired=True)
    assert (b, e) == (0, 12) and torch.equal(v, v_ref.reshape(12, 50))
