"""GPU: trilinear CachedSDF links (CachedSDF(interpolation="trilinear")) in the fused ComposedSDF / RobotSDF kernels.

The fused kernels evaluate a PVB_GRID_TRILINEAR link with the arithmetic of grid_trilinear_kernel, so a composition
equals the generic per-link path (links wrapped in an opaque ObjectFrameSDF) bit for bit in values and argmin; the
gradients differ only by the rotation back to the object frame (torch matmul there, FMAs here)."""
import ctypes

import pytest
import torch

import workloads
from helpers import arm_points, cached_arm, cached_from_golden, golden, opaque_sdfs

pytestmark = pytest.mark.gpu


def _assert_fused_equals_generic(pv, sdfs, tsf, q, monkeypatch=None):
    fused = pv.ComposedSDF(sdfs, tsf)
    generic = pv.ComposedSDF(opaque_sdfs(pv, sdfs), tsf)
    vg, gg, wg = generic.query(q, return_which=True)
    if monkeypatch is not None:           # the fused composition must not take the generic route
        def boom(*a, **k):
            raise AssertionError("generic path taken")
        monkeypatch.setattr(fused, "_generic_query", boom)
    vf, gf, wf = fused.query(q, return_which=True)
    assert torch.equal(wf, wg)
    assert torch.equal(vf, vg)
    assert float((gf - gg).abs().max()) < 1e-6
    return vf, gf, wf


def test_golden_composition_fused_equals_generic(tmp_path, monkeypatch):
    import pytorch_volumetric_b200 as pv
    zc = golden("ref_cachedsdf_probe")
    tri = cached_from_golden(zc, "probe", tmp_path, interpolation="trilinear")
    near = cached_from_golden(zc, "probe", tmp_path)
    assert tri.native_desc("cuda") is not None
    z = golden("ref_composed")
    S, A = int(z["S"]), int(z["A"])
    sph = pv.SphereSDF(float(z["sphere_radius"]))
    tmat = torch.from_numpy(z["tmat"]).cuda()
    q = torch.from_numpy(z["q"]).cuda()
    for sdfs in ([tri, tri, sph, tri], [near, tri, sph, tri], [tri, near, near, sph]):
        _assert_fused_equals_generic(pv, sdfs, pv.Transform3d(matrix=tmat), q, monkeypatch)     # A configurations
        _assert_fused_equals_generic(pv, sdfs, pv.Transform3d(matrix=tmat.reshape(S, A, 4, 4)[:, 0]), q)   # one
    # first index on ties, also for trilinear links visited out of index order
    for n_same in (2, 3, 7):
        same = pv.ComposedSDF([tri] * n_same, pv.Transform3d(matrix=tmat[:1].repeat(n_same, 1, 1)))
        _, _, w = same.query(q, return_which=True)
        assert int(w.max()) == 0


@pytest.mark.parametrize("n_cfg,n_pts", [(40, 4096), (5, 1001), (200, 100_000)])
def test_trilinear_arm_fused_equals_generic(tmp_path, monkeypatch, n_cfg, n_pts):
    """8 trilinear links: the point-serial robot kernel (>= 8 configurations) and the point-major kernel (5), and a
    mix of nearest and trilinear links; 200 x 100 000 is the C4 shape of bench.py."""
    import pytorch_volumetric_b200 as pv
    s = cached_arm(tmp_path, "trilinear")
    s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
    pts = arm_points(n_pts, seed=21)
    tsf = s.sdf.obj_frame_to_link_frame
    _assert_fused_equals_generic(pv, s.sdf.sdfs, tsf, pts, monkeypatch)
    if n_cfg != 200:
        near = cached_arm(tmp_path, "nearest").sdf.sdfs
        mixed = [t if i % 3 else n for i, (t, n) in enumerate(zip(s.sdf.sdfs, near))]
        _assert_fused_equals_generic(pv, mixed, tsf, pts, monkeypatch)
    # RobotSDF.__call__ takes the fused path too
    monkeypatch.setattr(s.sdf, "_generic_query", lambda *a, **k: (_ for _ in ()).throw(AssertionError("generic")))
    v, g = s(pts)
    assert v.shape == (n_cfg, n_pts) and g.shape == (n_cfg, n_pts, 3)


def test_trilinear_beyond_eight_links_takes_the_cfg_major_kernel(tmp_path, monkeypatch):
    """12 links (robot_query_kernel is nearest-voxel only): the configuration-major kernel at 64 configurations,
    equal to the generic path and, bit for bit, to the point-major kernel."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.transforms import matrix_of
    s = cached_arm(tmp_path, "trilinear")
    n_cfg = 64
    s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
    M = matrix_of(s.sdf.obj_frame_to_link_frame).detach().reshape(8, n_cfg, 4, 4)
    sdfs = list(s.sdf.sdfs) + list(s.sdf.sdfs[:4])
    tsf = pv.Transform3d(matrix=torch.cat([M, M[:4].flip(1)]).reshape(12 * n_cfg, 4, 4))
    pts = arm_points(4096, seed=17)
    v, g, w = _assert_fused_equals_generic(pv, sdfs, tsf, pts, monkeypatch)
    comp = pv.ComposedSDF(sdfs, tsf)
    for i in (0, 33, 63):
        v1, g1, w1 = comp.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
        sl = slice(i * 4096, (i + 1) * 4096)
        assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), i


def test_trilinear_serial_kernel_equals_point_major(tmp_path):
    """robot_serial_kernel's trilinear variant == the point-major composed kernel (one configuration per launch), bit
    for bit incl. the argmin index, at the shapes of test_robot_kernel_equals_point_major_and_ragged."""
    s = cached_arm(tmp_path, "trilinear")
    base = arm_points(100_004, seed=9)
    for n_cfg, n_pts, shift in ((64, 4096, 0), (40, 4100, 0), (33, 1001, 0), (32, 2048, 1), (25, 4096, 0),
                                (200, 100_000, 0), (31, 100_003, 1)):
        s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
        pts = base.reshape(-1)[3 * shift:3 * (shift + n_pts)].view(n_pts, 3)
        v, g, w = s.sdf.query(pts, return_which=True)
        for i in (0, n_cfg // 2, n_cfg - 1):
            v1, g1, w1 = s.sdf.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
            sl = slice(i * n_pts, (i + 1) * n_pts)
            assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), (n_cfg, n_pts, i)


def test_trilinear_serial_kernel_with_nonrigid_transforms(tmp_path):
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.transforms import matrix_of
    s = cached_arm(tmp_path, "trilinear")
    n_cfg, n_pts = 40, 4096
    s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
    S = len(s.sdf.sdfs)
    M = matrix_of(s.sdf.obj_frame_to_link_frame).detach().clone().reshape(S, n_cfg, 4, 4)
    M[:, 5:13, :3, :3] *= 1.03
    M[3, 20:26, :3, :3] *= 0.97
    M[0, 30:, :3, :3] *= 1.02
    comp = pv.ComposedSDF(s.sdf.sdfs, pv.Transform3d(matrix=M.reshape(S * n_cfg, 4, 4)))
    pts = arm_points(n_pts, seed=13)
    v, g, w = comp.query(pts, return_which=True)
    for i in (0, 5, 12, 22, 31, 39):
        v1, g1, w1 = comp.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
        sl = slice(i * n_pts, (i + 1) * n_pts)
        assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), i


def test_trilinear_robot_multi_destination_paths(tmp_path):
    """query_into (3 destinations), the host result pipeline and gather="peer" with a single-rank PeerResult work
    for a trilinear robot and equal the plain query."""
    from pytorch_volumetric_b200 import distributed as pd
    s = cached_arm(tmp_path, "trilinear")
    for n_cfg, n_pts in ((40, 4096), (5, 1001)):
        s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
        pts = arm_points(n_pts, seed=11)
        v_ref, g_ref = s.sdf.query(pts)
        bufs = [(torch.full((n_cfg * n_pts,), -7.0, device="cuda"),
                 torch.full((n_cfg * n_pts * 3,), -7.0, device="cuda")) for _ in range(3)]
        s.sdf.query_into(pts, bufs, cfg_begin=0, cfg_count=n_cfg // 2)
        s.sdf.query_into(pts, bufs, cfg_begin=n_cfg // 2, cfg_count=n_cfg - n_cfg // 2)
        for v, g in bufs:
            assert torch.equal(v, v_ref) and torch.equal(g, g_ref.reshape(-1))
    # host result pipeline: 32 + 32 + 7 configurations, bit-identical to the plain path
    s.set_joint_configuration(workloads.arm_configurations(71).cuda())
    hp = arm_points(3001, seed=12).cpu()
    v0, g0 = s(hp)
    s.sdf.host_result_pipeline_min_bytes = 1 << 20
    try:
        v1, g1 = s(hp)
        assert v1.is_pinned()
    finally:
        del s.sdf.host_result_pipeline_min_bytes
    assert torch.equal(v0, v1) and torch.equal(g0, g1)
    # gather="peer" through a single-rank PeerResult
    s.set_joint_configuration(workloads.arm_configurations(12).cuda())
    pts = arm_points(777, seed=3)
    res = pd.PeerResult(12, 777)
    try:
        v, g = pd.sharded_robot_query(s, pts, gather="peer", result=res)
        v_ref, g_ref = s(pts)
        assert torch.equal(v, v_ref) and torch.equal(g, g_ref)
    finally:
        res.close()


def test_chamfer_keeps_trilinear_on_its_call_path(tmp_path):
    """pvb_chamfer refuses a TRILINEAR descriptor; batch_chamfer_dist(obj_sdf=trilinear) evaluates the SDF through
    its __call__ (the interpolant), as before."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import _native as nat
    zc = golden("ref_cachedsdf_probe")
    tri = cached_from_golden(zc, "probe", tmp_path, interpolation="trilinear")
    g = torch.Generator().manual_seed(5)
    w2o = workloads.random_rigid(6, seed=2, t_range=0.01).cuda()
    pts = (torch.rand(2000, 3, generator=g) * 0.06 - 0.03).cuda()
    err = pv.batch_chamfer_dist(w2o, pts, obj_sdf=tri, scale=1)
    pts_obj = pts @ w2o[:, :3, :3].transpose(-1, -2) + w2o[:, :3, 3].unsqueeze(1)
    d, _ = tri(pts_obj)
    assert torch.equal(err, (d ** 2).mean(dim=-1))
    ws = torch.empty(int(nat.lib().pvb_chamfer_workspace(len(pts))) * 6, device="cuda")
    out = torch.empty(6, device="cuda")
    w = w2o.float().contiguous()
    rc = nat.lib().pvb_chamfer(ctypes.byref(tri.native_desc("cuda")), nat.ptr(w), 6,
                               nat.ptr(pts), len(pts), 1.0, nat.ptr(ws), nat.ptr(out), None, 0,
                               nat.stream_ptr(pts.device))
    assert rc == -1 and b"TRILINEAR" in nat.lib().pvb_last_error()
