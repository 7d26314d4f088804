"""GPU parity: ComposedSDF (reference sdf.py:332-433) and RobotSDF (model_to_sdf.py:12-125)."""
import math

import numpy as np
import pytest
import torch

import workloads
from helpers import cached_from_golden, classify_composed, golden, grid_spec, pv_factory, sphere_spec, write_wrench_urdf

pytestmark = pytest.mark.gpu

def _close(a, b, tol=1e-5):
    return np.abs(a - b) <= tol


def _composed_from_golden(tmp_path):
    import pytorch_volumetric_b200 as pv
    zc = golden("ref_cachedsdf_probe")
    cs = cached_from_golden(zc, "probe", tmp_path)
    z = golden("ref_composed")
    S, A = int(z["S"]), int(z["A"])
    sdfs = [cs, cs, pv.SphereSDF(float(z["sphere_radius"])), cs]
    return pv, z, S, A, sdfs


def test_composed_vs_reference_golden(tmp_path):
    pv, z, S, A, sdfs = _composed_from_golden(tmp_path)
    tmat = torch.from_numpy(z["tmat"]).cuda()
    q = torch.from_numpy(z["q"]).cuda()
    comp = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tmat[:S]))
    v, g = comp(q)
    assert v.shape == (len(q),) and g.shape == (len(q), 3)           # flat output without a config batch (B2)
    # every output within 1e-5 of the reference's, or a classified voxel-boundary flip of the fp32 rigid transform
    # in front of the nearest-voxel lookup (helpers.classify_composed); nothing unexplained
    specs = [grid_spec(s) if isinstance(s, pv.CachedSDF) else sphere_spec(s.radius) for s in sdfs]
    P = len(q)
    n_ex, n_un, rep = classify_composed(v.cpu().numpy()[None], g.cpu().numpy()[None], z["val_plain"][None],
                                        z["grad_plain"][None], specs, z["tmat"][:S].reshape(S, 1, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 2e-3 * P, rep
    comp.set_transforms(pv.Transform3d(matrix=tmat), batch_dim=(A,))
    vb, gb = comp(q.reshape(30, 100, 3))
    assert vb.shape == (A, 30, 100) and gb.shape == (A, 30, 100, 3)
    n_ex, n_un, rep = classify_composed(vb.cpu().numpy().reshape(A, P), gb.cpu().numpy().reshape(A, P, 3),
                                        z["val_batched"].reshape(A, P), z["grad_batched"].reshape(A, P, 3), specs,
                                        z["tmat"].reshape(S, A, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 2e-3 * A * P, rep
    bb = comp.surface_bounding_box(padding=0.01)
    np.testing.assert_allclose(bb.cpu().numpy(), z["bbox_batched"], atol=1e-6)
    # batched == per-configuration loop, exactly (tests/test_model_to_sdf.py:206-212)
    for a in range(A):
        comp_a = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tmat.reshape(S, A, 4, 4)[:, a]))
        va, ga = comp_a(q)
        assert torch.equal(va, vb[a].reshape(-1)) and torch.equal(ga, gb[a].reshape(-1, 3))


def test_composed_fused_equals_generic_path(tmp_path):
    """The fused kernel (incl. its AABB pruning) against the unfused per-SDF composition of the same package, and
    against a user-defined ObjectFrameSDF subclass that forces the generic path."""
    pv, z, S, A, sdfs = _composed_from_golden(tmp_path)

    class Opaque(pv.ObjectFrameSDF):          # no native descriptor -> generic path
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, p):
            return self.inner(p)

        def surface_bounding_box(self, **kw):
            return self.inner.surface_bounding_box(**kw)

    tmat = torch.from_numpy(z["tmat"]).cuda()
    q = torch.from_numpy(z["q"]).cuda()
    fused = pv.ComposedSDF(sdfs, pv.Transform3d(matrix=tmat))
    generic = pv.ComposedSDF([Opaque(s) for s in sdfs], pv.Transform3d(matrix=tmat))
    vf, gf, wf = fused.query(q, return_which=True)
    vg, gg, wg = generic.query(q, return_which=True)
    assert torch.equal(wf, wg)
    assert torch.equal(vf, vg)
    assert (gf - gg).abs().max() < 1e-6
    # argmin semantics: first index on ties -- two identical SDFs at the same pose must report index 0
    twin = pv.ComposedSDF([sdfs[0], sdfs[0]], pv.Transform3d(matrix=tmat[:1].repeat(2, 1, 1)))
    _, _, w = twin.query(q, return_which=True)
    assert int(w.max()) == 0
    # ... also when the kernel visits the sub-SDFs out of index order (bit-reversed: 0, 2, 1, 3, and 0, 4, 2, 6, ...)
    for n_same in (3, 4, 7):
        same = pv.ComposedSDF([sdfs[0]] * n_same, pv.Transform3d(matrix=tmat[:1].repeat(n_same, 1, 1)))
        _, _, w = same.query(q, return_which=True)
        assert int(w.max()) == 0


def test_composed_of_meshes_vs_oracle():
    """ComposedSDF([MeshSDF, MeshSDF], translations) as in tests/test_sdf.py:61-80, checked against the oracle."""
    import pytorch_volumetric_b200 as pv
    from oracle import port, tp_pytorch_kinematics as opk
    obj = pv_factory("probe", ray_seed=1)
    tm = torch.eye(4).repeat(2, 1, 1)
    tm[0, :3, 3] = torch.tensor([0.1, 0.0, 0.0])
    tm[1, :3, 3] = torch.tensor([-0.2, 0.0, 0.2])
    comp = pv.ComposedSDF([pv.MeshSDF(obj), pv.MeshSDF(obj)], pv.Transform3d(matrix=tm.cuda()))
    q = workloads.uniform_points(4000, (-0.2, -0.05, -0.1), (0.3, 0.05, 0.3), seed=4)
    v, g = comp(q.cuda())
    pv_, pf_ = workloads.fixture_mesh("probe")
    mesh = port.MeshPort(vertices=pv_, faces=pf_)
    ref = port.ComposedSDFPort([port.MeshSDFPort(mesh), port.MeshSDFPort(mesh)], opk.Transform3d(matrix=tm))
    np.random.seed(0)
    vr, gr = ref(q)
    assert (v.cpu() - vr).abs().max() < 1e-5
    from helpers import classify_mesh_mismatch
    bad_v, bad_g, rep = classify_mesh_mismatch(v.cpu().numpy(), g.cpu().numpy(), vr.numpy(), gr.numpy(), 1e-5,
                                               coord_scale=0.3)
    assert bad_v == 0 and bad_g == 0, rep       # gradient exceedances: 1e-3 shell or closest-feature ties only


def test_robot_vs_reference_golden(tmp_path):
    import pytorch_volumetric_b200 as pv
    z = golden("ref_robot_wrench")
    urdf = write_wrench_urdf(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), "offset_wrench").to(device="cuda")
    # preload the link table the reference built (same cache format / key)
    v, f = workloads.fixture_mesh("wrench")
    bb = np.stack([v.min(0), v.max(0)], axis=1)
    rng = bb.copy(); rng[:, 0] -= 0.05; rng[:, 1] += 0.05
    ranges = pv.get_divisible_range_by_resolution(0.004, rng)
    np.testing.assert_allclose(np.array(ranges), z["ranges"], atol=1e-12)
    shape = [int(s) for s in z["table_shape"]]
    cache_path = str(tmp_path / "robot_cache.pkl")
    torch.save({f"wrench.obj 0.004 {tuple(ranges)}": (torch.from_numpy(z["table_val"]).reshape(shape),
                                                       torch.from_numpy(z["table_grad"]))}, cache_path)
    rs = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                     link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.004, padding=0.05, device="cuda",
                                                            cache_path=cache_path))
    th = torch.from_numpy(z["th"]).cuda()
    rs.set_joint_configuration(th)
    # FK + offset composition: object->link transforms (model_to_sdf.py:99-113)
    np.testing.assert_allclose(rs.object_to_link_frames.get_matrix().cpu().numpy(), z["obj_to_link"], atol=2e-6)
    q = torch.from_numpy(z["q"]).cuda()
    val, grad = rs(q)
    assert val.shape == (5, len(q)) and grad.shape == (5, len(q), 3)
    # within 1e-5 of the reference's vectors, every exceedance a classified voxel-boundary flip
    n_ex, n_un, rep = classify_composed(val.cpu().numpy(), grad.cpu().numpy(), z["val"], z["grad"],
                                        [grid_spec(rs.sdf.sdfs[0])], z["obj_to_link"].reshape(1, 5, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 3e-3 * val.numel(), rep
    np.testing.assert_allclose(rs.surface_bounding_box(padding=0.05).cpu().numpy(), z["bbox"], atol=1e-5)


def test_single_link_robot_contract(tmp_path):
    """The shape / value contracts of the reference's tests/test_model_to_sdf.py:263-326."""
    import pytorch_volumetric_b200 as pv
    urdf = write_wrench_urdf(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), "offset_wrench").to(device="cuda")
    sdf = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                      link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.001, padding=0.05, device="cuda",
                                                             cache_path=str(tmp_path / "c.pkl")))
    th = torch.zeros(6, device="cuda")
    sdf.set_joint_configuration(th.view(1, -1))
    query_range = sdf.surface_bounding_box(padding=0.05)[0]
    coords, pts = pv.get_coordinates_and_points_in_grid(0.001, query_range.cpu(), device="cuda")
    sdf_val, sdf_grad = sdf(pts)
    assert sdf_val.shape == (1, len(pts)) and sdf_grad.shape == (1, len(pts), 3)
    near_surface = sdf_val[0].abs() < 0.001
    surf_pts = pts[near_surface]
    B = 5
    sdf.set_joint_configuration(th.view(1, -1).repeat(B, 1))
    query_range = sdf.surface_bounding_box(padding=0.05)
    assert query_range.shape == (B, 3, 2)
    for i in range(1, B):
        assert torch.allclose(query_range[0], query_range[i])
    BB, N = 10, 100
    assert surf_pts.shape[0] > BB * N
    test_pts = surf_pts[:BB * N]
    sdf_vals, sdf_grads = sdf(test_pts)
    assert sdf_vals.shape == (B, BB * N) and sdf_grads.shape == (B, BB * N, 3)
    assert torch.allclose(sdf_vals.abs(), torch.zeros_like(sdf_vals), atol=1e-3)
    batch_sdf_vals, batch_sdf_grads = sdf(test_pts.view(BB, N, 3))
    assert batch_sdf_vals.shape == (B, BB, N) and batch_sdf_grads.shape == (B, BB, N, 3)
    assert torch.allclose(batch_sdf_vals, sdf_vals.view(B, BB, N))
    lb = sdf.link_bounding_boxes()
    assert lb.shape == (B, 8, 3)


def test_robot_arm_batched_equals_looped(tmp_path):
    """tests/test_model_to_sdf.py:173-212 on the synthetic 7-DOF arm: one batched call == per-configuration loop,
    and the fused kernel == an independent torch recomposition of the per-link lookups."""
    import pytorch_volumetric_b200 as pv
    urdf, end = workloads.write_arm(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    s = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                    link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                           cache_path=str(tmp_path / "arm.pkl")))
    assert len(s.sdf.sdfs) == 8
    th = workloads.arm_configurations(30).cuda()     # 30 of 32 lanes: takes the configuration-major kernel
    s.set_joint_configuration(th)
    coords, pts = pv.get_coordinates_and_points_in_grid(0.01, np.array([[-1, 0.5], [0.02, 0.02], [-0.2, 0.8]]),
                                                        device="cuda")
    assert len(pts) == 15251
    all_val, all_grad = s(pts)
    assert all_val.shape == (30, 15251)
    for i in range(0, 30, 7):
        s.set_joint_configuration(th[i])
        v, g = s(pts)
        assert v.shape == (15251,)
        # the reference's own tolerances (tests/test_model_to_sdf.py:211-212): FK of one configuration and of the
        # batch may differ in the last bit of the transforms
        assert torch.allclose(v, all_val[i]) and torch.allclose(g, all_grad[i], atol=1e-6)
    # configuration-major kernel (>= 16 configurations per launch) == point-major kernel (one configuration
    # slab per launch), bit for bit, including the argmin index
    s.set_joint_configuration(th)
    v_all, g_all, w_all = s.sdf.query(pts, return_which=True)
    for i in (0, 7, 29):
        v1, g1, w1 = s.sdf.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
        sl = slice(i * len(pts), (i + 1) * len(pts))
        assert torch.equal(v1, v_all[sl]) and torch.equal(g1, g_all[sl]) and torch.equal(w1, w_all[sl])
    # ragged sizes: 29 configurations x 1001 points (partial configuration tile, partial point tile)
    s.set_joint_configuration(th[:29])
    vr, gr = s.sdf.query(pts[:1001])
    for i in (0, 28):
        v1, g1 = s.sdf.query(pts[:1001], cfg_begin=i, cfg_count=1)
        assert torch.equal(v1, vr[i * 1001:(i + 1) * 1001]) and torch.equal(g1, gr[i * 1001:(i + 1) * 1001])
    # independent recomposition: per-link CachedSDF calls on explicitly transformed points, argmin in torch
    s.set_joint_configuration(th)
    M = s.object_to_link_frames.get_matrix().reshape(8, 30, 4, 4)
    vals, grads = [], []
    for i, link in enumerate(s.sdf.sdfs):
        local = pts @ M[i, :, :3, :3].transpose(-1, -2) + M[i, :, :3, 3].unsqueeze(1)
        v, g = link(local)
        vals.append(v); grads.append(g @ M[i, :, :3, :3])
    vals = torch.stack(vals); grads = torch.stack(grads)
    which = vals.argmin(0)
    v_ref = vals.gather(0, which.unsqueeze(0))[0]
    g_ref = grads.gather(0, which[None, ..., None].expand(1, -1, -1, 3))[0]
    # bmm-vs-fma rounding of the transform flips a few voxel keys: every difference must be such a flip
    n_ex, n_un, rep = classify_composed(all_val.cpu().numpy(), all_grad.cpu().numpy(), v_ref.cpu().numpy(),
                                        g_ref.cpu().numpy(), [grid_spec(l) for l in s.sdf.sdfs],
                                        M.cpu().numpy(), pts.cpu().numpy())
    assert n_un == 0 and n_ex <= 1e-3 * all_val.numel(), rep


@pytest.mark.parametrize("which", ["arm", "wrench"])
def test_native_fk_equals_eager_and_oracle(tmp_path, which):
    """pvb_fk_serial (one kernel: chain walk + (FK @ visual_offset)^-1 per mesh link) against the eager
    forward_kinematics path of the same chain and against the oracle's pytorch_kinematics restatement
    (model_to_sdf.py:99-113): revolute-only arm with visual offsets, and the mixed prismatic / revolute wrench chain."""
    import pytorch_volumetric_b200 as pv
    from oracle import port, tp_pytorch_kinematics as opk
    if which == "arm":
        urdf, end = workloads.write_arm(str(tmp_path))
        th = workloads.arm_configurations(37)
    else:
        urdf, end = write_wrench_urdf(str(tmp_path)), "offset_wrench"
        th = torch.randn(37, 6, generator=torch.Generator().manual_seed(0)) * 0.4
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    rs = pv.RobotSDF(chain, path_prefix=str(tmp_path))            # MeshSDF links: no tables to build
    assert rs._fk_plan is not None
    rs.set_joint_configuration(th.cuda())
    m_native = rs.object_to_link_frames.get_matrix().clone()
    assert m_native.shape == (len(rs.sdf.sdfs) * 37, 4, 4)
    rs.native_fk = False
    rs.set_joint_configuration(th.cuda())
    m_eager = rs.object_to_link_frames.get_matrix()
    assert (m_native - m_eager).abs().max() < 2e-6
    ochain = opk.build_serial_chain_from_urdf(open(urdf).read(), end)
    ref = port.RobotSDFPort(ochain, path_prefix=str(tmp_path), link_sdf_factory=lambda mesh: port.MeshSDFPort(mesh))
    ref.set_joint_configuration(th)
    np.testing.assert_allclose(m_native.cpu().numpy(), ref.object_to_link.get_matrix().numpy(), atol=2e-6)
    # single configuration (no batch): same rows as the batch, bit for bit (per-thread arithmetic)
    rs.native_fk = True
    rs.set_joint_configuration(th[5].cuda())
    assert rs.configuration_batch is None
    one = rs.object_to_link_frames.get_matrix()
    assert torch.equal(one, m_native.view(-1, 37, 4, 4)[:, 5])
    # multi-dimensional configuration batch
    rs.set_joint_configuration(th[:36].view(4, 9, -1).cuda())
    assert tuple(rs.configuration_batch) == (4, 9)
    assert torch.equal(rs.object_to_link_frames.get_matrix().view(-1, 36, 4, 4), m_native.view(-1, 37, 4, 4)[:, :36])


def test_robot_kernel_equals_point_major_and_ragged(tmp_path):
    """robot_query_kernel (configuration-major, unrolled links, row epilogue) == the point-major composed kernel, bit
    for bit incl. the argmin index, on full and ragged shapes: n_pts % 4 != 0 (scalar rows), n_pts % 32 != 0 (tail
    tile), partial configuration tiles, and an unaligned point buffer."""
    import pytorch_volumetric_b200 as pv
    urdf, end = workloads.write_arm(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    s = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                    link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                           cache_path=str(tmp_path / "arm.pkl")))
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    base = workloads.uniform_points(100_004, lo, hi, seed=9).cuda()
    # small launches run 4-point warp steps, the 200 x 100 000 one (bench.py's C4) 8-point steps; 25 = 16 + 8 + 1 and
    # 200 = 6 x 32 + 8 exercise the lane-split remainder tiles
    for n_cfg, n_pts, shift in ((64, 4096, 0), (40, 4100, 0), (33, 1001, 0), (32, 2048, 1), (25, 4096, 0),
                                (200, 100_000, 0), (31, 100_003, 1)):
        s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
        pts = base.reshape(-1)[3 * shift:3 * (shift + n_pts)].view(n_pts, 3)       # shift=1: not 16-byte aligned
        v, g, w = s.sdf.query(pts, return_which=True)                               # >= 16 configurations: robot kernel
        for i in (0, n_cfg // 2, n_cfg - 1):
            v1, g1, w1 = s.sdf.query(pts, cfg_begin=i, cfg_count=1, return_which=True)     # point-major kernel
            sl = slice(i * n_pts, (i + 1) * n_pts)
            assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), (n_cfg, n_pts, i)


@pytest.mark.gpu
def test_host_result_pipeline_equals_plain_path(tmp_path):
    """ComposedSDF.__call__ with host points and a result above `host_result_pipeline_min_bytes` streams the result
    out slab by slab (32 configurations, then 64 at a time, copies on a side stream): bit-identical to the plain path,
    same shapes, pinned host tensors; non-qualifying calls (small result, fp64 points) keep the plain path."""
    import pytorch_volumetric_b200 as pv
    urdf, end = workloads.write_arm(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    s = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                    link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                           cache_path=str(tmp_path / "arm.pkl")))
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    pts = workloads.uniform_points(3001, lo, hi, seed=11)
    for n_cfg in (64, 135):                   # 32 + 32, 32 + 64 + 39
        s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
        v0, g0 = s(pts)                        # 16 * 135 * 3001 bytes < 64 MiB: plain path
        assert s.sdf._host_result_pipeline(pts) is None
        s.sdf.host_result_pipeline_min_bytes = 1 << 20
        try:
            assert s.sdf._host_result_pipeline(pts.double()) is None
            v1, g1 = s(pts)
        finally:
            del s.sdf.host_result_pipeline_min_bytes
        assert v1.device.type == "cpu" and v1.is_pinned() and v1.shape == (n_cfg, 3001) and g1.shape == (n_cfg, 3001, 3)
        assert torch.equal(v0, v1) and torch.equal(g0, g1)


@pytest.mark.gpu
def test_robot_kernel_with_nonrigid_transforms(tmp_path):
    """robot_serial_kernel's bounding-sphere bounds need isometries: (configuration, link) transforms that are not
    (scaled rotation blocks here) get no sphere bound at all -- their keys are NaN patterns in the nearest-sphere
    selection -- and must still produce what the point-major kernel (no sphere bounds) produces, bit for bit."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.transforms import matrix_of
    urdf, end = workloads.write_arm(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    s = pv.RobotSDF(chain, path_prefix=str(tmp_path),
                    link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                           cache_path=str(tmp_path / "arm.pkl")))
    n_cfg, n_pts = 40, 4096
    s.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
    S = len(s.sdf.sdfs)
    M = matrix_of(s.sdf.obj_frame_to_link_frame).detach().clone().reshape(S, n_cfg, 4, 4)
    M[:, 5:13, :3, :3] *= 1.03              # every link of configurations 5..12
    M[3, 20:26, :3, :3] *= 0.97             # one link of configurations 20..25
    M[0, 30:, :3, :3] *= 1.02               # link 0 (the slot whose -inf bound stays a valid float key)
    comp = pv.ComposedSDF(s.sdf.sdfs, pv.Transform3d(matrix=M.reshape(S * n_cfg, 4, 4)))
    assert tuple(comp.tsf_batch) == (n_cfg,)
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    pts = workloads.uniform_points(n_pts, lo, hi, seed=13).cuda()
    v, g, w = comp.query(pts, return_which=True)
    for i in (0, 5, 12, 22, 31, 39):
        v1, g1, w1 = comp.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
        sl = slice(i * n_pts, (i + 1) * n_pts)
        assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), i

