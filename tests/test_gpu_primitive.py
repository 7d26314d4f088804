"""GPU: analytic URDF primitives (BoxSDF, CylinderSDF, SphereSDF links) on the fused ComposedSDF / RobotSDF kernels.

The primitives against their fp64 restatements (tests/primitive_ref.py) and BoxSDF against MeshSDF of a closed box
mesh; the primitive arm and the mixed arm (some links the probe mesh through cache_link_sdf_factory) of
workloads.write_primitive_arm at the C4 shape: fused against an fp64 composition, the serial robot kernel against
per-configuration slab queries bit for bit, no generic path, paired queries, query_into and single-rank peer
re-assembly; and batch_chamfer_dist with a BoxSDF."""
import numpy as np
import pytest
import torch

import primitive_ref as pr
import workloads
from helpers import arm_points, no_generic

pytestmark = pytest.mark.gpu


def _tolerance(rv, q):
    """1e-6, or the conditioning of the outside gradient w / |w| (tests/test_primitive_cpu.py)."""
    return np.where(rv > 0, np.maximum(1e-6, 3e-7 * np.abs(q).max(1) / np.maximum(rv, 1e-30)), 1e-6)


@pytest.mark.parametrize("which", ["box", "cylinder", "disc"])
def test_primitive_call_vs_fp64_on_a_million_points(which):
    import pytorch_volumetric_b200 as pv
    s = {"box": pv.BoxSDF([0.3, 0.12, 0.2]), "cylinder": pv.CylinderSDF(0.05, 0.3),
         "disc": pv.CylinderSDF(0.1, 0.02)}[which]
    d = s.native_desc("cuda")
    h = np.array([float(d.bb_max[k]) for k in range(3)])
    q = (np.random.default_rng(1).uniform(-3, 3, (1_000_000, 3)) * h).astype(np.float32)
    v, g = s(torch.from_numpy(q).cuda())
    assert v.shape == (1_000_000,) and g.shape == (1_000_000, 3)
    v, g = v.cpu().numpy(), g.cpu().numpy()
    rv, rg = pr.primitive_ref(d, q.astype(np.float64))
    assert np.abs(v - rv).max() < 1e-6
    clear = pr.second_gap(d, q) > 1e-5
    assert clear.mean() > 0.95
    assert (np.abs(g - rg).max(1) <= _tolerance(rv, q))[clear].all()
    # batched leading dimensions and host tensors come back in the points' shape, device and dtype
    vb, gb = s(torch.from_numpy(q[:6000]).double().reshape(2, 3, 1000, 3))
    assert vb.shape == (2, 3, 1000) and gb.shape == (2, 3, 1000, 3) and vb.dtype == torch.float64
    assert torch.equal(vb.reshape(-1).float(), torch.from_numpy(v[:6000]))


def _box_mesh(h):
    v = np.array([[x, y, z] for x in (-h[0], h[0]) for y in (-h[1], h[1]) for z in (-h[2], h[2])], dtype=np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                  [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    return v, f


def test_box_against_the_mesh_path():
    """BoxSDF against MeshSDF of the closed 12-triangle box (the mesh path is pinned to the oracle): values within
    1e-5 everywhere, gradients within 1e-5 except where a classified rule applies."""
    import pytorch_volumetric_b200 as pv
    size = [0.25, 0.125, 0.375]
    box = pv.BoxSDF(size)
    h = np.array(size) / 2
    v, f = _box_mesh(h)
    mesh = pv.MeshSDF(pv.MeshObjectFactory("box", mesh=(v, f)))
    assert mesh.obj_factory.is_closed
    q = (np.random.default_rng(2).uniform(-2, 2, (400_000, 3)) * h).astype(np.float32)
    qt = torch.from_numpy(q).cuda()
    vb, gb = (t.cpu().numpy() for t in box(qt))
    vm, gm = (t.cpu().numpy() for t in mesh(qt))
    assert np.abs(vb - vm).max() < 1e-5
    bad = np.abs(gb - gm).max(1) > 1e-5
    # classification: (a) medial-axis ties of the inside rule (the closest face is not unique), (b) the mesh's
    # surface-normal rule (|d| < 1e-3: the face normal, which differs from the box gradient outside near an edge or a
    # corner), (c) another closest point: the mesh path's closest point q - d g lies on the box surface too (within
    # 2e-6) at the same distance -- its fp32 closest-point arithmetic (barycentric products with cancellation) places
    # it a few micrometres from the exact one, or a closest-feature tie at an edge picks the neighbouring face
    d = box.native_desc("cuda")
    medial = (vb <= 0) & (pr.second_gap(d, q) < 1e-5)
    normal_rule = np.abs(vm) < 1e-3
    c = q.astype(np.float64) - vm.astype(np.float64)[:, None] * gm.astype(np.float64)
    on_surface = np.abs(pr.box_ref([float(x) for x in d.bb_max], c)[0]) < 2e-6
    assert (~bad).mean() > 0.99
    assert (medial | normal_rule | on_surface)[bad].all()


# ---------------------------------------------------------------- the arms
def _arm(tmp_path, mixed):
    import pytorch_volumetric_b200 as pv
    d = tmp_path / ("mixed" if mixed else "prim")
    urdf, end = workloads.write_primitive_arm(str(d), mesh_links=workloads.MIXED_ARM_MESH_LINKS if mixed else ())
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    return pv.RobotSDF(chain, path_prefix=str(d), primitive_visuals=True,
                       link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                              cache_path=str(d / "cache.pkl")))


def _fp64_values(robot, pts):
    """Values [S, A, P] (fp64) of every link at every point: primitives restated in fp64 under the fp32 link
    transforms carried out in fp64; cached mesh links through their own CachedSDF (the voxel rule)."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.transforms import matrix_of
    S = len(robot.sdf.sdfs)
    M = matrix_of(robot.sdf.obj_frame_to_link_frame).detach().double().reshape(S, -1, 4, 4)
    A = M.shape[1]
    p = pts.double()
    out = torch.empty(S, A, len(pts), dtype=torch.float64, device="cuda")
    for s, link in enumerate(robot.sdf.sdfs):
        for a in range(A):
            q = p @ M[s, a, :3, :3].T + M[s, a, :3, 3]
            if isinstance(link, pv.BoxSDF):
                hh = torch.tensor([float(v) for v in link.native_desc("cuda").bb_max], dtype=torch.float64,
                                  device="cuda")
                e = q.abs() - hh
                n = e.clamp(min=0).norm(dim=1)
                out[s, a] = torch.where(n > 0, n, e.max(1).values)
            elif isinstance(link, pv.CylinderSDF):
                d = link.native_desc("cuda")
                dr = torch.hypot(q[:, 0], q[:, 1]) - float(d.radius)
                dz = q[:, 2].abs() - float(d.bb_max[2])
                n = torch.hypot(dr.clamp(min=0), dz.clamp(min=0))
                out[s, a] = torch.where(n > 0, n, torch.maximum(dr, dz))
            elif isinstance(link, pv.SphereSDF):
                out[s, a] = q.norm(dim=1) - float(np.float32(link.radius))
            else:
                out[s, a] = link(q.float())[0].double()          # the cached link's voxel rule
    return out


@pytest.mark.parametrize("mixed", [False, True])
def test_arm_fused_vs_fp64_composition(tmp_path, monkeypatch, mixed):
    robot = _arm(tmp_path, mixed)
    assert len(robot.sdf.sdfs) == 8
    A, P = 200, 100_000
    robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
    pts = arm_points(P, seed=31)
    no_generic(monkeypatch, robot.sdf)
    v, g, w = robot.sdf.query(pts, return_which=True)
    ref = _fp64_values(robot, pts)
    rv, rw = ref.min(0)
    v, w = v.reshape(A, P).double(), w.reshape(A, P).long()
    # cached mesh links: the fp32 transform of the kernel and the fp64 one here may pick neighbouring voxels
    import pytorch_volumetric_b200 as pv
    cached = torch.tensor([isinstance(s, pv.CachedSDF) for s in robot.sdf.sdfs], device="cuda")
    voxel_flip = cached[w] | cached[rw]
    bad = (v - rv).abs() > 1e-5
    assert not bool((bad & ~voxel_flip).any()), float((v - rv).abs()[~voxel_flip].max())
    assert float(bad.float().mean()) < 2e-3
    differ = w != rw
    assert float(differ.float().mean()) < 1e-3
    # an argmin disagreement only at a near-tie of the restated values, or a voxel flip of a cached link
    a_i, p_i = torch.nonzero(differ, as_tuple=True)
    near_tie = (ref[w[differ], a_i, p_i] - ref[rw[differ], a_i, p_i]).abs() < 1e-5
    assert bool((near_tie | voxel_flip[differ]).all())
    assert len(set(w.unique().tolist())) == 8          # every link wins somewhere


@pytest.mark.parametrize("mixed", [False, True])
def test_arm_serial_kernel_equals_slab_queries(tmp_path, mixed):
    """robot_serial_kernel (>= 8 configurations) == the point-major kernel (one configuration per launch), bit for bit
    with the argmin index, at full and ragged shapes."""
    robot = _arm(tmp_path, mixed)
    base = arm_points(100_004, seed=9)
    for n_cfg, n_pts, shift in ((200, 100_000, 0), (40, 4100, 0), (33, 1001, 1), (8, 2048, 0)):
        robot.set_joint_configuration(workloads.arm_configurations(n_cfg).cuda())
        pts = base.reshape(-1)[3 * shift:3 * (shift + n_pts)].view(n_pts, 3)
        v, g, w = robot.sdf.query(pts, return_which=True)
        for i in (0, n_cfg // 2, n_cfg - 1):
            v1, g1, w1 = robot.sdf.query(pts, cfg_begin=i, cfg_count=1, return_which=True)
            sl = slice(i * n_pts, (i + 1) * n_pts)
            assert torch.equal(v1, v[sl]) and torch.equal(g1, g[sl]) and torch.equal(w1, w[sl]), (n_cfg, n_pts, i)


def test_sphere_sets_unchanged_by_the_extension_route(tmp_path, monkeypatch):
    """Sets containing SphereSDF now run the extension instantiations (and the serial robot kernel): values, argmin
    and gradients equal the generic per-link composition, where the sphere is pvb_sphere_query."""
    import pytorch_volumetric_b200 as pv
    robot = _arm(tmp_path, False)
    robot.set_joint_configuration(workloads.arm_configurations(40).cuda())
    pts = arm_points(4096, seed=5)

    class Opaque(pv.ObjectFrameSDF):
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, p):
            return self.inner(p)

        def surface_bounding_box(self, **kw):
            return self.inner.surface_bounding_box(**kw)

    tsf = robot.sdf.obj_frame_to_link_frame
    sph = [pv.SphereSDF(r) for r in (0.05, 0.08, 0.11, 0.06, 0.09, 0.07, 0.05, 0.1)]
    fused = pv.ComposedSDF(sph, tsf)
    no_generic(monkeypatch, fused)
    vf, gf, wf = fused.query(pts, return_which=True)
    vg, gg, wg = pv.ComposedSDF([Opaque(s) for s in sph], tsf).query(pts, return_which=True)
    assert torch.equal(vf, vg) and torch.equal(wf, wg) and float((gf - gg).abs().max()) < 1e-6


@pytest.mark.parametrize("mixed", [False, True])
def test_arm_paired_and_multi_destination(tmp_path, mixed):
    from pytorch_volumetric_b200 import distributed as pd
    robot = _arm(tmp_path, mixed)
    A, N = 24, 1000
    robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
    per = arm_points(A * N, seed=41).reshape(A, N, 3)
    pv_, pg = robot.paired(per)
    assert pv_.shape == (A, N) and pg.shape == (A, N, 3)
    for a in (0, 7, A - 1):
        v1, g1 = robot.sdf.query(per[a], cfg_begin=a, cfg_count=1)
        assert torch.equal(pv_[a], v1) and torch.equal(pg[a], g1.reshape(N, 3)), a
    # query_into with 3 destinations, in two slabs
    pts = arm_points(4096, seed=42)
    v_ref, g_ref = robot.sdf.query(pts)
    bufs = [(torch.full((A * 4096,), -7.0, device="cuda"), torch.full((A * 4096 * 3,), -7.0, device="cuda"))
            for _ in range(3)]
    robot.sdf.query_into(pts, bufs, cfg_begin=0, cfg_count=A // 2)
    robot.sdf.query_into(pts, bufs, cfg_begin=A // 2, cfg_count=A - A // 2)
    for v, g in bufs:
        assert torch.equal(v, v_ref) and torch.equal(g, g_ref.reshape(-1))
    # gather="peer" through a single-rank PeerResult
    res = pd.PeerResult(A, 777)
    try:
        p7 = pts[:777].contiguous()
        v, g = pd.sharded_robot_query(robot, p7, gather="peer", result=res)
        v_ref, g_ref = robot(p7)
        assert torch.equal(v, v_ref) and torch.equal(g, g_ref)
    finally:
        res.close()


def test_chamfer_with_a_box():
    import pytorch_volumetric_b200 as pv
    box = pv.BoxSDF([0.05, 0.03, 0.04])
    g = torch.Generator().manual_seed(5)
    w2o = workloads.random_rigid(6, seed=2, t_range=0.01).cuda()
    pts = (torch.rand(5000, 3, generator=g) * 0.08 - 0.04).cuda()
    err = pv.batch_chamfer_dist(w2o, pts, obj_sdf=box, scale=1000)
    pts_obj = pts @ w2o[:, :3, :3].transpose(-1, -2) + w2o[:, :3, 3].unsqueeze(1)
    d, _ = box(pts_obj)
    ref = ((1000 * d) ** 2).mean(dim=-1)
    assert err.shape == (6,) and torch.allclose(err, ref, rtol=1e-4, atol=1e-6)
