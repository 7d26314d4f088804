"""GPU parity: CachedSDF (reference sdf.py:441-614) -- voxel index / occupancy bit-exact, table gathers exact,
out-of-range rule within 2 ulp, against golden vectors from the reference source and against oracle/port.py."""
import numpy as np
import pytest
import torch

import workloads
from helpers import cached_from_golden, golden, pv_factory

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["probe", "drill"])
def test_cached_lookup_vs_reference_golden(name, tmp_path):
    z = golden(f"ref_cachedsdf_{name}")
    c = cached_from_golden(z, name, tmp_path)
    assert tuple(c.voxels.shape) == tuple(int(s) for s in z["table_shape"])
    q = torch.from_numpy(z["q"]).cuda()
    inb = z["inbound"]
    # voxel index + in-range mask: BIT-EXACT (north_star)
    keys = c.voxel_keys(q).cpu().numpy()
    assert np.array_equal(keys >= 0, inb)
    assert np.array_equal(keys[inb], z["keys"][inb])
    val, grad = c(q)
    val, grad = val.cpu().numpy(), grad.cpu().numpy()
    # in-range values are pure gathers: exactly equal
    assert np.array_equal(val[inb], z["val"][inb])
    assert np.array_equal(grad[inb], z["grad"][inb])
    # out-of-range: point-to-AABB rule (sdf.py:555-571), fp32; the reference's torch-CPU norm accumulates
    # in double, the kernel in fp32: 2 ulp
    oob = ~inb
    assert np.abs(val[oob] - z["val"][oob]).max() <= 2 * np.spacing(np.abs(z["val"][oob]).max())
    assert np.abs(grad[oob] - z["grad"][oob]).max() <= 3e-7
    # occupancy (sdf.py:593-602): bit-exact
    assert np.array_equal(c.outside_surface(q).cpu().numpy(), z["outside"])
    assert np.array_equal(c.outside_surface(q, surface_level=0.003).cpu().numpy(),
                          np.where(inb, z["val"] > 0.003, True))


def test_cached_lookup_fp32_range_mode(tmp_path):
    """Range given as Python floats: the reference's view does its index arithmetic in fp32."""
    z = golden("ref_cachedsdf_probe")
    rng32 = [(float(a), float(b)) for a, b in z["range_in"]]
    c = cached_from_golden(z, "probe32", tmp_path, "table_val_f32range", "table_grad_f32range", range_in=rng32)
    q = torch.from_numpy(z["q"]).cuda()
    inb = z["inbound_f32range"]
    keys = c.voxel_keys(q).cpu().numpy()
    assert np.array_equal(keys >= 0, inb)
    assert np.array_equal(keys[inb], z["keys_f32range"][inb])
    val, grad = c(q)
    assert np.array_equal(val.cpu().numpy()[inb], z["val_f32range"][inb])
    assert np.array_equal(grad.cpu().numpy()[inb], z["grad_f32range"][inb])


def test_cached_lookup_gt_strategy(tmp_path):
    """OutOfBoundsStrategy.LOOKUP_GT_SDF (sdf.py:553-554): out-of-range points take the mesh query inside the
    same kernel."""
    import pytorch_volumetric_b200 as pv
    z = golden("ref_cachedsdf_probe")
    c = cached_from_golden(z, "probe", tmp_path, out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    n = len(z["val_gt"])
    q = torch.from_numpy(z["q"][:n]).cuda()
    val, grad = c(q)
    val, grad = val.cpu().numpy(), grad.cpu().numpy()
    inb = z["inbound"][:n]
    assert np.array_equal(val[inb], z["val_gt"][inb])
    assert np.abs(val[~inb] - z["val_gt"][~inb]).max() < 1e-6
    dg = np.abs(grad[~inb] - z["grad_gt"][~inb]).max(axis=-1)
    assert (dg > 1e-5).mean() < 2e-3     # medial-axis ties only


@pytest.mark.parametrize("name", ["probe", "drill"])
def test_cached_table_build_on_gpu(name, tmp_path):
    """Tables built by the GPU MeshSDF (sdf.py:502-505) against the tables the reference built over the
    brute-force oracle: same lattice, values within 1e-5; gradient exceedances only on closest-feature ties."""
    import pytorch_volumetric_b200 as pv
    z = golden(f"ref_cachedsdf_{name}")
    gt = pv.MeshSDF(pv_factory(name))
    c = pv.CachedSDF(name, float(z["resolution"]), z["range_in"], gt, device="cuda",
                     cache_path=str(tmp_path / "fresh.pkl"), debug_check_sdf=True)
    assert tuple(c.voxels.shape) == tuple(int(s) for s in z["table_shape"])
    np.testing.assert_array_equal(np.array(c.ranges), z["ranges"])
    tv = c.voxels.raw_data.cpu().numpy()
    tg = c.voxels_grad.cpu().numpy()
    sign_bad = (np.sign(tv) != np.sign(z["table_val"])) & (np.abs(z["table_val"]) > 1e-6)
    assert sign_bad.sum() == 0
    assert np.abs(tv - z["table_val"]).max() < 1e-5
    dg = np.abs(tg - z["table_grad"]).max(axis=-1)
    assert (dg > 1e-5).mean() < 5e-3
    # the cache file is in the reference's format and reloads
    data = torch.load(str(tmp_path / "fresh.pkl"))
    (k, (cv, cg)), = data.items()
    assert k == c.name and cv.shape == c.voxels.shape and cg.shape == (tv.size, 3)
    with pytest.raises(RuntimeError):
        pv.CachedSDF("other", 0.01, z["range_in"], None, cache_path=str(tmp_path / "missing.pkl"))


def test_cached_c2_full_size_properties(tmp_path):
    """BASELINE config C2 (drill, res 0.005, 10^7 points) through size-independent properties."""
    import pytorch_volumetric_b200 as pv
    obj = pv_factory("drill")
    gt = pv.MeshSDF(obj)
    c = pv.CachedSDF("drill", 0.005, obj.bounding_box(padding=0.1), gt, device="cuda",
                     cache_path=str(tmp_path / "c2.pkl"))
    assert tuple(c.voxels.shape) == (74, 66, 78)
    lo = np.array([r[0] for r in c.ranges]); hi = np.array([r[1] for r in c.ranges])
    n = 10_000_000
    q = workloads.uniform_points(n, lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo), seed=0, device="cuda")
    val, grad = c(q)
    keys = c.voxel_keys(q)
    inb = keys >= 0
    assert 0.5 < inb.float().mean() < 0.65
    # gather consistency: values are exactly table[key]
    assert torch.equal(val[inb], c.voxels.raw_data[keys[inb]])
    assert torch.equal(grad[inb], c.voxels_grad[keys[inb]])
    # every voxel centre reads back its own cell (the reference's own self-check, sdf.py:509-512); a centre on
    # the upper face can round up in fp32 to just above the fp64 range end, which the reference's own
    # all(min <= p <= max) test then calls out of range -- the oracle decides
    from oracle import port
    coords, centres = pv.get_coordinates_and_points_in_grid(0.005, c.ranges)
    kc = c.voxel_keys(centres.cuda()).cpu()
    ref = port.CachedSDFPort("drill", 0.005, obj.bounding_box(padding=0.1), port.SphereSDFPort(1.0),
                             tables=(c.voxels.raw_data.cpu().reshape(tuple(c.voxels.shape)), c.voxels_grad.cpu()))
    _, flat, inb_ref = ref.index_and_mask(centres)
    assert torch.equal(kc >= 0, inb_ref) and torch.equal(kc[inb_ref], flat[inb_ref])
    assert torch.equal(kc[inb_ref], torch.arange(len(centres))[inb_ref])
    assert inb_ref.float().mean() > 0.9
    # vectorised (4 points / thread) and scalar kernels agree bit-for-bit: a view offset by one point is not
    # 16-byte aligned and takes the scalar kernel
    v2, g2 = c(q[1:1_000_001])
    assert torch.equal(v2, val[1:1_000_001]) and torch.equal(g2, grad[1:1_000_001])
    # out-of-range: value equals the distance to the mesh AABB, gradient is unit and points away from it
    oob = ~inb
    bb = torch.tensor(obj.bounding_box(), dtype=torch.float32, device="cuda")
    d = torch.clamp(torch.maximum(bb[:, 0] - q[oob], q[oob] - bb[:, 1]), min=0).norm(dim=-1)
    assert (val[oob] - d).abs().max() < 1e-6
    assert (grad[oob].norm(dim=-1) - 1).abs().max() < 1e-5
    # permutation equivariance
    perm = torch.randperm(n, device="cuda")[:1_000_000]
    vp, gp = c(q[perm])
    assert torch.equal(vp, val[perm]) and torch.equal(gp, grad[perm])
    # host path: pinned host tensor in, host tensors out through the chunked three-stream pipeline, bit-identical
    ch = pv.CachedSDF("drill", 0.005, obj.bounding_box(padding=0.1), gt, device="cpu",
                      cache_path=str(tmp_path / "c2.pkl"))
    qh = q[:5_000_003].cpu().pin_memory()
    vh, gh = ch(qh)
    assert vh.device.type == "cpu" and vh.is_pinned()
    assert torch.equal(vh, val[:5_000_003].cpu()) and torch.equal(gh, grad[:5_000_003].cpu())
    vh2, gh2 = ch(qh[:1000].double())                       # small batch, other dtype: plain path
    assert vh2.dtype == torch.float64 and torch.equal(vh2.float(), val[:1000].cpu())
    # batch dims
    vb, gb = c(q[:6000].view(2, 30, 100, 3))
    assert vb.shape == (2, 30, 100) and gb.shape == (2, 30, 100, 3)


def test_trilinear_extension_vs_its_cpu_restatement(tmp_path):
    """Opt-in extension (not reference behaviour): trilinear value + gradient of the interpolant, checked against
    oracle.port.trilinear_lookup_port (fp64) and through its defining properties."""
    import pytorch_volumetric_b200 as pv
    from oracle import port
    z = golden("ref_cachedsdf_probe")
    c = cached_from_golden(z, "probe", tmp_path, interpolation="trilinear")
    q = torch.from_numpy(z["q"]).cuda()
    v, g = c(q)
    shape = tuple(int(s) for s in z["table_shape"])
    rv, rg, inb = port.trilinear_lookup_port(torch.from_numpy(z["table_val"]).reshape(shape), c.ranges,
                                             z["bb"], q.cpu())
    assert np.array_equal(inb.numpy(), z["inbound"])          # same in-range rule as the reference
    assert (v.cpu().double() - rv).abs().max() < 2e-6
    # the gradient of a trilinear interpolant jumps across cell faces: compare away from the lattice planes (the
    # query set deliberately contains exact voxel centres and cell-boundary points)
    lo = np.array([float(min(r)) for r in c.ranges]); hi = np.array([float(max(r)) for r in c.ranges])
    u = (q.cpu().double().numpy() - lo) / ((hi - lo) / (np.array(shape) - 1))
    off_lattice = torch.from_numpy((np.abs(u - np.round(u)) > 1e-3).all(axis=1)) & inb
    assert off_lattice.float().mean() > 0.4
    assert (g.cpu().double() - rg)[off_lattice].abs().max() < 1e-4
    assert (g.cpu().double() - rg)[~inb].abs().max() < 1e-6
    # exact at the voxel centres, continuous (Lipschitz) in between, within one cell of the nearest-voxel lookup
    coords, centres = pv.get_coordinates_and_points_in_grid(float(z["resolution"]), c.ranges)
    vc, _ = c(centres.cuda())
    inside = c.voxel_keys(centres.cuda()) >= 0
    assert (vc.cpu() - torch.from_numpy(z["table_val"]))[inside.cpu()].abs().max() < 1e-6
    near = cached_from_golden(z, "probe", tmp_path)
    vn, _ = near(q)
    assert (v - vn)[torch.from_numpy(z["inbound"]).cuda()].abs().max() < 2 * float(z["resolution"])
    # the fused composition kernels keep the reference rule: a trilinear CachedSDF composes through the generic path
    comp = pv.ComposedSDF([c], pv.Transform3d(matrix=torch.eye(4, device="cuda").unsqueeze(0)))
    vcmp, _ = comp(q)
    assert torch.equal(vcmp, v)
    with pytest.raises(ValueError):
        cached_from_golden(z, "probe", tmp_path, interpolation="cubic")
