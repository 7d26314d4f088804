"""GPU: the occupancy distance transform (pvb_occupancy_sdf, occupancy_distance_transform, OccupancySDF).

1. D, sites and tables equal the host build of the device routines (tests/hostsim/hostsim_edt.cpp) bit for bit, on
   random grids up to 192^3 and on 1024-long axes; two calls return the same bits.
2. D equals scipy's, and the sites pass the lattice check of tests/edt_ref.py.
3. from_points' occupancy equals the VoxelGrid scatter of the same points.
4. OccupancySDF.__call__, nearest and trilinear, in and out of range, equals tests/grid_ref.py on its table and box.
5. An OccupancySDF of the tabletop cloud as the scene of the cached arm and of the hand: the fused route equals the
   composition route (clearance bit for bit, cost within 1e-5 of each row), as tests/test_gpu_scene.py requires."""
import numpy as np
import pytest
import torch

import edt_ref
import grid_ref

pytestmark = pytest.mark.gpu


def _random(shape, p, seed):
    g = np.random.default_rng(seed)
    occ = g.random(shape) < p
    occ.reshape(-1)[0], occ.reshape(-1)[-1] = True, False
    return occ


def _native(occ, resolution):
    """(D, site, table) of pvb_occupancy_sdf, on the host."""
    from pytorch_volumetric_b200 import sdf as S
    o = torch.from_numpy(occ.astype(np.uint8)).cuda()
    d, s, t = S._occupancy_sdf(o, resolution, sqdist=True, site=True, table=True)
    return d.cpu().numpy(), s.cpu().numpy(), t.cpu().numpy()


CASES = [((64, 64, 64), 0.01), ((64, 64, 64), 0.3), ((96, 80, 70), 0.001), ((128, 128, 128), 0.05),
         ((192, 192, 192), 0.01), ((192, 192, 192), 0.3), ((1024, 3, 5), 0.01), ((3, 1024, 5), 0.2),
         ((5, 3, 1024), 0.01), ((1024, 2, 2), 0.002)]


# ---------------------------------------------------------------- 1 and 2. transform against the host build and scipy
@pytest.mark.parametrize("shape,p", CASES)
def test_transform_equals_host_build_and_scipy(shape, p):
    occ = _random(shape, p, seed=int(p * 1e4) + shape[0])
    r = 0.0137
    d, s, t = _native(occ, r)
    hd, hs, ht = edt_ref.host_build(occ, r)
    assert np.array_equal(d, hd) and np.array_equal(s, hs)
    assert np.array_equal(t.view(np.uint32), ht.view(np.uint32))
    d2, s2, t2 = _native(occ, r)
    assert np.array_equal(d2, d) and np.array_equal(s2, s) and np.array_equal(t2.view(np.uint32), t.view(np.uint32))
    assert np.array_equal(d, edt_ref.scipy_sqdist(occ))
    if occ.size <= 128 ** 3 and d.max() <= 2500:       # the lattice check enumerates every offset at distance D
        edt_ref.check_sites(occ, d, s)
    assert np.array_equal(t.view(np.uint32), edt_ref.record(occ, d, s, r).view(np.uint32))


def test_public_transform_on_the_callers_device():
    import pytorch_volumetric_b200 as pv
    occ = _random((40, 50, 60), 0.1, seed=2)
    for src in (torch.from_numpy(occ), torch.from_numpy(occ).cuda(), occ.astype(np.uint8)):
        D, site = pv.occupancy_distance_transform(src)
        want = "cuda" if torch.is_tensor(src) and src.is_cuda else "cpu"
        assert D.device.type == want and D.dtype == torch.int32 and site.dtype == torch.int64
        hd, hs, _ = edt_ref.host_build(occ, 1.0)
        assert np.array_equal(D.cpu().numpy(), hd) and np.array_equal(site.cpu().numpy(), hs)


# ---------------------------------------------------------------- 3. from_points
def test_from_points_occupancy_equals_the_voxel_grid_scatter():
    import pytorch_volumetric_b200 as pv
    g = torch.Generator().manual_seed(0)
    rng = [[-0.5, 0.5], [-0.3, 0.4], [0.0, 0.6]]
    pts = (torch.rand(20000, 3, generator=g) * 1.4 - 0.7).cuda()     # some fall outside the range
    sdf = pv.OccupancySDF.from_points(pts, 0.02, rng, device="cuda")
    grid = pv.VoxelGrid(0.02, rng, dtype=torch.bool, device="cuda")
    grid[pts] = True
    assert torch.equal(sdf.occupancy, grid.get_voxel_values())
    d, s, t = _native(grid.get_voxel_values().cpu().numpy(), 0.02)
    assert torch.equal(sdf._table.cpu(), torch.from_numpy(t))
    assert np.array_equal(sdf.voxels.raw_data.cpu().numpy().view(np.uint32), t[:, 0].view(np.uint32))
    assert np.array_equal(sdf.voxels_grad.cpu().numpy().view(np.uint32), t[:, 1:].view(np.uint32))
    # the box of the occupied voxel centres, widened by half a cell
    idx = torch.nonzero(sdf.occupancy).cpu().numpy()
    lo = np.array([min(r) for r in sdf.ranges])
    box = np.stack([lo + idx.min(0) * 0.02 - 0.01, lo + idx.max(0) * 0.02 + 0.01], 1)
    assert np.allclose(sdf.surface_bounding_box().numpy(), box, atol=1e-12)
    assert np.allclose(sdf.surface_bounding_box(padding=0.1).numpy(), box + [[-0.1, 0.1]], atol=1e-12)


# ---------------------------------------------------------------- 4. lookups
@pytest.mark.parametrize("interpolation", ["nearest", "trilinear"])
def test_call_equals_the_grid_reference(interpolation):
    import pytorch_volumetric_b200 as pv
    rng = [[-0.4, 0.4], [-0.3, 0.35], [-0.2, 0.5]]
    grid = pv.VoxelGrid(0.01, rng, dtype=torch.bool, device="cuda")
    occ = torch.from_numpy(_random(tuple(grid.get_voxel_values().shape), 0.02, seed=5)).cuda()
    sdf = pv.OccupancySDF(occ, 0.01, rng, interpolation=interpolation, device="cuda")
    ref = grid_ref.Grid.of(sdf)
    g = torch.Generator().manual_seed(1)
    pts = torch.rand(50000, 3, generator=g) * torch.tensor([1.2, 1.1, 1.1]) - torch.tensor([0.6, 0.55, 0.4])
    val, grad = sdf(pts.cuda())
    p = pts.numpy()
    if interpolation == "nearest":
        rep, bad = grid_ref.compare_nearest(ref.nearest(p), val.cpu().numpy(), grad.cpu().numpy(),
                                            key=sdf.voxel_keys(pts.cuda()).cpu().numpy())
    else:
        rep, bad = grid_ref.compare_trilinear(ref.trilinear(p), val.cpu().numpy(), grad.cpu().numpy())
    assert all(len(b) == 0 for b in bad.values()), (rep, {k: len(b) for k, b in bad.items()})
    inb = ref.in_range(grid_ref.as_points(p))
    assert inb.any() and (~inb).any()
    # the inherited views work without a ground-truth SDF
    if interpolation == "nearest":                  # in range, outside_surface reads the same voxel
        outside = sdf.outside_surface(pts.cuda()).cpu().numpy()
        assert np.array_equal(outside[inb], (val.cpu().numpy() > 0)[inb])
    assert sdf.get_voxel_view() is sdf.voxels
    view = sdf.get_voxel_view(pv.VoxelGrid(0.05, rng, device="cuda"))
    assert torch.isfinite(view.raw_data).all()
    inside = sdf.get_filtered_points(lambda v: v < 0)
    assert len(inside) == int(occ.sum())
    out_of_range = torch.tensor([[2.0, 0.0, 0.0]], device="cuda")
    assert torch.isfinite(sdf.voxels[out_of_range]).all()


# ---------------------------------------------------------------- 5. as a scene
@pytest.mark.parametrize("kind", ["nearest", "hand"])
def test_tabletop_cloud_as_a_scene(tmp_path, monkeypatch, kind):
    import sys
    import os
    import pytorch_volumetric_b200 as pv
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import c4bench
    from test_gpu_scene import _check, robot_of
    cloud = c4bench.scene_points(10 ** 5, 200).cuda()
    if kind == "hand":         # the cloud scaled and moved about the fingers
        cloud = cloud * 0.15 + torch.tensor([0.0, 0.0, 0.25], device="cuda")
        rng, r = [[-0.2, 0.2], [-0.2, 0.2], [0.1, 0.45]], 0.005
    else:
        rng, r = [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]], 0.02
    robot, q = robot_of(tmp_path, kind)
    robot.set_joint_configuration(q)
    lp = robot.link_surface_points(num_points=256, seed=1)
    seen = False
    for interp in ("nearest", "trilinear"):
        scene = pv.OccupancySDF.from_points(cloud, r, rng, interpolation=interp, device="cuda")
        for m in (0.02, 0.1):
            fused, cost = _check(monkeypatch, robot, scene, lp, None, m, (kind, interp, m))
            seen |= bool((cost[0] > 0).any())
    assert seen
