"""CPU tier of the fp64 grid reference (tests/grid_ref.py): it reproduces the reference's own vectors, it agrees with
the host build of the device code (pvb_device.cuh: grid_eval and grid_trilinear_eval) on boundary-dense point sets in
both range modes, and each of its bounds is within 10x of the error that build actually shows."""
import numpy as np
import pytest
import torch

import grid_ref as gr
import hostsim_lib as hs
from helpers import golden


def golden_grid(name, fp32_range=False):
    """(Grid, z, suffix) of a golden table; fp32_range: the range given as Python floats."""
    import pytorch_volumetric_b200 as pv
    z = golden(f"ref_cachedsdf_{name}")
    sfx = "_f32range" if fp32_range else ""
    rin = [(float(a), float(b)) for a, b in z["range_in"]] if fp32_range else z["range_in"]
    ranges = pv.get_divisible_range_by_resolution(float(z["resolution"]), rin)
    shape = tuple(int(s) for s in z["table_shape"])
    return gr.Grid(z["table_val" + sfx].reshape(shape), z["table_grad" + sfx], ranges, z["bb"]), z, sfx


def dyadic_grid(fp32_range):
    import pytorch_volumetric_b200 as pv
    val, grad = gr.dyadic_table()
    bb = pv.SphereSDF(gr.DYADIC_RADIUS).surface_bounding_box().numpy()
    return gr.Grid(val, grad, gr.dyadic_ranges(fp32_range), bb)


GRIDS = [("probe", False), ("probe", True), ("drill", False), ("dyadic", False), ("dyadic", True)]


def make_grid(name, fp32_range):
    return dyadic_grid(fp32_range) if name == "dyadic" else golden_grid(name, fp32_range)[0]


def points(g, seed=0):
    return gr.all_points(gr.point_sets(g.lo64, g.hi64, g.shape, seed=seed))


def host_desc(g, interpolation="nearest"):
    tv = torch.from_numpy(g.val32)
    tg = torch.from_numpy(g.grad.astype(np.float32))
    return hs.grid_desc(tv, tg, g.ranges, g.bb32, interpolation=interpolation)


@pytest.mark.parametrize("name,fp32_range", [("probe", False), ("probe", True), ("drill", False)])
def test_reference_equals_golden_vectors(name, fp32_range):
    """Keys, in-range mask and in-range values / gradients bit-exact; out-of-range values and gradients within the
    bounding-box bound of the reference's fp32 result."""
    g, z, sfx = golden_grid(name, fp32_range)
    q = z["q"]
    key, _ = g.keys(q)
    inb = z["inbound" + sfx]
    assert np.array_equal(key >= 0, inb)
    assert np.array_equal(key[inb], z["keys" + sfx][inb])
    ref = g.nearest(q)
    rep, bad = gr.compare_nearest(ref, z["val" + sfx], z["grad" + sfx], key=np.where(inb, z["keys" + sfx], -1))
    assert all(len(b) == 0 for b in bad.values()), (rep, {k: v[:5] for k, v in bad.items()})


@pytest.mark.parametrize("name,fp32_range", GRIDS)
def test_nearest_equals_host_build(name, fp32_range):
    """grid_eval compiled for the host: keys and in-range gathers bit-exact, the bounding-box rule within its bound,
    NaN where the reference is NaN -- on uniform, boundary-dense, half-way, range-end, lattice, outside and NaN points."""
    g = make_grid(name, fp32_range)
    p = points(g)
    d, _keep = host_desc(g)
    val, grad, key = hs.grid_lookup(d, p)
    ref = g.nearest(p)
    rep, bad = gr.compare_nearest(ref, val, grad, key=key)
    assert all(len(b) == 0 for b in bad.values()), (rep, {k: p[v[:5]] for k, v in bad.items()})


@pytest.mark.parametrize("name,fp32_range", GRIDS)
def test_trilinear_within_bounds_on_host_build(name, fp32_range):
    """grid_trilinear_eval compiled for the host within the trilinear bounds (gradients off cell faces, or either
    face's cell on them); values at lattice nodes whose cell fraction is 0 on every axis are bit-exact."""
    g = make_grid(name, fp32_range)
    sets = gr.point_sets(g.lo64, g.hi64, g.shape)
    p = gr.all_points(sets)
    d, _keep = host_desc(g, "trilinear")
    val, grad = hs.grid_trilinear(d, p)
    rep, bad = gr.compare_trilinear(g.trilinear(p), val, grad)
    assert all(len(b) == 0 for b in bad.values()), (rep, {k: p[v[:5]] for k, v in bad.items()})
    node, key = gr.exact_nodes(g, p)
    assert np.array_equal(val[node], g.val32.reshape(-1)[key[node]])
    if name == "dyadic":
        assert node.sum() > 2000                  # every lattice node off the upper faces is exact in fp32 here


def test_bounds_are_tight():
    """Each bound is within 10x of the largest error the host build shows over all tables and point sets: the
    bounding-box value and gradient, the trilinear value and gradient."""
    worst = {"box value": 0.0, "box grad": 0.0, "trilinear value": 0.0, "trilinear grad": 0.0}
    for name, fp32_range in GRIDS:
        g = make_grid(name, fp32_range)
        p = points(g, seed=1)
        d, _keep = host_desc(g)
        val, grad, key = hs.grid_lookup(d, p)
        rep, _ = gr.compare_nearest(g.nearest(p), val, grad, key=key)
        worst["box value"] = max(worst["box value"], rep["value"])
        worst["box grad"] = max(worst["box grad"], rep["grad"])
        d, _keep = host_desc(g, "trilinear")
        val, grad = hs.grid_trilinear(d, p)
        ref = g.trilinear(p)
        inb = ref["inb"]
        rep, _ = gr.compare_trilinear({k: (v[inb] if k != "alt" else v[:, inb]) for k, v in ref.items()},
                                      val[inb], grad[inb])
        worst["trilinear value"] = max(worst["trilinear value"], rep["value"])
        worst["trilinear grad"] = max(worst["trilinear grad"], rep["grad"])
    print("largest error / bound on the host build:", {k: round(v, 3) for k, v in worst.items()})
    for k, v in worst.items():
        assert 0.1 <= v <= 1.0, (k, v)


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("fp32_range", [False, True])
def test_voxel_index_rule_equals_host_gridview(d, fp32_range):
    """The reference's VoxelGrid index rule equals the torch indexing of a host GridView (the reference's own
    formula) on boundary-dense points, in 1-3 dimensions and both range modes."""
    import pytorch_volumetric_b200 as pv
    box = [(-0.37, 0.41), (0.1, 0.9), (-2.0, -1.3)][:d]
    box = [(float(a), float(b)) for a, b in box] if fp32_range else np.array(box)
    vg = pv.VoxelGrid(0.02, box)
    vg.get_voxel_values().reshape(-1).copy_(torch.arange(1, vg.get_voxel_values().numel() + 1, dtype=torch.float32))
    p, want = gr.voxel_case(vg, box)
    got = vg[torch.from_numpy(p)].numpy()
    assert np.array_equal(got, np.where(want >= 0, want + 1, 0).astype(np.float32))
