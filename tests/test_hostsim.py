"""CPU tier: the DEVICE code of the kernels (pvb_device.cuh, compiled for the host by tests/hostsim) against the
reference's golden vectors and the oracle -- the same assertions as the -m gpu parity tests, on the per-thread
arithmetic of grid_eval / mesh_eval / the crossing-parity walks / sphere_eval.  What this cannot see is the kernel
scaffolding around those functions (tiling, TMA staging, running min, stores); the -m gpu tests cover that."""
import numpy as np
import pytest
import torch

import hostsim_lib as hs
import workloads
from helpers import classify_composed, classify_mesh_mismatch, golden, port_mesh, pv_factory, ray_noise, sphere_spec
from pytorch_volumetric_b200 import _native as nat

TOL = 1e-5


def _golden_grid(z, val_key="table_val", grad_key="table_grad", ranges=None, **kw):
    shape = tuple(int(s) for s in z["table_shape"])
    ranges = [tuple(r) for r in z["ranges"]] if ranges is None else ranges
    return hs.grid_desc(torch.from_numpy(z[val_key]).reshape(shape), torch.from_numpy(z[grad_key]), ranges, z["bb"], **kw)


@pytest.mark.parametrize("name", ["probe", "drill"])
def test_grid_eval_vs_reference_golden(name, built_lib):
    z = golden(f"ref_cachedsdf_{name}")
    d, keep = _golden_grid(z)
    val, grad, key = hs.grid_lookup(d, z["q"])
    inb = z["inbound"]
    assert np.array_equal(key >= 0, inb)                        # in-range mask: bit-exact
    assert np.array_equal(key[inb], z["keys"][inb])             # ravelled voxel key: bit-exact
    assert np.array_equal(val[inb], z["val"][inb]) and np.array_equal(grad[inb], z["grad"][inb])     # pure gathers
    oob = ~inb
    assert np.abs(val[oob] - z["val"][oob]).max() <= 2 * np.spacing(np.abs(z["val"][oob]).max())
    assert np.abs(grad[oob] - z["grad"][oob]).max() <= 3e-7
    vb, gb = hs.grid_lookup(d, z["q"], branchy=True)             # the composed kernels' instantiation
    assert np.array_equal(vb, val) and np.array_equal(gb, grad)


def test_grid_eval_fp32_range_mode(built_lib):
    z = golden("ref_cachedsdf_probe")
    rng32 = [(float(a), float(b)) for a, b in z["ranges_f32range"]]
    d, keep = _golden_grid(z, "table_val_f32range", "table_grad_f32range", ranges=rng32)
    assert d.flags & nat.PVB_GRID_INDEX_FP32
    val, grad, key = hs.grid_lookup(d, z["q"])
    inb = z["inbound_f32range"]
    assert np.array_equal(key >= 0, inb) and np.array_equal(key[inb], z["keys_f32range"][inb])
    assert np.array_equal(val[inb], z["val_f32range"][inb]) and np.array_equal(grad[inb], z["grad_f32range"][inb])


def test_grid_eval_boundary_points_take_the_exact_path(built_lib):
    """Points a few ulps around every cell boundary of every axis: the key still equals the reference formula
    (oracle port, fp64 index arithmetic), i.e. the rare out-of-line exact path is wired correctly."""
    from oracle import port
    z = golden("ref_cachedsdf_probe")
    d, keep = _golden_grid(z)
    shape = tuple(int(s) for s in z["table_shape"])
    c = port.CachedSDFPort("probe", float(z["resolution"]), z["range_in"], port.MeshSDFPort(port_mesh("probe")),
                           tables=(torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"])))
    rng = np.random.default_rng(0)
    lo = np.array([r[0] for r in z["ranges"]]); hi = np.array([r[1] for r in z["ranges"]])
    pts = []
    for ax in range(3):
        res = (hi[ax] - lo[ax]) / (shape[ax] - 1)
        b = (lo[ax] + (np.arange(shape[ax] - 1) + 0.5) * res).astype(np.float32)
        for step in range(-3, 4):
            col = b.copy()
            for _ in range(abs(step)):
                col = np.nextafter(col, np.float32(np.inf if step > 0 else -np.inf))
            p = rng.uniform(lo, hi, size=(len(col), 3)).astype(np.float32)
            p[:, ax] = col
            pts.append(p)
    pts = np.concatenate(pts)
    _, _, key = hs.grid_lookup(d, pts)
    _, flat, inb = c.index_and_mask(torch.from_numpy(pts))
    assert np.array_equal(key >= 0, inb.numpy())
    assert np.array_equal(key[inb.numpy()], flat.numpy()[inb.numpy()])


def test_grid_eval_gt_strategy(built_lib):
    from pytorch_volumetric_b200.sdf import OutOfBoundsStrategy
    z = golden("ref_cachedsdf_probe")
    d, keep = _golden_grid(z, strategy=OutOfBoundsStrategy.LOOKUP_GT_SDF, gt_obj=pv_factory("probe"))
    n = len(z["val_gt"])
    val, grad, _ = hs.grid_lookup(d, z["q"][:n])
    inb = z["inbound"][:n]
    assert np.array_equal(val[inb], z["val_gt"][inb])
    assert np.abs(val[~inb] - z["val_gt"][~inb]).max() < 1e-6
    assert (np.abs(grad[~inb] - z["grad_gt"][~inb]).max(axis=-1) > 1e-5).mean() < 2e-3


@pytest.mark.parametrize("name", ["probe", "wrench", "drill"])
def test_mesh_eval_vs_reference_golden(name, built_lib):
    z = golden(f"ref_meshsdf_{name}")
    obj = pv_factory(name)
    d, keep = hs.mesh_desc(obj)
    dist, grad, closest, face = hs.mesh_query(d, z["pts"])
    sign_bad = (np.sign(dist) != np.sign(z["distance"])) & (np.abs(z["distance"]) > 1e-6)
    assert sign_bad.mean() <= (0.0 if obj.is_closed else 2e-3)
    ok = ~sign_bad
    bad_v, bad_g, rep = classify_mesh_mismatch(dist[ok], grad[ok], z["distance"][ok], z["gradient"][ok], TOL)
    assert bad_v == 0 and bad_g == 0, rep
    assert (face >= 0).all() and (face < len(workloads.fixture_mesh(name)[1])).all()


@pytest.mark.parametrize("name,n", [("probe", 8000), ("wrench", 8000), ("scene_overlap", 4000), ("scene_separated", 4000)])
def test_mesh_eval_vs_oracle(name, n, oracle_lib, built_lib):
    obj = pv_factory(name, ray_seed=5)
    mesh = port_mesh(name)
    v, _ = workloads.fixture_mesh(name)
    pts = workloads.uniform_points(n, v.min(0) - 0.02, v.max(0) + 0.02, 21)
    d, keep = hs.mesh_desc(obj)
    dist, grad, closest, face = hs.mesh_query(d, pts)
    c_ref, d_ref, g_ref, _ = mesh.closest_point(pts, compute_normal=True, ray_noise=ray_noise(5, n))
    d_ref, g_ref = d_ref.numpy(), g_ref.numpy()
    scale = float(np.abs(v).max())
    assert np.abs(np.abs(dist) - np.abs(d_ref)).max() < 5e-6 * max(1.0, scale / 0.1)
    sign_bad = (np.sign(dist) != np.sign(d_ref)) & (np.abs(d_ref) > 1e-6)
    assert sign_bad.mean() <= (0.0 if obj.is_closed else 2e-3)
    ok = ~sign_bad
    bad_v, bad_g, rep = classify_mesh_mismatch(dist[ok], grad[ok], d_ref[ok], g_ref[ok], TOL, coord_scale=scale)
    assert bad_v == 0 and bad_g == 0, rep


def test_jitter_hash_matches_the_host_mirror(built_lib):
    """tests/helpers.py ray_noise (numpy) == pvb_device.cuh hash_normal, bit for bit."""
    want = ray_noise(5, 1000)
    got = np.array([[hs.lib().sim_hash_normal(5, i, c) for c in range(3)] for i in range(1000)], dtype=np.float32)
    assert np.array_equal(got, want)


def test_axis_parity_is_exact_on_lattice_aligned_queries(oracle_lib, built_lib):
    """Closed meshes: the +x walk with symbolic perturbation must give the true inside/outside even when the ray
    passes exactly through vertices and along edges -- queries ON the vertex lattice of a box mesh and of the
    bumpy sphere (y, z copied from mesh vertices), checked against an analytic / generic-direction answer."""
    # axis-aligned box [0,1]^3, 12 triangles: rays through corners, along edges and through the face diagonals
    v = np.array([[x, y, z] for x in (0., 1.) for y in (0., 1.) for z in (0., 1.)], dtype=np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                  [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    import pytorch_volumetric_b200 as pv
    box = pv.MeshObjectFactory("box", mesh=(v, f))
    assert box.is_closed
    d, keep = hs.mesh_desc(box)
    g = np.array([-0.5, 0.0, 0.25, 0.5, 0.75, 1.0, 1.5])
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    px, _ = hs.parity(d, pts)
    strictly_inside = ((pts > 0) & (pts < 1)).all(1)
    strictly_outside = ((pts < 0) | (pts > 1)).any(1)
    assert (px[strictly_inside] == 1).all() and (px[strictly_outside] == 0).all()
    # bumpy sphere: (y, z) of every query copied from a vertex, x swept: compare with a generic diagonal ray
    vs, fs = workloads.bumpy_sphere(40, 21)
    sph = pv.MeshObjectFactory("bumpy", mesh=(vs, fs))
    d2, keep2 = hs.mesh_desc(sph)
    rng = np.random.default_rng(0)
    pick = rng.integers(0, len(vs), 3000)
    q = vs[pick].astype(np.float32)
    q[:, 0] = rng.uniform(vs[:, 0].min() - 0.02, vs[:, 0].max() + 0.02, len(q)).astype(np.float32)
    dirs = np.tile(np.array([[0.5377, 0.6123, 0.5796]], dtype=np.float32), (len(q), 1))
    px, pr = hs.parity(d2, q, dirs)
    dist, _, _, _ = hs.mesh_query(d2, q, mode=0)
    clear = np.abs(dist) > 1e-6                  # not on the surface itself
    assert np.array_equal(px[clear], pr[clear])


def test_winding_and_sphere(oracle_lib, built_lib):
    from oracle import port
    obj = pv_factory("probe")
    d, keep = hs.mesh_desc(obj, with_winding=True)
    v, f = workloads.fixture_mesh("probe")
    pts = workloads.uniform_points(3000, v.min(0) - 0.02, v.max(0) + 0.02, 4)
    w = hs.winding(d, pts)
    w_ref = port.winding_number_port(v, f, pts.numpy())
    assert np.abs(w - w_ref).max() < 0.05 and np.array_equal(np.abs(w) > 0.5, np.abs(w_ref) > 0.5)
    p = workloads.uniform_points(1000, [-1] * 3, [1] * 3, 9)
    val, grad = hs.sphere(0.3, p)
    r = p.norm(dim=-1)
    assert np.allclose(val, (r - 0.3).numpy(), atol=1e-6) and np.allclose(grad, (p / r[:, None]).numpy(), atol=1e-5)


def test_c1_full_size_drill_grid_vs_oracle(oracle_lib, built_lib):
    """BASELINE configs[0] (C1, SURVEY 8d): 50^3 = 125 000 grid points over the drill's bounding box (padding 0.01)
    + 1e-6 jitter, seed 0 -- the reference's own CPU-runnable case -- device code against the oracle's BVH
    evaluator at full size."""
    from oracle import tp_open3d
    obj = pv_factory("drill", ray_seed=0)
    mesh = port_mesh("drill")
    bb = obj.bounding_box(padding=0.01)
    axes = [torch.linspace(float(bb[k, 0]), float(bb[k, 1]), 50, dtype=torch.float64) for k in range(3)]
    g = torch.Generator().manual_seed(0)
    pts = (torch.cartesian_prod(*axes) + 1e-6 * torch.randn(125000, 3, generator=g, dtype=torch.float64)).float()
    d, keep = hs.mesh_desc(obj)
    dist, grad, closest, face = hs.mesh_query(d, pts)
    prev = tp_open3d.QUERY_METHOD
    tp_open3d.QUERY_METHOD = "bvh"
    try:
        _, d_ref, g_ref, _ = mesh.closest_point(pts, compute_normal=True, ray_noise=ray_noise(0, len(pts)))
    finally:
        tp_open3d.QUERY_METHOD = prev
    d_ref, g_ref = d_ref.numpy(), g_ref.numpy()
    assert np.abs(np.abs(dist) - np.abs(d_ref)).max() < 1e-5
    sign_bad = (np.sign(dist) != np.sign(d_ref)) & (np.abs(d_ref) > 1e-6)
    assert sign_bad.sum() == 0
    bad_v, bad_g, rep = classify_mesh_mismatch(dist, grad, d_ref, g_ref, TOL, coord_scale=float(np.abs(bb).max()))
    assert bad_v == 0 and bad_g == 0, rep


# ---------------------------------------------------------------- ComposedSDF / RobotSDF device logic
def _close(a, b, tol=1e-5):
    return np.abs(a - b) <= tol


def _composed_golden_descs():
    zc = golden("ref_cachedsdf_probe")
    grid, keep = _golden_grid(zc)
    z = golden("ref_composed")
    return z, [grid, grid, hs.sphere_desc(float(z["sphere_radius"])), grid], keep


def _table_spec(z, bb):
    shape = tuple(int(s) for s in z["table_shape"])
    return {"kind": "grid", "val": z["table_val"].reshape(shape).astype(np.float64),
            "grad": z["table_grad"].reshape(*shape, 3).astype(np.float64),
            "lo": np.array([r[0] for r in z["ranges"]], dtype=np.float64),
            "hi": np.array([r[1] for r in z["ranges"]], dtype=np.float64), "bb": np.asarray(bb, dtype=np.float64)}


def _composed_golden_specs(z):
    zc = golden("ref_cachedsdf_probe")
    g = _table_spec(zc, zc["bb"])
    return [g, g, sphere_spec(float(z["sphere_radius"])), g]


def test_composed_logic_vs_reference_golden(built_lib):
    """composed_xform / composed_consider / composed_rotate_back (the arithmetic of both composed kernels) against
    the vectors the reference's ComposedSDF produced: plain (S transforms) and configuration-batched (S x A)."""
    z, descs, keep = _composed_golden_descs()
    S, A = int(z["S"]), int(z["A"])
    v, g, w = hs.composed(descs, z["tmat"][:S], 1, z["q"])
    # within 1e-5 of the reference's vectors; an fp32 rigid transform in front of a nearest-voxel lookup may flip a key
    # at a cell boundary -- every exceedance must classify as such a flip (helpers.classify_composed)
    specs = _composed_golden_specs(z)
    P = len(z["q"])
    n_ex, n_un, rep = classify_composed(v[None], g[None], z["val_plain"][None], z["grad_plain"][None], specs,
                                        z["tmat"][:S].reshape(S, 1, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 2e-3 * P, rep
    vb, gb, wb = hs.composed(descs, z["tmat"], A, z["q"])
    n_ex, n_un, rep = classify_composed(vb.reshape(A, P), gb.reshape(A, P, 3), z["val_batched"].reshape(A, P),
                                        z["grad_batched"].reshape(A, P, 3), specs, z["tmat"].reshape(S, A, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 2e-3 * A * P, rep
    # batched == per-configuration loop, exactly (tests/test_model_to_sdf.py:206-212)
    tm = z["tmat"].reshape(S, A, 4, 4)
    for a in range(A):
        va, ga, wa = hs.composed(descs, np.ascontiguousarray(tm[:, a]), 1, z["q"])
        sl = slice(a * len(z["q"]), (a + 1) * len(z["q"]))
        assert np.array_equal(va, vb[sl]) and np.array_equal(ga, gb[sl]) and np.array_equal(wa, wb[sl])


def test_composed_result_does_not_depend_on_the_visiting_order(built_lib):
    """Exact pruning + the explicit first-index tie rule: index order, reversed order and the kernels' bit-reversed
    order give bit-identical values, gradients and argmin indices -- and equal the unpruned evaluation."""
    z, descs, keep = _composed_golden_descs()
    S, A = int(z["S"]), int(z["A"])
    ref = hs.composed(descs, z["tmat"], A, z["q"], order=range(S))
    for order in (list(range(S))[::-1], hs.bit_reversed_order(S), [2, 0, 3, 1]):
        got = hs.composed(descs, z["tmat"], A, z["q"], order=order)
        assert all(np.array_equal(a, b) for a, b in zip(ref, got)), order
    # unpruned evaluation: every sub-SDF evaluated alone (a one-element composition never prunes), argmin in numpy
    per = [hs.composed([descs[s]], z["tmat"][s * A:(s + 1) * A], A, z["q"]) for s in range(S)]
    vals = np.stack([p[0] for p in per]); grads = np.stack([p[1] for p in per])
    which = vals.argmin(0)                       # numpy: first index on ties, like torch
    assert np.array_equal(ref[2], which.astype(np.int32))
    assert np.array_equal(ref[0], np.take_along_axis(vals, which[None], 0)[0])
    assert np.array_equal(ref[1], np.take_along_axis(grads, which[None, :, None], 0)[0])
    # ties: identical sub-SDFs at the same pose resolve to index 0 in every order
    for n_same in (2, 3, 4, 7):
        tm = np.repeat(z["tmat"][:1], n_same, axis=0)
        for order in (range(n_same), list(range(n_same))[::-1], hs.bit_reversed_order(n_same)):
            _, _, w = hs.composed([descs[0]] * n_same, tm, 1, z["q"], order=order)
            assert int(w.max()) == 0
    assert hs.bit_reversed_order(8) == [0, 4, 2, 6, 1, 5, 3, 7] and hs.bit_reversed_order(3) == [0, 2, 1]


def test_robot_logic_vs_reference_golden(built_lib):
    """The reference's RobotSDF vectors (offset_wrench.urdf, 5 configurations): link table + object->link transforms
    from the golden file through the composed device logic."""
    z = golden("ref_robot_wrench")
    shape = tuple(int(s) for s in z["table_shape"])
    v_, _ = workloads.fixture_mesh("wrench")
    bb = np.stack([v_.min(0), v_.max(0)], axis=1)
    grid, keep = hs.grid_desc(torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"]),
                              [tuple(r) for r in z["ranges"]], bb)
    val, grad, _ = hs.composed([grid], z["obj_to_link"], 5, z["q"])
    n_ex, n_un, rep = classify_composed(val.reshape(5, -1), grad.reshape(5, -1, 3), z["val"], z["grad"],
                                        [_table_spec(z, bb)], z["obj_to_link"].reshape(1, 5, 4, 4), z["q"])
    assert n_un == 0 and n_ex <= 3e-3 * val.size, rep


def test_composed_of_meshes_logic_vs_oracle(oracle_lib, built_lib):
    """Mesh sub-SDFs (the kMesh instantiation: bounded search radius, sign walk skipped outside a closed mesh's box)
    against the oracle's ComposedSDF of MeshSDFs, as in tests/test_sdf.py:61-80."""
    from oracle import port, tp_pytorch_kinematics as opk
    obj = pv_factory("probe", ray_seed=1)
    d, keep = hs.mesh_desc(obj)
    tm = torch.eye(4).repeat(2, 1, 1)
    tm[0, :3, 3] = torch.tensor([0.1, 0.0, 0.0])
    tm[1, :3, 3] = torch.tensor([-0.2, 0.0, 0.2])
    q = workloads.uniform_points(4000, (-0.2, -0.05, -0.1), (0.3, 0.05, 0.3), seed=4)
    v, g, w = hs.composed([d, d], tm, 1, q)
    mesh = port_mesh("probe")
    ref = port.ComposedSDFPort([port.MeshSDFPort(mesh), port.MeshSDFPort(mesh)], opk.Transform3d(matrix=tm))
    np.random.seed(0)
    vr, gr = ref(q)
    assert np.abs(v - vr.numpy()).max() < 1e-5
    assert (np.abs(g - gr.numpy()).max(-1) > 1e-5).mean() < 2e-3
    # pruned == unpruned for meshes too
    per = [hs.composed([d], tm[s:s + 1], 1, q) for s in range(2)]
    vals = np.stack([p[0] for p in per])
    assert np.array_equal(w, vals.argmin(0).astype(np.int32)) and np.array_equal(v, vals.min(0))


def test_closest_point_fuzz_on_degenerate_soups(oracle_lib, built_lib):
    """BVH4 nearest-first descent + Ericson triangle test of the device code against the oracle's brute force on
    random triangle soups: coplanar, coincident / duplicated vertices, slivers, far from the origin, zero-area
    triangles; queries around, near and exactly on the vertices."""
    import pytorch_volumetric_b200 as pv
    from oracle import _geom
    rng = np.random.default_rng(0)
    for it in range(24):
        kind = it % 6
        nv, nf = int(rng.integers(4, 300)), int(rng.integers(1, 600))
        v = rng.normal(size=(nv, 3)) * 10 ** rng.uniform(-2, 1)
        if kind == 1: v[:, 2] = 0.0
        if kind == 2: v = np.round(v, 1)
        if kind == 3: v[:, 0] *= 1e-3
        if kind == 4: v += 100.0
        f = rng.integers(0, nv, size=(nf, 3)).astype(np.int32)
        if kind == 5: f[:, 2] = f[:, 1]
        d, keep = hs.mesh_desc(pv.MeshObjectFactory(f"fuzz{it}", mesh=(v, f)))
        lo, hi = v.min(0), v.max(0)
        ext = (hi - lo).max() + 1e-3
        pts = np.concatenate([rng.uniform(lo - 0.3 * ext, hi + 0.3 * ext, size=(1500, 3)),
                              v[rng.integers(0, nv, 300)] + rng.normal(size=(300, 3)) * 1e-4 * ext,
                              v[rng.integers(0, nv, 100)]]).astype(np.float32)
        dist, grad, closest, face = hs.mesh_query(d, pts, mode=0)
        c_ref = _geom.TriangleSoup(v.astype(np.float32), f).closest_points(pts, method="brute")[0]
        d_dev = np.linalg.norm(closest.astype(np.float64) - pts, axis=1)
        d_ref = np.linalg.norm(c_ref.astype(np.float64) - pts, axis=1)
        scale = max(1.0, float(np.abs(v).max()))
        assert np.abs(d_dev - d_ref).max() <= 2e-6 * scale, (it, kind)
        assert (np.abs(np.abs(dist) - d_dev) <= 1e-5 * scale).all() and (dist >= 0).all()      # unsigned mode
        assert ((face >= 0) & (face < nf)).all()


def test_axis_parity_fuzz_on_perturbed_closed_meshes(built_lib):
    """Closed meshes with vertices snapped to a coarse lattice (aligned coordinates, degenerate faces) and random
    rigid poses: the exact +x walk equals the unanimous answer of three generic-direction watertight rays, for
    random queries and for queries whose (y, z) are copied from mesh vertices (rays through vertices)."""
    import pytorch_volumetric_b200 as pv
    rng = np.random.default_rng(1)
    checked = 0
    for it in range(8):
        v, f = workloads.bumpy_sphere(int(rng.integers(6, 40)), int(rng.integers(4, 30)))
        v = v * (1 + 0.06 * rng.normal(size=(len(v), 1)))
        if it % 2 == 0:
            v = np.round(v, 2)
        if it % 4 < 2:
            R = workloads.random_rigid(1, seed=it)[0].numpy().astype(np.float64)
            v = v @ R[:3, :3].T + R[:3, 3]
        obj = pv.MeshObjectFactory(f"closed{it}", mesh=(v, f))
        if not obj.is_closed:
            continue
        d, keep = hs.mesh_desc(obj)
        n = 1500
        q = np.concatenate([rng.uniform(v.min(0) - 0.02, v.max(0) + 0.02, size=(n, 3)),
                            v[rng.integers(0, len(v), n)]]).astype(np.float32)
        q[n:, 0] = rng.uniform(v[:, 0].min() - 0.02, v[:, 0].max() + 0.02, n)
        px, _ = hs.parity(d, q)
        votes = np.zeros(len(q), int)
        for _ in range(3):
            dr = rng.normal(size=3)
            votes += hs.parity(d, q, np.tile((dr / np.linalg.norm(dr)).astype(np.float32), (len(q), 1)))[1]
        dist = hs.mesh_query(d, q, mode=0)[0]
        m = (np.abs(dist) > 1e-5) & ((votes == 0) | (votes == 3))
        assert np.array_equal(px[m], (votes[m] == 3).astype(np.int32)), it
        checked += int(m.sum())
    assert checked > 10_000


def test_robot_serial_tiles_and_flush_pieces_cover_everything_once(built_lib):
    """Index arithmetic of robot_serial_kernel (pvb_device.cuh rs_tile / rs_flush_piece): for every configuration count
    the tiles are full, disjoint and cover [0, cfg_count); for every tile shape (LC = 32..1), step size (4 / 8 points) and
    flush mode (per warp / per block) the 16-byte pieces cover every value and gradient float of the tile exactly once,
    consecutive pieces are consecutive in memory, and every piece is 16-byte aligned in the output."""
    import ctypes
    L = hs.lib()
    for cfg_count in list(range(1, 300)) + [1000, 4097]:
        seen = np.zeros(cfg_count, dtype=np.int32)
        n_tiles = (cfg_count >> 5) + bin(cfg_count & 31).count("1")
        for t in range(n_tiles):
            c0, lc = ctypes.c_int(), ctypes.c_int()
            L.sim_rs_tile(cfg_count, t, ctypes.byref(c0), ctypes.byref(lc))
            assert 0 <= lc.value <= 5 and c0.value % (1 << lc.value) == 0
            seen[c0.value:c0.value + (1 << lc.value)] += 1
        assert (seen == 1).all(), cfg_count
    for w_log2 in (0, 3):
        for chunk_log2 in (2, 3):
            for sub_log2 in range(6):
                LC = 32 >> sub_log2
                row_pts = 1 << (w_log2 + chunk_log2 + sub_log2)
                n_pieces = LC * row_pts
                val = np.zeros((LC, row_pts), dtype=np.int32)
                grad = np.zeros((LC, 3 * row_pts), dtype=np.int32)
                prev = None
                for c in range(n_pieces):
                    iv, row, part = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
                    L.sim_rs_flush_piece(c, chunk_log2, sub_log2, w_log2, ctypes.byref(iv), ctypes.byref(row), ctypes.byref(part))
                    assert 0 <= row.value < LC
                    if iv.value:
                        val[row.value, 4 * part.value:4 * part.value + 4] += 1
                    else:
                        grad[row.value, 4 * part.value:4 * part.value + 4] += 1
                    cur = (iv.value, row.value, part.value)
                    if prev is not None and prev[0] == cur[0] and prev[1] == cur[1]:
                        assert cur[2] == prev[2] + 1            # consecutive pieces are neighbours in the row
                    prev = cur
                assert (val == 1).all() and (grad == 1).all(), (w_log2, chunk_log2, sub_log2)


INT_MAX = 2 ** 31 - 1


def _robot_int_extreme(n_pts):
    """The largest int intermediate robot_serial_kernel (pvb_kernels.cu) and robot_query_kernel form from n_pts, over
    every tile shape (LC = 32..1 lanes per point), step size (4 / 8 points) and flush mode (per warp / per block of 8
    warps): the step count's rounding n_pts + pts_per_step - 1, the tile ends tile_base + row_pts and pt_base +
    pts_per_step of every warp the super-step loop runs (inactive ones included), the last point index, and
    robot_query_kernel's 32-point tiles."""
    worst = n_pts + 31                                                       # (n_pts + kRbTilePts - 1) / kRbTilePts
    worst = max(worst, -(-n_pts // 32) * 32)                                 # tile * 32 + 32 of its last tile
    for chunk_log2 in (2, 3):
        for sub_log2 in range(6):
            pps = (1 << chunk_log2) << sub_log2                              # points a warp finishes per step
            n_chunks = -(-n_pts // pps)
            n_super = -(-n_chunks // 8)
            last_chunk = 8 * n_super - 1                                     # sup * 8 + warp, every warp
            for coop in (False, True):
                tile_end = (n_super * 8 * pps) if coop else (last_chunk + 1) * pps
                worst = max(worst, n_pts + pps - 1, tile_end, last_chunk * pps + pps - 1, n_chunks + 7)
    return worst


def test_robot_int_point_guard_is_exact(built_lib):
    """rs_int_pts_ok (pvb_device.cuh), the guard that sends a batch to the int-indexed robot kernels: every point count
    it accepts keeps every int intermediate of robot_serial_kernel and robot_query_kernel at or below INT_MAX, and the
    first count it refuses is the first that would wrap -- the guard is exact, not merely safe."""
    import ctypes
    L = hs.lib()
    ok = lambda n: bool(L.sim_rs_int_pts_ok(ctypes.c_longlong(n)))
    limit = 2 ** 31 - 2048
    assert ok(limit) and not ok(limit + 1)
    assert _robot_int_extreme(limit) <= INT_MAX < _robot_int_extreme(limit + 1)
    for n in list(range(limit - 4200, limit + 4200)) + [0, 1, 255, 256, 2047, 2048, 2 ** 31 - 1, 2 ** 31, 2 ** 40]:
        assert ok(n) == (n <= limit), n
        if ok(n):
            assert _robot_int_extreme(n) <= INT_MAX, n


def test_robot_tile_count_at_the_grid_row_limit(built_lib):
    """rs_tile_count (pvb_device.cuh), the grid rows robot_serial_kernel and robot_clearance_kernel launch: the tiles
    rs_tile enumerates, on both sides of 65535 rows (2 097 120 = 65535 x 32 configurations, and the counts just below it
    whose remainder splits into more than one tile)."""
    import ctypes
    L = hs.lib()
    counts = list(range(65530 * 32, 65537 * 32)) + [1, 31, 32, 33, 2 ** 31 - 1]
    for c in counts:
        n = L.sim_rs_tile_count(c)
        assert n == (c >> 5) + bin(c & 31).count("1"), c
        if c in (1, 31, 32, 33, 65535 * 32 - 1, 65535 * 32 + 33):
            seen, last = 0, -1
            for t in range(n):
                c0, lc = ctypes.c_int(), ctypes.c_int()
                L.sim_rs_tile(c, t, ctypes.byref(c0), ctypes.byref(lc))
                assert c0.value == last + 1 or (t == 0 and c0.value == 0), (c, t)
                last = c0.value + (1 << lc.value) - 1
                seen += 1 << lc.value
            assert seen == c and last == c - 1, c
    assert L.sim_rs_tile_count(65535 * 32) == 65535
    assert L.sim_rs_tile_count(65535 * 32 + 1) == 65536
    # the largest counts below 65535 x 32 that still need more than 65535 rows: remainders of 2+ binary digits
    assert [c for c in range(65534 * 32, 65535 * 32) if L.sim_rs_tile_count(c) > 65535] == \
        [c for c in range(65534 * 32, 65535 * 32) if bin(c & 31).count("1") >= 2]


def test_robot_serial_nearest_sphere_key(built_lib):
    """rs_bound_key / rs_nearest (pvb_device.cuh): the link index rides in the 3 low mantissa bits of each sphere bound
    and the smallest key names the first link to visit.  Always a real link (0 <= pred < n_sdf), whatever mix of finite,
    -inf (bound not valid) and +inf (slot beyond n_sdf) bounds comes in; the argmin whenever the smallest finite bound
    is separated from the rest by more than the 7-ulp blur of the keys; -inf at slot 0 wins (it is a valid float)."""
    import ctypes
    L = hs.lib()
    rng = np.random.default_rng(7)
    n = 200_000
    for n_sdf in range(1, 9):
        lb = rng.normal(0.0, 0.3, size=(n, 8)).astype(np.float32)
        lb[rng.random((n, 8)) < 0.05] = -np.inf                      # bounds that are not valid
        lb[:n // 4] = np.abs(lb[:n // 4])                            # all-positive rows
        lb[n // 4:n // 2] = -np.abs(lb[n // 4:n // 2])               # all-negative rows
        lb[:, n_sdf:] = np.inf                                       # slots beyond n_sdf
        lb[:16] = -np.inf; lb[:16, n_sdf:] = np.inf                  # nothing valid at all
        pred = np.empty(n, np.int32)
        L.sim_rs_nearest(lb.ctypes.data_as(ctypes.c_void_p), ctypes.c_longlong(n), n_sdf,
                         pred.ctypes.data_as(ctypes.c_void_p))
        assert pred.min() >= 0 and pred.max() < n_sdf
        valid = lb[:, :n_sdf].copy()
        fin = np.isfinite(valid)
        rows = fin.all(axis=1)
        v = np.where(fin, valid, np.inf)
        order = np.sort(v, axis=1)
        with np.errstate(invalid="ignore"):
            gap = order[:, 1] - order[:, 0] if n_sdf > 1 else np.full(n, np.inf, np.float32)
        clear = rows & (gap > 16 * np.spacing(np.abs(order[:, 0]).astype(np.float32)))
        assert clear.sum() > n // 3
        assert np.array_equal(pred[clear], np.argmin(v, axis=1)[clear])
        neg0 = np.isneginf(lb[:, 0])
        assert (pred[neg0] == 0).all()

