"""CPU: pins the fp64 chamfer restatement (tests/chamfer_ref.py) to the vectors the unmodified reference wrote for
pairwise_distance_chamfer and PlausibleDiversity (oracle/make_golden.py: ref_chamfer_pairwise), checks its mesh
distance against the analytic box, and confirms on the host build of the device header the premise of the exact
box cloud that tests/test_gpu_chamfer_fp64.py compares bit for bit."""
import numpy as np
import pytest

import chamfer_ref as cr
import primitive_ref as pr
import workloads
from helpers import golden

U = cr.U32


def _probe_spec():
    return cr.mesh_spec(*workloads.fixture_mesh("probe"))


def _reference_bound(spec, left, right, pts, scale=1000.0):
    """Bound on |reference fp32 - fp64| of every composite's chamfer value: the fp32 composite and transform, the
    oracle's fp32 closest point (2e-6, the bound tests/test_hostsim.py holds at unit scale), and torch's fp32 mean of
    N terms (N u of the value)."""
    comp = np.einsum("bij,pjk->bpik", np.asarray(left, np.float64), np.asarray(right, np.float64)).reshape(-1, 4, 4)
    d = cr.per_pair(spec, comp, pts)
    dd = cr.transform_error(comp, pts) + cr.composite_error(left, right, pts) + 2e-6
    val = ((scale * d) ** 2).mean(axis=1)
    return val, cr.square_bound(d, dd, scale).mean(axis=1) + (len(pts) + 4) * U * val


def test_pairwise_restatement_equals_reference_golden():
    z = golden("ref_chamfer_pairwise")
    spec, pts = _probe_spec(), z["pts"]
    A, Bw = z["A"], z["B_w2l"]
    # B_world_to_link_tfs given, |A| = 5 != |B| = 3: the view re-chunks the B-major flat data into (5, 3)
    ref = cr.pairwise_distance_chamfer(spec, pts, A, Bw)
    assert ref.shape == z["err_given"].shape == (5, 3)
    val, tol = _reference_bound(spec, Bw, A, pts)
    assert np.array_equal(val.reshape(5, 3), ref)
    assert (np.abs(ref - z["err_given"]).reshape(-1) <= tol).all(), np.abs(ref - z["err_given"]).max()
    # the bound is far below the spread of the matrix: a transposed or re-ordered view cannot pass
    assert tol.max() < 0.1 * np.abs(np.diff(np.sort(z["err_given"].reshape(-1)))).min()
    # None: the inverses of A
    ref0 = cr.pairwise_distance_chamfer(spec, pts, A)
    _, tol0 = _reference_bound(spec, cr.rigid_inverse(A), A, pts)
    assert ref0.shape == (5, 5)
    assert (np.abs(ref0 - z["err_none"]).reshape(-1) <= tol0 + 3 * U * 1e6).all()
    # T^-1 T = I (up to the fp32 rounding of A's rotation) on the diagonal: the points' own distances
    assert (np.abs(np.diag(ref0) - cr.chamfer(spec, np.eye(4)[None], pts)[0]) <= np.diag(tol0.reshape(5, 5))).all()


def test_plausible_diversity_restatement_equals_reference_golden():
    z = golden("ref_chamfer_pairwise")
    spec, pts = _probe_spec(), z["pts"]
    T_est_inv, T_p = z["T_est_inv"], z["T_p"]
    pl, cov, best_est, best_pl = cr.plausible_diversity(spec, pts, T_est_inv, T_p)
    _, tol = _reference_bound(spec, T_est_inv, T_p, pts)
    assert abs(pl - z["pd_plausibility"]) <= tol.max() and abs(cov - z["pd_coverage"]) <= tol.max()
    assert np.array_equal(best_est, z["pd_best_est"]) and np.array_equal(best_pl, z["pd_best_pl"])
    assert len(best_est) == 4 and len(best_pl) == 6
    pl2, cov2, _, _ = cr.plausible_diversity(spec, pts, T_est_inv, T_p, bidirectional=True)
    _, tol2 = _reference_bound(spec, T_p, T_est_inv, pts)
    t = max(tol.max(), tol2.max())
    assert abs(pl2 - z["pd2_plausibility"]) <= t and abs(cov2 - z["pd2_coverage"]) <= t
    # the swap matters: one-way and bidirectional differ by far more than the bound
    assert abs(pl2 - pl) > 100 * t or abs(cov2 - cov) > 100 * t


def test_mesh_distance_equals_analytic_box():
    rng = np.random.default_rng(0)
    v, f = cr.box_mesh(0.25)
    q = rng.uniform(-0.6, 0.6, (4000, 3))
    d = cr.mesh_distance(v[f], q)
    ref = np.abs(pr.box_ref([0.25] * 3, q)[0])
    assert np.abs(d - ref).max() < 1e-15


@pytest.mark.parametrize("half", [0.25, 0.5])
def test_exact_box_cloud_premise_on_host(half):
    """The exactness argument of the binned-path test: for a point straight above a face interior of the box mesh,
    the device header's tree walk (bvh_closest, host build) returns a closest point whose coordinate along the face
    normal equals the face's exactly, and the in-face residue is too small to change the fp32 distance, so the
    kernel's d = sqrtf(fmaf(gx, gx, fmaf(gy, gy, gz * gz))) is exactly the dyadic height."""
    import hostsim_lib as hs
    import pytorch_volumetric_b200 as pv
    rng = np.random.default_rng(1)
    v, f = cr.box_mesh(half)
    desc, _keep = hs.mesh_desc(pv.MeshObjectFactory(f"box{half}", mesh=(v, f)))
    q, h = cr.exact_box_cloud(20000, half, [2.0 ** -6, 2.0 ** -5], rng)
    q32 = q.astype(np.float32)
    assert np.array_equal(q32.astype(np.float64), q)
    dist, _grad, closest, _face = hs.mesh_query(desc, q32, mode=0)
    g = closest.astype(np.float32) - q32
    axis = np.argmax(np.abs(q) - half, axis=1)
    rows = np.arange(len(q))
    assert np.array_equal(np.abs(g[rows, axis]).astype(np.float64), h)
    other = np.where(np.arange(3)[None] == axis[:, None], 0.0, g.astype(np.float64))
    # the in-face residue adds less than a quarter ulp of h^2 under the square root
    assert ((other ** 2).sum(1) < 0.25 * U * h ** 2).all()
    assert np.array_equal(np.abs(dist).astype(np.float64), h)
