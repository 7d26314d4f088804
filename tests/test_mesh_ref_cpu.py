"""CPU: the fp64 MeshSDF (tests/mesh_ref.py) pinned to the reference's own vectors and to the host build of the device
code (tests/hostsim: mesh_eval, bvh_parity, bvh_parity_x, bvh_winding), and its stated fp32 bounds checked to cover
the host build's measured error with at most a 10x margin -- the bounds tests/test_gpu_mesh_fp64.py applies to the
kernels."""
import functools

import numpy as np
import pytest

import hostsim_lib as hs
import mesh_ref as mr
import workloads
from helpers import golden, pv_factory

MESHES = ["probe", "wrench", "drill", "scene_overlap"]
N_PER_KIND = {"probe": 1500, "wrench": 1000, "drill": 200, "scene_overlap": 1500}


def _check(rep, bad, where):
    assert all(len(v) == 0 for v in bad.values()), (where, {k: v[:10] for k, v in bad.items() if len(v)}, rep)


@pytest.mark.parametrize("name", ["probe", "wrench", "drill"])
def test_matches_the_reference_vectors(name):
    """closest, distance, gradient and normal of the reference's sdf.py over its restated third-party layer.  The
    reference jitters the ray of an open mesh with unseeded numpy noise, so the wrench's sign may differ where the
    ray grazes the open boundary."""
    z = golden(f"ref_meshsdf_{name}")
    if name == "drill":                       # brute force over 15 728 faces: a quarter of the vectors
        z = {k: (x[::4] if k in ("pts", "closest", "distance", "gradient", "normal") else x) for k, x in z.items()}
    obj = pv_factory(name)
    ref = mr.MeshRef(obj).query(z["pts"])
    if obj.is_closed:
        assert np.array_equal(ref["inside"], z["distance"] < 0)
    else:
        assert ((ref["inside"] != (z["distance"] < 0)) & (ref["dist"] > 1e-6)).mean() <= 2e-3
        ref["sign_margin"] = ref["sign_margin"] | (ref["inside"] != (z["distance"] < 0))
    rep, bad = mr.compare(ref, z["closest"], z["distance"], z["gradient"], z["normal"])
    _check(rep, bad, name)
    assert rep["value"] <= 1 and rep["closest"] <= 1 and rep["grad"] <= 1


CASES = [(name, axis_ray) for name in MESHES for axis_ray in (True, False) if axis_ray or name != "wrench"]


@functools.lru_cache(maxsize=None)
def host_build_case(name, axis_ray):
    """mesh_eval of the host build against the fp64 reference on uniform, near-surface and far points: (factory,
    host descriptor, its keepalive, [(kind, points, MeshRef, geometry, reference, host outputs (dist, grad, closest,
    face), compare report, unexplained rows)]).  Cached so that the per-mesh tests and the tightness check share one measurement, whichever of them runs."""
    obj = pv_factory(name, ray_seed=11)
    obj.axis_ray_when_closed = axis_ray
    ref_obj = mr.MeshRef(obj)
    desc, keep = hs.mesh_desc(obj, with_winding=True)
    v, f = workloads.fixture_mesh(name)
    out = []
    for kind, pts in mr.point_kinds(v, f, N_PER_KIND[name], seed=7).items():
        geo = ref_obj.geometry(pts, winding=True)          # the open mesh's winding number too
        ref = ref_obj.query(pts, geo=geo)
        host = hs.mesh_query(desc, pts)
        excuse = None if axis_ray or not obj.is_closed else (lambda r, pts=pts: ref_obj.ray_grazes(pts[r], r))
        rep, bad = mr.compare(ref, host[2], host[0], host[1], sign_excuse=excuse)
        out.append((kind, pts, ref_obj, geo, ref, host, rep, bad))
    return obj, desc, keep, out


@pytest.mark.parametrize("name,axis_ray", CASES)
def test_matches_the_host_build_of_the_device_code(name, axis_ray):
    """mesh_eval (closest point, face, sign, gradient) on uniform, near-surface and far points: every difference
    within the stated bounds or in a class the reference names, the face index equal off ties, and the crossing
    parity / winding number of the host build equal to the exact ones away from their margins."""
    obj, desc, _, cases = host_build_case(name, axis_ray)
    for kind, pts, ref_obj, geo, ref, (dist, grad, closest, face), rep, bad in cases:
        _check(rep, bad, (name, kind))
        assert np.array_equal(face[~ref["tie_face"]], ref["face"][~ref["tie_face"]])
        # the ray the kernel casts, bit for bit
        idx = np.arange(len(pts))
        dirs = ref_obj.ray_dirs(idx)
        lib = hs.lib()
        for k in (0, 1, 2):
            h = np.array([lib.sim_hash_normal(ref_obj.ray_seed, int(i), k) for i in idx[:64]], np.float32)
            np.testing.assert_array_equal(np.float32(np.float32(1e-4) * h + ref_obj.ray_far[k]), dirs[:64, k])
        px, pr = hs.parity(desc, pts, dirs.astype(np.float32))
        if obj.is_closed:
            exact = (np.rint(ref["w"]).astype(int) & 1)
            assert np.array_equal(px[~ref["sign_margin"]], exact[~ref["sign_margin"]])
            differ = np.nonzero((pr != exact) & ~ref["sign_margin"])[0]
            assert ref_obj.ray_grazes(pts[differ], differ).all(), differ
        else:
            par, _ = ref_obj.ray_parity(pts, idx)
            assert np.array_equal(pr[~ref["sign_margin"]], par[~ref["sign_margin"]])
        w = hs.winding(desc, pts)
        clear = ref["dist"] > mr.C_SIGN * mr.U * ref["scale"]
        assert np.abs(w - ref["w"])[clear].max() < mr.WINDING_MARGIN
        if obj.is_closed:
            wref = ref_obj.query(pts, sign="winding", geo=geo)
            assert np.array_equal((np.abs(w) > 0.5)[~wref["sign_margin"]], wref["inside"][~wref["sign_margin"]])


def test_bounds_are_tight():
    """The bounds cover the host build's error on every mesh and point set, and are at most 10x the largest of it
    (the GPU file would otherwise accept far more than fp32 arithmetic produces).  Measures every case itself."""
    ratios = {}
    for name, axis_ray in CASES:
        for kind, *_, rep, bad in host_build_case(name, axis_ray)[3]:
            _check(rep, bad, (name, kind))
            ratios[(name, kind, axis_ray)] = (rep["value"], rep["closest"], rep["grad"])
    worst = np.max(np.array(list(ratios.values())), axis=0)
    print("error / bound (value, closest, gradient):", worst)
    for k, r in ratios.items():
        print(k, ["%.3f" % x for x in r])
    assert (worst <= 1).all() and (worst >= 0.1).all(), worst
