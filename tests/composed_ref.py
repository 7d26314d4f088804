"""fp64 restatement of the composed query (ComposedSDF.query(..., return_which=True)) over (configuration, point,
sub-SDF), for the CPU and GPU tiers.  Every sub-SDF is evaluated at every pair -- no pruning, no visiting order, no
kernel code -- under fp64 matrices, its gradient is rotated back with the same matrix, and the argmin takes the first
index on ties (torch.argmin, sdf.py:421 of the reference).

A sub-SDF is described by a spec:
  helpers.grid_spec(cached)   nearest-voxel CachedSDF with the bounding-box rule (table lookup + helpers._aabb_rule)
  primitive_spec(desc)        SphereSDF / BoxSDF / CylinderSDF descriptor (tests/primitive_ref.py)
  mesh_spec(port_mesh)        a closed mesh through the oracle's closest point and crossing parity (oracle.port)
  trilinear_spec(cached)      trilinear CachedSDF: the interpolant in range, the bounding-box rule outside it
                              (tests/grid_ref.py)
  grid_gt_spec(cached, mesh)  nearest-voxel CachedSDF with OutOfBoundsStrategy.LOOKUP_GT_SDF: the signed fp64 mesh
                              (tests/mesh_ref.MeshRef) outside the range
Test infrastructure only."""
import numpy as np

import grid_ref
import helpers
import primitive_ref as pr
from helpers import classify_mesh_mismatch, ray_noise


def primitive_spec(desc):
    """Spec of a SPHERE / BOX / CYLINDER descriptor (its fp32 fields, as the kernels read them)."""
    from pytorch_volumetric_b200 import _native as nat
    half = [float(desc.bb_max[k]) for k in range(3)]
    if desc.kind == nat.PVB_KIND_BOX:
        return {"kind": "box", "half": half}
    if desc.kind == nat.PVB_KIND_CYLINDER:
        return {"kind": "cylinder", "radius": float(desc.radius), "half_length": half[2]}
    assert desc.kind == nat.PVB_KIND_SPHERE
    return {"kind": "sphere", "radius": float(desc.radius)}


def mesh_spec(port_mesh, seed=0):
    """Spec of a closed mesh (oracle.port.MeshPort).  The sign of a closed mesh does not depend on the ray direction
    off the surface, so any seeded ray noise stands in for the reference's random draw."""
    return {"kind": "mesh", "port": port_mesh, "seed": seed}


def trilinear_spec(cached):
    return {"kind": "trilinear", "ref": grid_ref.Grid.of(cached)}


def grid_gt_spec(cached, mesh):
    """mesh: the tests/mesh_ref.MeshRef of the CachedSDF's ground-truth mesh (closed: its sign does not depend on the
    point's index in the call)."""
    s = helpers.grid_spec(cached)
    s.update(kind="grid_gt", ref=grid_ref.Grid.of(cached), mesh=mesh)
    return s


def grid_gt_eval(spec, q):
    r = spec["ref"].nearest(q)
    v, g = r["value"].copy(), r["grad"].copy()
    out = ~r["inb"]
    if out.any():
        m = spec["mesh"].query(q[out])
        v[out], g[out] = m["value"], m["grad"]
    return v, g


def grid_eval(spec, q):
    """Nearest voxel inside the cached range [lo, hi] (round half to even, like torch.round), the bounding-box rule
    outside it.  q [n, 3] fp64."""
    lo, hi, val, grad, bb = spec["lo"], spec["hi"], spec["val"], spec["grad"], spec["bb"]
    n = np.array(val.shape)
    res = (hi - lo) / (n - 1)
    inb = np.all((q >= lo) & (q <= hi), axis=1)
    k = np.clip(np.rint((q - lo) / res), 0, n - 1).astype(np.int64)
    v_in, g_in = val[k[:, 0], k[:, 1], k[:, 2]], grad[k[:, 0], k[:, 1], k[:, 2]]
    below = np.maximum(bb[:, 0] - q, 0.0)
    above = np.maximum(q - bb[:, 1], 0.0)
    delta = np.where(below > 0, -below, above)
    dist = np.linalg.norm(delta, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        g_out = np.where(dist[:, None] > 0, delta / dist[:, None], delta)
    return np.where(inb, v_in, dist), np.where(inb[:, None], g_in, g_out)


def mesh_eval(spec, q):
    """The oracle's closest point (fp32 arithmetic, as the reference) and crossing parity."""
    _c, d, g, _n = spec["port"].closest_point(q.astype(np.float32), ray_noise=ray_noise(spec["seed"], len(q)))
    return d.numpy().astype(np.float64), g.numpy().astype(np.float64)


def evaluate(spec, q):
    """(value [n], sub-frame gradient [n, 3]) of one sub-SDF at sub-frame points q [n, 3]."""
    kind = spec["kind"]
    if kind == "grid":
        return grid_eval(spec, q)
    if kind == "mesh":
        return mesh_eval(spec, q)
    if kind == "trilinear":
        r = spec["ref"].trilinear(q)
        return r["value"], r["grad"]
    if kind == "grid_gt":
        return grid_gt_eval(spec, q)
    if kind == "box":
        return pr.box_ref(spec["half"], q)
    if kind == "cylinder":
        return pr.cylinder_ref(spec["radius"], spec["half_length"], q)
    assert kind == "sphere", kind
    return pr.sphere_ref(spec["radius"], q)


def compose(specs, mats, pts, per_sub=False):
    """The composition of `specs` under mats (S, A, 4, 4) object->sub-frame matrices at points (P, 3) shared by every
    configuration, or (A, P, 3) with configuration a at its own points (the paired form).
    Returns (value (A, P), object-frame gradient (A, P, 3), which (A, P)), and with per_sub=True also every sub-SDF's
    value (S, A, P) and object-frame gradient (S, A, P, 3)."""
    mats = np.asarray(mats, dtype=np.float64)
    pts = np.asarray(pts, dtype=np.float64)
    S, A = mats.shape[:2]
    P = pts.shape[-2]
    own = pts.ndim == 3
    best = np.full((A, P), np.inf)
    bgrad = np.zeros((A, P, 3))
    which = np.full((A, P), -1, dtype=np.int64)
    allv, allg = (np.empty((S, A, P)), np.empty((S, A, P, 3))) if per_sub else (None, None)
    for s, spec in enumerate(specs):
        R, t = mats[s, :, :3, :3], mats[s, :, :3, 3]
        q = np.einsum("aij,apj->api" if own else "aij,pj->api", R, pts) + t[:, None, :]
        v, g = evaluate(spec, q.reshape(-1, 3))
        v = v.reshape(A, P)
        g = np.einsum("apj,aji->api", g.reshape(A, P, 3), R)          # g @ R: back to the object frame
        better = (v < best) | (which < 0)                                # strict: the first index keeps its ties
        best = np.where(better, v, best)
        bgrad = np.where(better[..., None], g, bgrad)
        which = np.where(better, s, which)
        if per_sub:
            allv[s], allg[s] = v, g
    return (best, bgrad, which, allv, allg) if per_sub else (best, bgrad, which)


def mesh_mismatch(v, g, w, ref, tol=1e-5, coord_scale=0.1):
    """Compare a composition of closed meshes with compose(..., per_sub=True): values within `tol` everywhere,
    gradients by helpers.classify_mesh_mismatch (the 1e-3 shell and closest-feature ties), and the reported sub-SDF
    an argmin within `tol` (a tie between sub-SDFs may report another one than the fp64 argmin).
    Returns (n_bad_value, n_bad_gradient, n_bad_which, report)."""
    rv, rg, _rw, allv, _allg = ref
    v, g, w = (np.asarray(x) for x in (v, g, w))
    bad_v, bad_g, rep = classify_mesh_mismatch(v.reshape(-1), g.reshape(-1, 3), rv.reshape(-1), rg.reshape(-1, 3),
                                               tol, coord_scale)
    ok_w = (w >= 0) & (w < allv.shape[0])
    wv = np.take_along_axis(allv, np.clip(w, 0, allv.shape[0] - 1)[None], 0)[0]
    bad_w = int((~ok_w | (np.abs(wv - rv) > tol)).sum())
    rep["bad_which"] = bad_w
    return bad_v, bad_g, bad_w, rep
