"""Shared helpers for the parity tests (test infrastructure; may use oracle/)."""
import math
import os

import numpy as np
import torch

import workloads
from oracle import port

GOLDEN = workloads.GOLDEN


def golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def port_mesh(name):
    v, f = workloads.fixture_mesh(name)
    return port.MeshPort(vertices=v, faces=f, name=name)


def pv_factory(name, **kw):
    import pytorch_volumetric_b200 as pv
    v, f = workloads.fixture_mesh(name)
    return pv.MeshObjectFactory(name, mesh=(v, f), **kw)


# ---- host mirror of the kernel's deterministic ray jitter (pvb_device.cuh: mix32 / hash_normal) ----
def _mix32(x):
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16)
    x = (x * np.uint32(0x7feb352d)).astype(np.uint32)
    x ^= x >> np.uint32(15)
    x = (x * np.uint32(0x846ca68b)).astype(np.uint32)
    x ^= x >> np.uint32(16)
    return x


def hash_normal(seed, idx, comp):
    idx = np.asarray(idx, dtype=np.uint64)
    lo = (idx & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (idx >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        a = _mix32(lo * np.uint32(3) + np.uint32(comp) + np.uint32(0x9e3779b9))
        b = _mix32(hi + np.uint32(0x85ebca6b))
        h0 = _mix32(np.uint32(seed) ^ a ^ b)
        h1 = _mix32(h0 + np.uint32(0x6a09e667))
    s = ((h0 & np.uint32(0xffff)).astype(np.float32) + (h0 >> np.uint32(16)).astype(np.float32)
         + (h1 & np.uint32(0xffff)).astype(np.float32) + (h1 >> np.uint32(16)).astype(np.float32))
    return (s - np.float32(131070.0)) * np.float32(2.6428816e-05)


def ray_noise(seed, n):
    idx = np.arange(n, dtype=np.uint64)
    return np.stack([hash_normal(seed, idx, c) for c in range(3)], axis=1).astype(np.float64)


def classify_mesh_mismatch(d_gpu, g_gpu, d_ref, g_ref, tol=1e-5, coord_scale=0.1):
    """Returns (n_bad_value, n_bad_grad_unexplained, report).

    Gradient tolerance: `tol` plus the fp32 conditioning of (closest - p) / |d| -- the closest point carries a
    few ulps of the coordinate magnitude, which the division by a small |d| amplifies.  A remaining exceedance
    is 'explained' when the point sits on the |d| = 1e-3 shell (sdf.py:162) or when the two sides agree on the
    distance but pick different closest features (ties on the medial axis)."""
    dv = np.abs(d_gpu - d_ref)
    bad_v = dv > tol
    dg = np.abs(g_gpu - g_ref).max(axis=-1)
    gtol = tol + 8 * np.finfo(np.float32).eps * coord_scale / np.maximum(np.abs(d_ref), 1e-12)
    bad_g = dg > gtol
    shell = np.abs(np.abs(d_ref) - 1e-3) < 2e-6
    explained = bad_g & (shell | (dv <= tol))     # same distance, different closest feature / shell flip
    unexplained = bad_g & ~explained
    rep = dict(n=len(d_ref), bad_val=int(bad_v.sum()), bad_grad=int(bad_g.sum()), explained=int(explained.sum()),
               max_dval=float(dv.max()), max_dgrad=float(dg.max()))
    return int(bad_v.sum()), int(unexplained.sum()), rep


# ---------------------------------------------------------------------------------------------------------------
# Per-exceedance classification for composed / robot queries (SURVEY 8c): every output that differs from the
# reference by more than the tolerance must be one of
#   (i)   a voxel-boundary flip: the fp32 rigid transform (an FMA chain here, a bmm in the reference) moved the
#         link-frame point across a cell boundary it sits on (|frac - 0.5| < FLIP_BAND cells) or across the edge of
#         the cached range, and the output equals the entry of that neighbouring cell / the other side's rule;
#   (ii)  the |d| = 1e-3 shell of sdf.py:162 or a closest-feature tie (same distance, another gradient) of a mesh;
#   (iii) an argmin tie between sub-SDFs (values within the tolerance, the other one's gradient reported);
#   (iv)  a trilinear cell-face flip: the link-frame point lies within FLIP_BAND cells of an interior cell face of a
#         trilinear grid, and the gradient is that of another cell touching the face (the interpolant is continuous
#         there, its gradient is not).
# Anything else is unexplained and fails the test.
FLIP_BAND = 1.5e-4      # cells; rounding of the S*|A| rigid transforms: ~3 ulp of |q| over the cell size


def grid_spec(cached):
    """What the classifier needs from a pytorch_volumetric_b200.CachedSDF (tables are the ones the kernel reads)."""
    shape = tuple(cached.voxels.shape)
    return {"kind": "grid", "val": cached.voxels.raw_data.detach().cpu().numpy().reshape(shape).astype(np.float64),
            "grad": cached.voxels_grad.detach().cpu().numpy().reshape(*shape, 3).astype(np.float64),
            "lo": np.array([float(min(r)) for r in cached.ranges]), "hi": np.array([float(max(r)) for r in cached.ranges]),
            "bb": cached.bb.detach().cpu().numpy().astype(np.float64)}


def sphere_spec(radius):
    return {"kind": "sphere", "radius": float(radius)}


def _aabb_rule(bb, q):
    below = np.maximum(bb[:, 0] - q, 0.0)
    above = np.maximum(q - bb[:, 1], 0.0)
    delta = np.where(below > 0, -below, above)
    dist = np.linalg.norm(delta)
    return dist, (delta / dist if dist > 0 else delta)


def _primitive_alternatives(spec, q):
    """(value, sub-frame gradient, gradient slack) pairs of a BOX / CYLINDER spec at q (3,): the fp64 result, plus
    the other axis of the inside rule wherever two of its terms are within 1e-5 (fp32 rounding may pick either).  The
    slack is the fp32 conditioning of the outside gradient w / |w| near the surface and of the radial direction near
    a cylinder's axis (tests/test_gpu_primitive.py)."""
    import primitive_ref as pr
    q = np.asarray(q, dtype=np.float64)
    scale = 3e-7 * np.abs(q).max()
    if spec["kind"] == "box":
        v, g = pr.box_ref(spec["half"], q[None])
        v, g = float(v[0]), g[0]
        slack = scale / max(abs(v), 1e-30) if v > -1e-6 else 0.0
        out = [(v, g, slack)]
        if v <= 0:
            e = np.abs(q) - np.asarray(spec["half"])
            for k in np.nonzero(e >= e.max() - 1e-5)[0]:
                gk = np.zeros(3)
                gk[k] = 1.0 if q[k] >= 0 else -1.0
                out.append((v, gk, slack))
        return out
    v, g = pr.cylinder_ref(spec["radius"], spec["half_length"], q[None])
    v, g = float(v[0]), g[0]
    rho = float(np.hypot(q[0], q[1]))
    slack = scale / max(min(abs(v) if v > -1e-6 else np.inf, rho), 1e-30)
    out = [(v, g, slack)]
    dr, dz = rho - spec["radius"], abs(q[2]) - spec["half_length"]
    if v <= 0 and abs(dr - dz) < 1e-5:
        ux, uy = (q[0] / rho, q[1] / rho) if rho > 0 else (1.0, 0.0)
        out += [(v, np.array([ux, uy, 0.0]), slack), (v, np.array([0.0, 0.0, 1.0 if q[2] >= 0 else -1.0]), slack)]
    return out


def flip_candidates(specs, M, p):
    """All (value, object-frame gradient, sub-SDF, gradient slack) the reference's rules can produce for point p (3,)
    under the object->sub-frame matrices M (S,4,4, fp64) when every link-frame coordinate within FLIP_BAND of a cell
    boundary (or 1e-6 m of the range edge) is allowed to fall on either side, and a primitive's inside rule may pick
    either of two near-equal axes.  The slack is added to the gradient tolerance of that candidate."""
    out = []
    for s, spec in enumerate(specs):
        R, t = M[s, :3, :3], M[s, :3, 3]
        q = R @ p + t
        if spec["kind"] == "sphere":
            r = np.linalg.norm(q)
            out.append((r - spec["radius"], (q / (r + 1e-12)) @ R, s, 0.0))
            continue
        if spec["kind"] in ("box", "cylinder"):
            out += [(v, g @ R, s, slack) for v, g, slack in _primitive_alternatives(spec, q)]
            continue
        if spec["kind"] == "trilinear":
            out += _trilinear_alternatives(spec["ref"], q, R, s)
            continue
        lo, hi, val, grad = spec["lo"], spec["hi"], spec["val"], spec["grad"]
        n = np.array(val.shape)
        res = (hi - lo) / (n - 1)
        edge = 1e-6
        maybe_in = np.all((q >= lo - edge) & (q <= hi + edge))
        maybe_out = np.any((q < lo + edge) | (q > hi - edge))
        if maybe_in:
            u = (q - lo) / res
            opts = []
            for a in range(3):
                k = int(np.clip(np.rint(u[a]), 0, n[a] - 1))
                o = {k}
                f = u[a] - np.floor(u[a])
                if abs(f - 0.5) < FLIP_BAND:
                    o.update({int(np.clip(np.floor(u[a]), 0, n[a] - 1)), int(np.clip(np.floor(u[a]) + 1, 0, n[a] - 1))})
                opts.append(sorted(o))
            for kx in opts[0]:
                for ky in opts[1]:
                    for kz in opts[2]:
                        out.append((val[kx, ky, kz], grad[kx, ky, kz] @ R, s, 0.0))
        if maybe_out and spec["kind"] == "grid_gt":
            m = spec["mesh"].query(q[None])
            tie = bool(m["tie_face"][0] | m["tie_normal"][0] | m["shell_edge"][0] | m["sign_margin"][0])
            slack = 2.0 if tie else float(mesh_grad_bound(m["scale"], m["cond"])[0])
            out.append((float(m["value"][0]), m["grad"][0] @ R, s, slack))
        elif maybe_out:
            d, g = _aabb_rule(spec["bb"], q)
            out.append((d, g @ R, s, 0.0))
    return out


def mesh_grad_bound(scale, cond):
    import mesh_ref
    return mesh_ref.grad_bound(scale, cond)


def _trilinear_alternatives(ref, q, R, s):
    """Candidates of a trilinear grid (tests/grid_ref.Grid) at q (3,): the interpolant with the gradient of every cell
    touching a cell face within FLIP_BAND of q, and the bounding-box rule near the range's edge.  The slack is the
    gradient bound of grid_ref."""
    import grid_ref
    out = []
    r = ref.trilinear(q[None], band=FLIP_BAND)
    if r["inb"][0] or np.all((q >= ref.lo - 1e-6) & (q <= ref.hi + 1e-6)):
        qc = np.clip(q, ref.lo64, ref.hi64)
        rc = ref.trilinear(qc[None], band=FLIP_BAND) if not r["inb"][0] else r
        slack = float(rc["gbound"][0].max())
        v = float(rc["value"][0])
        out.append((v, rc["grad"][0] @ R, s, slack))
        for g in rc["alt"][:, 0]:
            if np.isfinite(g).all():
                out.append((v, g @ R, s, slack))
    if not r["inb"][0] or np.any((q < ref.lo + 1e-6) | (q > ref.hi - 1e-6)):
        d, g = grid_ref.box_rule(ref.bb32, q[None])
        out.append((float(d[0]), g[0] @ R, s, 0.0))
    return out


def classify_composed(v_gpu, g_gpu, v_ref, g_ref, specs, mats, pts, tol=1e-5):
    """v_*: (A, P) values, g_*: (A, P, 3); mats: (S, A, 4, 4) object->sub-frame; pts (P, 3).
    Returns (n_exceed, n_unexplained, report).  An exceedance is explained when the GPU output equals, within `tol`,
    one of the legitimate alternatives of flip_candidates AND is a possible minimum over the sub-SDFs (between the
    min over sub-SDFs of their smallest and of their largest alternative)."""
    v_gpu = np.asarray(v_gpu, dtype=np.float64); g_gpu = np.asarray(g_gpu, dtype=np.float64)
    bad = (np.abs(v_gpu - v_ref) > tol) | (np.abs(g_gpu - g_ref).max(-1) > tol)
    idx = np.argwhere(bad)
    mats = np.asarray(mats, dtype=np.float64)
    pts = np.asarray(pts, dtype=np.float64)
    unexplained = []
    for a, i in idx:
        cands = flip_candidates(specs, mats[:, a], pts[i])
        # a valid output is min over sub-SDFs of ONE alternative each: it lies between the two extreme choices
        per_s = {}
        for cv, _cg, s_, _sl in cands:
            lo_hi = per_s.setdefault(s_, [cv, cv])
            lo_hi[0], lo_hi[1] = min(lo_hi[0], cv), max(lo_hi[1], cv)
        lower = min(v[0] for v in per_s.values())
        upper = min(v[1] for v in per_s.values())
        ok = False
        if lower - tol <= v_gpu[a, i] <= upper + tol:
            for cv, cg, _s, slack in cands:
                if abs(cv - v_gpu[a, i]) <= tol and np.abs(cg - g_gpu[a, i]).max() <= tol + slack:
                    ok = True
                    break
        if not ok:
            unexplained.append((int(a), int(i), float(v_gpu[a, i]), float(v_ref[a, i])))
    rep = {"n": int(bad.size), "exceed": int(len(idx)), "unexplained": len(unexplained), "first": unexplained[:5]}
    return len(idx), len(unexplained), rep


# ---------------------------------------------------------------------------------------------------------------
# GPU-tier compositions the query-form tests share: CachedSDF links from the golden tables, the golden and arm sets,
# route guards and the per-configuration reductions the fused queries are checked against.
def cached_from_golden(z, name, tmp_path, table_key="table_val", grad_key="table_grad", range_in=None, **kw):
    """Write the reference-built tables into a reference-format cache file and let CachedSDF load them
    (sdf.py:487-495): exercises on-disk cache compatibility and isolates the lookup from the table build."""
    import pytorch_volumetric_b200 as pv
    res = float(z["resolution"])
    range_in = z["range_in"] if range_in is None else range_in
    ranges = pv.get_divisible_range_by_resolution(res, range_in)
    key = f"{name} {res} {tuple(ranges)}"
    shape = [int(s) for s in z["table_shape"]]
    cache = {key: (torch.from_numpy(z[table_key]).reshape(shape), torch.from_numpy(z[grad_key]))}
    path = str(tmp_path / f"sdf_cache_{name}.pkl")
    torch.save(cache, path)
    gt = pv.MeshSDF(pv_factory(name.rstrip("32")))
    return pv.CachedSDF(name, res, range_in, gt, device="cuda", cache_path=path, **kw)


def golden_sets(tmp_path):
    import pytorch_volumetric_b200 as pv
    zc = golden("ref_cachedsdf_probe")
    near = cached_from_golden(zc, "probe", tmp_path)
    tri = cached_from_golden(zc, "probe", tmp_path, interpolation="trilinear")
    z = golden("ref_composed")
    sph = pv.SphereSDF(float(z["sphere_radius"]))
    return z, {"nearest": [near, near, near, near], "trilinear": [tri, tri, tri], "mixed": [near, tri, near],
               "nearest+sphere": [near, near, sph, near], "mixed+sphere": [tri, near, sph, tri]}


def no_generic(monkeypatch, comp):
    def boom(*a, **k):
        raise AssertionError("generic path taken")
    monkeypatch.setattr(comp, "_generic_query", boom)


def opaque_sdfs(pv, sdfs):
    class Opaque(pv.ObjectFrameSDF):          # no native descriptor -> generic path
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, p):
            return self.inner(p)

        def surface_bounding_box(self, **kw):
            return self.inner.surface_bounding_box(**kw)

    return [Opaque(s) for s in sdfs]


def cached_arm(tmp_path, interpolation):
    """The arm of workloads.write_arm with CachedSDF links of the given interpolation."""
    import pytorch_volumetric_b200 as pv
    urdf, end = workloads.write_arm(str(tmp_path))
    chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
    return pv.RobotSDF(chain, path_prefix=str(tmp_path),
                       link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                              cache_path=str(tmp_path / "arm.pkl"),
                                                              interpolation=interpolation))


def arm_robot(tmp_path, kind):
    """cached_arm for kind "nearest" / "trilinear", the primitive arm of workloads.write_primitive_arm otherwise."""
    import pytorch_volumetric_b200 as pv
    if kind == "primitive":
        urdf, end = workloads.write_primitive_arm(str(tmp_path / "prim"))
        return pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"),
                           primitive_visuals=True)
    return cached_arm(tmp_path, kind)


def arm_points(n, seed):
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    return workloads.uniform_points(n, lo, hi, seed=seed).cuda()


def own_points(q, A, seed):
    """[A, P, 3] on the GPU: the points q, shuffled and shifted differently for every configuration."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = q.cpu()
    return torch.stack([q[torch.randperm(len(q), generator=g)] + 0.01 * torch.randn(3, generator=g)
                        for _ in range(A)]).cuda()


def swept_reduce(v, g, w, cfg_count, cfg_begin=0):
    """Lexicographic (value, configuration, sub-SDF) minimum of flat per-configuration results [cfg_count * P]."""
    P = v.numel() // cfg_count
    v, g, w = v.reshape(cfg_count, P), g.reshape(cfg_count, P, 3), w.reshape(cfg_count, P)
    c = (v == v.amin(dim=0)).int().argmax(dim=0)          # the first configuration attaining the minimum
    return (v.gather(0, c[None])[0], g.gather(0, c[None, :, None].expand(1, P, 3))[0],
            (c + cfg_begin).to(torch.int32), w.gather(0, c[None])[0])


def clearance_reduce(v, g, w, cfg_count, n_seg):
    """First point attaining the minimum of every (configuration, segment) of flat results [cfg_count * n_seg * N]."""
    v = v.reshape(cfg_count, n_seg, -1)
    N = v.shape[-1]
    g, w = g.reshape(cfg_count, n_seg, N, 3), w.reshape(cfg_count, n_seg, N)
    i = (v == v.amin(-1, keepdim=True)).int().argmax(-1, keepdim=True)
    return (v.gather(-1, i).reshape(-1), g.gather(-2, i[..., None].expand(-1, -1, 1, 3)).reshape(-1, 3),
            i.reshape(-1).to(torch.int32), w.gather(-1, i).reshape(-1))


def _which_values(specs, tm, pts, w):
    """fp64 value of the reported sub-SDF w (A, P) at every pair."""
    import composed_ref as cr
    out = np.full(w.shape, np.nan)
    for s, spec in enumerate(specs):
        a, i = np.nonzero(w == s)
        if len(a):
            q = np.einsum("nij,nj->ni", tm[s, a, :3, :3], pts[i].astype(np.float64)) + tm[s, a, :3, 3]
            out[a, i] = cr.evaluate(spec, q)[0]
    return out


def assert_fp64(members, tm, pts, v, g, w, what, tol=1e-5):
    """query(..., return_which=True) against the fp64 composition: grids and primitives through
    classify_composed (every exceedance a classified flip or tie), meshes through composed_ref.mesh_mismatch;
    `which` names a sub-SDF whose fp64 value is the result's within the tolerance.  Returns the exceedance mask."""
    import composed_ref as cr
    S, A = tm.shape[:2]
    P = len(pts)
    v, g, w = (t.cpu().numpy() for t in (v, g, w))
    v, g, w = v.reshape(A, P), g.reshape(A, P, 3), w.reshape(A, P)
    specs = [m[1] for m in members]
    assert ((w >= 0) & (w < S)).all(), what
    if specs[0]["kind"] == "mesh":
        ref = cr.compose(specs, tm, pts, per_sub=True)
        bad_v, bad_g, bad_w, rep = cr.mesh_mismatch(v, g, w, ref, tol, coord_scale=0.2)
        assert bad_v == 0 and bad_g == 0 and bad_w == 0, (what, rep)
        return np.zeros((A, P), bool)
    rv, rg, _rw = cr.compose(specs, tm, pts)
    n_ex, n_un, rep = classify_composed(v, g, rv, rg, specs, tm, pts, tol)
    assert n_un == 0, (what, rep)
    assert n_ex <= 2e-3 * A * P, (what, rep)
    exceed = (np.abs(v - rv) > tol) | (np.abs(g - rg).max(-1) > tol)
    assert ((np.abs(_which_values(specs, tm, pts, w) - rv) <= tol) | exceed).all(), what
    return exceed


# ---- self-clearance inputs
def wide_configurations(A, seed, dtype=torch.float32):
    """Joint values uniform in +-pi: wide enough that the arm's links pass through one another."""
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(A, 7, generator=g, dtype=torch.float64) * 2 - 1) * math.pi).to(dtype)


def allowed_matrix(S, kind):
    """[S, S] bool: links at least two apart ("default"), an asymmetric pattern, or nothing."""
    i = torch.arange(S)
    if kind == "default":
        return (i[:, None] - i[None, :]).abs() >= 2
    if kind == "asymmetric":
        return (i[None, :] - i[:, None] >= 3) | ((i[:, None] == S - 1) & (i[None, :] == 0))
    return torch.zeros(S, S, dtype=torch.bool)


def surface_points(link_sdf, n, seed):
    from pytorch_volumetric_b200.model_to_sdf import _primitive_surface
    return _primitive_surface(link_sdf, n, np.random.default_rng(seed))


# ---- the reference project's offset wrench robot
WRENCH_URDF = """<robot name="wrench">
{links}
  <link name="offset_wrench"><visual><geometry><mesh filename="wrench.obj"/></geometry></visual></link>
{joints}
</robot>"""


def write_wrench_urdf(dirname):
    """Procedural equivalent of the reference's tests/offset_wrench.urdf: 3 prismatic + 3 revolute joints
    (x, y, z each) in front of one mesh link."""
    from pytorch_volumetric_b200.meshio import write_obj
    v, f = workloads.fixture_mesh("wrench")
    write_obj(os.path.join(dirname, "wrench.obj"), v, f)
    names = ["link_x_trans", "link_y_trans", "link_z_trans", "link_x_rot", "link_y_rot", "link_z_rot", "offset_wrench"]
    links = "\n".join(f'  <link name="{n}"/>' for n in names[:-1])
    axes = ["1 0 0", "0 1 0", "0 0 1"] * 2
    jn = ["x_trans", "y_trans", "z_trans", "x_rot", "y_rot", "z_rot"]
    joints = "\n".join(
        f'  <joint name="{jn[i]}" type="{"prismatic" if i < 3 else "revolute"}"><origin rpy="0 0 0" xyz="0 0 0"/>'
        f'<parent link="{names[i]}"/><child link="{names[i + 1]}"/><axis xyz="{axes[i]}"/></joint>' for i in range(6))
    path = os.path.join(dirname, "offset_wrench.urdf")
    with open(path, "w") as fh:
        fh.write(WRENCH_URDF.format(links=links, joints=joints))
    return path
