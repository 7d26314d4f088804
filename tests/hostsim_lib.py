"""ctypes front end of tests/hostsim: the DEVICE header pvb_device.cuh compiled for the host (g++, see
tests/hostsim/cuda_runtime.h), so the per-thread arithmetic of the kernels can be checked in the CPU tier.  Every
tests/hostsim/*.cpp goes into one library, lib().  Below the simulators every query form uses, the descriptor sets and
inputs the CPU-tier test modules share.
Test infrastructure only; descriptors carry host pointers (numpy / CPU torch memory)."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import torch

from helpers import golden
from pytorch_volumetric_b200 import _native as nat

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = os.path.join(_HERE, "_build", "libpvb_hostsim.so")
_lib = None


def lib():
    """Every tests/hostsim/*.cpp in one library, rebuilt when any host source, the device header or pvb.h is newer."""
    global _lib
    if _lib is None:
        units = sorted(glob.glob(os.path.join(_HERE, "*.cpp")))
        sources = units + glob.glob(os.path.join(_HERE, "*.h")) + [
            os.path.join(_ROOT, "pytorch_volumetric_b200", "csrc", "pvb_device.cuh"),
            os.path.join(_ROOT, "include", "pvb.h")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in sources):
            os.makedirs(os.path.dirname(_LIB), exist_ok=True)
            # -ffp-contract=off: every fp32 operation rounds once, like the *_rn intrinsics the header relies on
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                            "-I", _HERE, *units, "-o", _LIB], check=True)
        _lib = ctypes.CDLL(_LIB)
        for name, restype, argtypes in (
                ("sim_hash_normal", ctypes.c_float, [ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32]),
                ("simcc_chunk", ctypes.c_longlong, [ctypes.c_longlong]),
                ("simcc_chunks", ctypes.c_longlong, [ctypes.c_longlong]),
                ("simrs_visit_margin", ctypes.c_float, None),
                ("simscl_key", ctypes.c_uint64, [ctypes.c_float, ctypes.c_int, ctypes.c_int])):
            getattr(_lib, name).restype = restype
            if argtypes is not None:
                getattr(_lib, name).argtypes = argtypes
    return _lib


def _p(a):
    """The data pointer of a numpy array; None stays a null pointer."""
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _pts(points):
    return np.ascontiguousarray(points.detach().cpu().numpy() if torch.is_tensor(points) else points, dtype=np.float32)


def grid_lookup(desc, points, branchy=False):
    p = _pts(points); n = len(p)
    val, grad, key = np.empty(n, np.float32), np.empty((n, 3), np.float32), np.empty(n, np.int64)
    if branchy:
        lib().sim_grid_lookup_branchy(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(val), _p(grad))
        return val, grad
    lib().sim_grid_lookup(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(val), _p(grad), _p(key))
    return val, grad, key


def grid_trilinear(desc, points):
    """(val, grad) of grid_trilinear_eval per query: the per-thread work of grid_trilinear_kernel."""
    p = _pts(points); n = len(p)
    val, grad = np.empty(n, np.float32), np.empty((n, 3), np.float32)
    lib().simtri_grid_trilinear(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(val), _p(grad))
    return val, grad


def mesh_query(desc, points, mode=nat.PVB_MESH_DEFAULT, stats=False):
    """(dist, grad, closest, face) and, with stats=True, a dict of traversal counts per query."""
    p = _pts(points); n = len(p)
    dist, grad = np.empty(n, np.float32), np.empty((n, 3), np.float32)
    closest, face = np.empty((n, 3), np.float32), np.empty(n, np.int32)
    st = np.zeros(4, np.int64)
    lib().sim_mesh_query(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), ctypes.c_uint32(mode), _p(dist), _p(grad),
                         _p(closest), _p(face), _p(st))
    if stats:
        names = ("closest_nodes", "closest_tris", "parity_nodes", "parity_tris")
        return dist, grad, closest, face, {k: float(v) / max(n, 1) for k, v in zip(names, st)}
    return dist, grad, closest, face


def parity(desc, points, dirs=None):
    p = _pts(points); n = len(p)
    px = np.empty(n, np.int32)
    pr = np.empty(n, np.int32) if dirs is not None else None
    d = _pts(dirs) if dirs is not None else None
    lib().sim_parity(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(d), _p(px), _p(pr))
    return px, pr


def winding(desc, points):
    p = _pts(points); n = len(p)
    w = np.empty(n, np.float32)
    lib().sim_winding(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(w))
    return w


def bit_reversed_order(n):
    """The visiting order the composed kernels use (pvb_kernels.cu fill_order)."""
    bits = max(0, (n - 1).bit_length())
    out = []
    for i in range(1 << bits):
        r = int(format(i, f"0{bits}b")[::-1], 2) if bits else 0
        if r < n:
            out.append(r)
    return out


def composed(descs, xforms, n_cfg, points, order=None, mesh_mode=nat.PVB_MESH_DEFAULT, mesh=True, ext=False):
    """(val [n_cfg*P], grad [n_cfg*P,3], which [n_cfg*P]) of the composition of `descs` under xforms
    [(S*n_cfg),4,4] (sub-SDF-major), visiting the sub-SDFs in `order` (default: the kernels' bit-reversed order),
    through composed_consider<kMesh = mesh, kExt = ext>."""
    p = _pts(points); n = len(p); S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms.detach().cpu().numpy() if torch.is_tensor(xforms) else xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4)
    order = bit_reversed_order(S) if order is None else list(order)
    assert sorted(order) == list(range(S))
    od = np.asarray(order, dtype=np.uint8)
    val, grad = np.empty(n_cfg * n, np.float32), np.empty((n_cfg * n, 3), np.float32)
    which = np.empty(n_cfg * n, np.int32)
    lib().sim_composed(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), _p(p), ctypes.c_longlong(n),
                       ctypes.c_uint32(mesh_mode), ctypes.c_int(mesh), ctypes.c_int(ext), _p(val), _p(grad), _p(which))
    return val, grad, which


def sphere_desc(radius):
    import pytorch_volumetric_b200 as pv
    return pv.SphereSDF(radius).native_desc("cpu")      # the product's own descriptor; no device memory involved


def sphere(radius, points):
    p = _pts(points); n = len(p)
    val, grad = np.empty(n, np.float32), np.empty((n, 3), np.float32)
    lib().sim_sphere(ctypes.c_float(radius), _p(p), ctypes.c_longlong(n), _p(val), _p(grad))
    return val, grad


# ---------------------------------------------------------------- descriptors over host memory
def mesh_desc(obj, with_winding=False):
    """pvb_sdf_desc (MESH) of a MeshObjectFactory with the BVH / triangles / normals in host memory, filled by the
    product's own `_fill_mesh_part`.  Returns (desc, keepalive)."""
    from pytorch_volumetric_b200.sdf import _winding_moments
    nodes, tris, _ = obj._bvh_host
    st = {"nodes": torch.from_numpy(np.ascontiguousarray(nodes)), "tris": torch.from_numpy(np.ascontiguousarray(tris)),
          "fn32": torch.from_numpy(obj._face_normals.astype(np.float32)).contiguous()}
    d = nat.SdfDesc()
    d.kind = nat.PVB_KIND_MESH
    d.flags = 0
    obj._fill_mesh_part(d, st)
    if with_winding:
        st["wn"] = torch.from_numpy(np.ascontiguousarray(_winding_moments(nodes, tris)))
        d.wn_nodes = st["wn"].data_ptr()
    return d, st


def grid_desc(table_val, table_grad, ranges, bb, strategy=None, gt_obj=None, interpolation="nearest"):
    """pvb_sdf_desc (GRID) built by the product's CachedSDF._make_desc over CPU tensors.  Returns (desc, keepalive)."""
    from pytorch_volumetric_b200 import sdf as S
    from pytorch_volumetric_b200.voxel import GridView
    c = object.__new__(S.CachedSDF)
    c.ranges = ranges
    c.voxels = GridView(table_val, ranges, invalid_value=None)
    c.voxels_grad = table_grad
    c._table = torch.cat([table_val.reshape(-1, 1), table_grad], 1).contiguous()
    c.bb = torch.as_tensor(np.asarray(bb))
    c._cdev = torch.device("cpu")
    c.out_of_bounds_strategy = S.OutOfBoundsStrategy.BOUNDING_BOX
    c.interpolation = interpolation
    d = c._make_desc()
    keep = [c]
    if strategy == S.OutOfBoundsStrategy.LOOKUP_GT_SDF:      # what _make_desc does when the ground truth is native
        bbf = np.asarray(bb, dtype=np.float32)
        md, st = mesh_desc(gt_obj)
        keep.append(st)
        gt_obj._fill_mesh_part(d, st)
        d.flags = (d.flags | nat.PVB_GRID_OOB_GT | (md.flags & nat.PVB_MESH_CLOSED)) & ~nat.PVB_GRID_PRUNE_OK
        for k in range(3):
            d.bb_min[k] = float(bbf[k, 0]); d.bb_max[k] = float(bbf[k, 1])
    return d, keep


# ---------------------------------------------------------------- descriptor sets the CPU-tier query forms share
def unpruned(descs):
    """Copies of `descs` without PVB_GRID_PRUNE_OK: every pruning bound is -inf."""
    out = []
    for d in descs:
        c = d.copy()
        c.flags &= ~nat.PVB_GRID_PRUNE_OK
        out.append(c)
    return out


def margin_max(descs):
    return max([0.0] + [float(d.prune_margin) for d in descs])


def table_descs(name):
    """(nearest, trilinear, keepalive): GRID descriptors over the golden ref_cachedsdf_<name> tables."""
    z = golden(f"ref_cachedsdf_{name}")
    shape = tuple(int(s) for s in z["table_shape"])
    args = (torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"]),
            [tuple(r) for r in z["ranges"]], z["bb"])
    near, k1 = grid_desc(*args, interpolation="nearest")
    tri, k2 = grid_desc(*args, interpolation="trilinear")
    return near, tri, (k1, k2)


def sets():
    """(golden composition, [(name, descriptors)], keepalive): nearest, trilinear, mixed and drill grid sets with the
    golden sphere."""
    zc = golden("ref_composed")
    sph = sphere_desc(float(zc["sphere_radius"]))
    pn, pt, k1 = table_descs("probe")
    dn, dt, k2 = table_descs("drill")
    return zc, [("nearest", [pn, pn, sph, pn]), ("trilinear", [pt, pt, sph, pt]), ("mixed", [pn, pt, sph, dt]),
                ("drill", [dn, dt, dn, sph])], (k1, k2)


def all_sets():
    """sets() plus a primitive set and a primitive+grid set."""
    import pytorch_volumetric_b200 as pv
    zc, grid_sets, keep = sets()
    _, tri_probe, keep2 = table_descs("probe")
    prim = [pv.BoxSDF([0.05, 0.03, 0.04]).native_desc("cpu"), pv.CylinderSDF(0.015, 0.06).native_desc("cpu"),
            pv.SphereSDF(0.02).native_desc("cpu"), pv.BoxSDF([0.02, 0.02, 0.08]).native_desc("cpu")]
    mixed = [prim[0], grid_sets[0][1][0], prim[1], tri_probe]
    return zc, grid_sets + [("primitive", prim), ("primitive+grid", mixed)], (keep, keep2)


def trajectory(tmat, S, A0, A, seed):
    """[S * A, 4, 4]: A configurations, configuration a the golden configuration a % A0 moved by a small rigid motion
    of the object frame (a robot-like sweep: the same motion for every sub-SDF of a configuration)."""
    g = np.random.default_rng(seed)
    m = np.asarray(tmat, dtype=np.float64).reshape(S, A0, 4, 4)
    out = np.empty((S, A, 4, 4))
    for a in range(A):
        w = g.normal(0.0, 0.15, 3)
        th = np.linalg.norm(w)
        k = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / max(th, 1e-12)
        T = np.eye(4)
        T[:3, :3] = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)
        T[:3, 3] = g.normal(0.0, 0.01, 3)
        out[:, a] = m[:, a % A0] @ T
    return out.reshape(S * A, 4, 4).astype(np.float32)


def own_points(q, A, seed):
    """[A, P, 3]: the golden points, shuffled and shifted differently for every configuration."""
    g = np.random.default_rng(seed)
    q = np.asarray(q, dtype=np.float32)
    return np.stack([q[g.permutation(len(q))] + g.normal(0.0, 0.01, 3).astype(np.float32) for _ in range(A)])


# ---------------------------------------------------------------- simulators several query forms build on
def sim_paired(descs, xforms, n_cfg, points, cfg_begin=0, order=None, nearest_first=1):
    """(val, grad, which) of configurations cfg_begin.. at their own points [cfg_count, P, 3]."""
    p = np.ascontiguousarray(points, dtype=np.float32)
    cfg_count, P = p.shape[0], p.shape[1]
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4)
    order = bit_reversed_order(S) if order is None else list(order)
    od = np.asarray(order, dtype=np.uint8)
    n = cfg_count * P
    val, grad, which = np.empty(n, np.float32), np.empty((n, 3), np.float32), np.empty(n, np.int32)
    lib().simpair_composed(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                           ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(P), ctypes.c_int(nearest_first),
                           ctypes.c_float(margin_max(descs)), _p(val), _p(grad), _p(which))
    return val, grad, which


def pcl_keys(descs, xforms, n_cfg, own, cfg_begin=0, chunk=None, lanes=32, share=1, unit_order=0, shuffle_seed=0,
             seeded=1, first=-1, steps_reversed=0):
    """Paired clearance: (keys [cfg_count * n_seg], lookups) of robot_paired_clearance_kernel's sequence; own
    [cfg_count, n_seg, L, 3]."""
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4) and S <= 8
    keys = np.empty(cfg_count * n_seg, np.uint64)
    evals = ctypes.c_longlong(0)
    lib().simpcl_fused(arr, ctypes.c_int(S), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                       ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                       ctypes.c_int(chunk or L), ctypes.c_int(lanes), ctypes.c_int(share),
                       ctypes.c_int(unit_order), ctypes.c_int(shuffle_seed), ctypes.c_int(seeded),
                       ctypes.c_int(first), ctypes.c_int(steps_reversed), _p(keys), ctypes.byref(evals))
    return keys, evals.value


def pcl_finish(descs, xforms, n_cfg, own, keys, cfg_begin=0, mesh=0):
    """Paired clearance: (val, grad, point, which) of paired_clearance_finish_kernel for the keys of pcl_keys."""
    cfg_count, n_seg, L = own.shape[:3]
    p = np.ascontiguousarray(own, dtype=np.float32)
    S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    od = np.asarray(bit_reversed_order(S), dtype=np.uint8)
    R = len(keys)
    out = np.empty(R, np.float32), np.empty((R, 3), np.float32), np.empty(R, np.int32), np.empty(R, np.int32)
    lib().simpcl_finish(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), ctypes.c_int(cfg_begin),
                        ctypes.c_int(cfg_count), _p(p), ctypes.c_longlong(n_seg), ctypes.c_int(L),
                        ctypes.c_int(mesh), ctypes.c_float(margin_max(descs)), _p(np.ascontiguousarray(keys)),
                        *[_p(a) for a in out])
    return out


# ---------------------------------------------------------------- self-clearance inputs
def masks(allowed):
    """The kernels' per-source bit masks of an [S][S] allowed matrix (the diagonal never set)."""
    S = len(allowed)
    return np.array([sum(1 << j for j in range(S) if allowed[i][j] and j != i) for i in range(S)], dtype=np.uint8)


def inverse(xforms):
    """W = M^-1 in fp64, rounded to fp32 (any fp32 matrix serves: both routes read the same W)."""
    return np.linalg.inv(np.asarray(xforms, dtype=np.float64)).astype(np.float32)


def link_points(zc, tm, S, n_cfg, K, seed):
    """[S, K, 3] fp32: golden query points near the object, carried into every sub-SDF's frame by configuration 0's
    transform -- posed by another configuration they land near the other sub-SDFs."""
    g = np.random.default_rng(seed)
    q = np.asarray(zc["q"], dtype=np.float64)
    m = np.asarray(tm, dtype=np.float64).reshape(S, n_cfg, 4, 4)[:, 0]
    out = np.empty((S, K, 3))
    for i in range(S):
        pts = q[g.choice(len(q), K, replace=K > len(q))] + g.normal(0.0, 0.01, 3)
        out[i] = pts @ m[i, :3, :3].T + m[i, :3, 3]
    return out.astype(np.float32)


def allowed_cases(S):
    full = [[i != j for j in range(S)] for i in range(S)]
    asym = [[j > i for j in range(S)] for i in range(S)]                        # upper triangle only
    row0 = [[i != j and i != 1 for j in range(S)] for i in range(S)]            # row 1 empty
    sparse = [[False] * S for _ in range(S)]
    sparse[S - 1][0] = True
    return {"full": full, "asymmetric": asym, "empty row": row0, "one pair": sparse,
            "empty": [[False] * S for _ in range(S)]}
