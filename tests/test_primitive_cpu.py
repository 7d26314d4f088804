"""CPU tier for analytic URDF primitives (BoxSDF, CylinderSDF, SphereSDF links) in the fused composed kernels.

1. The device arithmetic (pvb_device.cuh compiled for the host by tests/hostsim/hostsim_primitive.cpp): box_eval,
   cylinder_eval and primitive_eval against the fp64 restatements of tests/primitive_ref.py, with the tie rules.
2. The bound contract the kernels' pruning relies on: value >= dist(q, bb) - prune_margin, with dist(q, bb) as the
   kernels compute it, and the serial robot kernel's sphere bound with primitive descriptors.
3. composed_consider with the extension flag over a mixed set (golden probe table, nearest and trilinear, with box,
   cylinder and sphere): independent of pruning and visiting order, and equal to an fp64 composition.
4. The C ABI refusals of unknown kinds, and the Python construction of primitive links from a URDF."""
import ctypes
import logging
import os
import subprocess

import numpy as np
import pytest
import torch

import hostsim_lib as hs
import primitive_ref as pr
from helpers import golden
from oracle import port
from pytorch_volumetric_b200 import _native as nat

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_primitive.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_primitive.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_primitive.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
                   os.path.join(root, "pytorch_volumetric_b200", "csrc", "pvb_device.cuh"),
                   os.path.join(root, "include", "pvb.h")]
        if not os.path.exists(_SIM_LIB) or any(os.path.getmtime(f) > os.path.getmtime(_SIM_LIB) for f in sources):
            os.makedirs(os.path.dirname(_SIM_LIB), exist_ok=True)
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                            "-I", _SIM_DIR, sources[0], "-o", _SIM_LIB], check=True)
        _sim = ctypes.CDLL(_SIM_LIB)
    return _sim


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _sim_eval(desc, points, fn=2):
    p = np.ascontiguousarray(points, dtype=np.float32); n = len(p)
    val, grad = np.empty(n, np.float32), np.empty((n, 3), np.float32)
    _simlib().simprim_eval(ctypes.byref(desc), ctypes.c_int(fn), _p(p), ctypes.c_longlong(n), _p(val), _p(grad))
    return val, grad


def _sim_lb2(desc, points):
    p = np.ascontiguousarray(points, dtype=np.float32); n = len(p)
    lb2 = np.empty(n, np.float32)
    _simlib().simprim_aabb_lb2(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(lb2))
    return lb2


def _sim_composed(descs, xforms, n_cfg, points, order=None):
    p = np.ascontiguousarray(points, dtype=np.float32); n = len(p); S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4)
    order = hs.bit_reversed_order(S) if order is None else list(order)
    assert sorted(order) == list(range(S))
    od = np.asarray(order, dtype=np.uint8)
    val, grad = np.empty(n_cfg * n, np.float32), np.empty((n_cfg * n, 3), np.float32)
    which = np.empty(n_cfg * n, np.int32)
    _simlib().simprim_composed(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), _p(p), ctypes.c_longlong(n),
                               _p(val), _p(grad), _p(which))
    return val, grad, which


def _prims():
    import pytorch_volumetric_b200 as pv
    return [("box", pv.BoxSDF([0.24, 0.1, 0.15]).native_desc("cpu"), 0),
            ("cube", pv.BoxSDF([0.2, 0.2, 0.2]).native_desc("cpu"), 0),
            ("cylinder", pv.CylinderSDF(0.06, 0.22).native_desc("cpu"), 1),
            ("disc", pv.CylinderSDF(0.1, 0.04).native_desc("cpu"), 1),
            ("sphere", pv.SphereSDF(0.07).native_desc("cpu"), 2)]


def _half(desc):
    return np.array([float(desc.bb_max[k]) for k in range(3)])


def _planted(desc):
    """Centre, face, edge, corner, axis and rim points, on the surface and just off it, plus exact interior ties."""
    h = _half(desc)
    s = np.array(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij")).reshape(3, -1).T   # 27 sign patterns
    pts = [s * h * f for f in (0.0, 0.5, 0.999, 1.0, 1.001, 1.5)]
    if desc.kind == nat.PVB_KIND_CYLINDER:
        r, hz = float(desc.radius), h[2]
        ang = np.linspace(0, 2 * np.pi, 16, endpoint=False)
        for rr in (0.0, 0.5 * r, r, 1.2 * r):
            for zz in (-1.2 * hz, -hz, -0.5 * hz, 0.0, -0.0, hz, 1.2 * hz):
                pts.append(np.stack([rr * np.cos(ang), rr * np.sin(ang), np.full_like(ang, zz)], 1))
    pts.append(np.array([[-0.0, -0.0, -0.0], [0.0, -0.0, 0.0]]))
    return np.concatenate(pts).astype(np.float32)


def _ties(desc):
    """Interior points where the rule's top two terms are EXACTLY equal in fp32 and fp64 (dyadic coordinates)."""
    if desc.kind == nat.PVB_KIND_SPHERE:
        return np.zeros((0, 3), np.float32)
    if desc.kind == nat.PVB_KIND_CYLINDER:
        # rho - r == |z| - h == -t on a coordinate axis of the xy-plane: rho = |x| exactly (sqrt of a rounded
        # square); with t a power of two <= min(r, h) / 2, r - t and h - t and the differences back are exact
        r, hz = np.float32(desc.radius), np.float32(desc.bb_max[2])
        p = []
        t0 = 2.0 ** np.floor(np.log2(min(r, hz) / 2))
        for t in (np.float32(t0), np.float32(t0 / 2)):
            x, z = r - t, hz - t
            assert x - r == z - hz and float(x) - float(r) == float(z) - float(hz)
            p += [[x, 0, z], [-x, 0, -z], [0, x, -z], [0, -x, z], [x, -0.0, z]]
        return np.asarray(p, np.float32)
    h = _half(desc).astype(np.float32)
    m = np.float32(min(h) / 2)
    p = []
    for sx in (1, -1):
        for sy in (1, -1):
            for sz in (1, -1):
                p.append([sx * (h[0] - m), sy * (h[1] - m), sz * (h[2] - m)])        # all three axes tie
                p.append([sx * (h[0] - m), sy * (h[1] - m), 0.0])                    # x and y tie (z deeper)
    p.append([-0.0, -0.0, -0.0]) if h[0] == h[1] == h[2] else None
    return np.asarray(p, np.float32)


@pytest.mark.parametrize("name", ["box", "cube", "cylinder", "disc", "sphere"])
def test_primitive_eval_vs_fp64_restatement(name):
    _, desc, fn = next(t for t in _prims() if t[0] == name)
    h = _half(desc)
    g = np.random.default_rng(7)
    rnd = (g.uniform(-3.0, 3.0, (200_000, 3)) * h).astype(np.float32)            # 3x the box
    q = np.concatenate([rnd, _planted(desc)])
    v, gr = _sim_eval(desc, q, fn)
    v2, gr2 = _sim_eval(desc, q, 2)                      # primitive_eval dispatches to the same function
    assert np.array_equal(v, v2) and np.array_equal(gr, gr2)
    rv, rg = pr.primitive_ref(desc, q.astype(np.float64))
    assert np.abs(v - rv).max() < 1e-6, np.abs(v - rv).max()
    clear = pr.second_gap(desc, q) > 1e-5                # fp32 and fp64 may pick different axes at near-ties
    assert clear.mean() > 0.95
    # outside, the gradient is w / |w| with w a difference of fp32 numbers (absolute error ~ ulp(|q|)): its direction
    # is only as good as ulp(|q|) / |w| close to an edge or the rim, so the tolerance follows that conditioning
    tol = np.where(rv > 0, np.maximum(1e-6, 3e-7 * np.abs(q).max(1) / np.maximum(rv, 1e-30)), 1e-6)
    err = np.abs(gr - rg).max(1)
    assert (err <= tol)[clear].all(), float((err - tol)[clear].max())
    assert (tol[clear] == 1e-6).mean() > 0.85
    assert np.isfinite(gr).all() and np.isfinite(v).all()
    # the planted points: inside, on and just off every face / edge / corner / axis / rim
    n_pl = len(_planted(desc))
    assert (rv[-n_pl:] < 0).any() and (rv[-n_pl:] == 0).any() and (rv[-n_pl:] > 0).any()


@pytest.mark.parametrize("name", ["box", "cube", "cylinder", "disc"])
def test_primitive_tie_rules_are_exact(name):
    _, desc, fn = next(t for t in _prims() if t[0] == name)
    q = _ties(desc)
    assert len(q) > 0
    v, gr = _sim_eval(desc, q, fn)
    rv, rg = pr.primitive_ref(desc, q.astype(np.float64))
    assert np.array_equal(v.astype(np.float64), rv)
    assert np.array_equal(gr.astype(np.float64), rg), (gr, rg)
    # and the stated rules themselves: first axis (box) / radial (cylinder), + at -0
    if desc.kind == nat.PVB_KIND_BOX:
        assert (gr[:, 0] != 0).all() and (np.abs(gr).sum(1) == 1).all()
        assert (gr[q[:, 0] >= 0, 0] == 1).all()
    else:
        assert (gr[:, 2] == 0).all() and (np.abs(gr).sum(1) == 1).all()      # radial


def test_box_on_the_surface_and_at_signed_zeros():
    import pytorch_volumetric_b200 as pv
    d = pv.BoxSDF([1.0, 2.0, 4.0]).native_desc("cpu")
    q = np.array([[0.5, 0, 0], [-0.5, 0, 0], [0, 1.0, 0], [0, 0, -2.0], [-0.0, 0, 0], [0.5, 1.0, 2.0]], np.float32)
    v, gr = _sim_eval(d, q, 0)
    assert np.array_equal(v, [0, 0, 0, 0, -0.5, 0])
    assert np.array_equal(gr, np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, 0, -1], [1, 0, 0], [1, 0, 0]],
                                       np.float32))


@pytest.mark.parametrize("name", ["box", "cube", "cylinder", "disc", "sphere"])
def test_bound_contract_holds_in_fp32(name):
    """value >= dist(q, bb) - prune_margin, with dist(q, bb) the kernels' own fp32 composed_aabb_lb2 -- dense fp32
    samples near the surface and out to 30 m -- and the margin is not far above the inradius."""
    _, desc, fn = next(t for t in _prims() if t[0] == name)
    h = _half(desc)
    g = np.random.default_rng(11)
    dirs = g.normal(size=(300_000, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    near = np.concatenate([
        (g.uniform(-1.05, 1.05, (300_000, 3)) * h),                                     # inside and just outside
        np.clip(g.uniform(-1, 1, (300_000, 3)) * h * 1.2, -h, h) + g.normal(scale=1e-4, size=(300_000, 3)),
        dirs * np.linalg.norm(h) * g.uniform(0.5, 3.0, (300_000, 1)),
        dirs * g.uniform(1.0, 30.0, (300_000, 1)),                                        # far field
    ]).astype(np.float32)
    q = np.concatenate([near, _planted(desc)])
    v, _ = _sim_eval(desc, q, fn)
    lb = np.sqrt(_sim_lb2(desc, q).astype(np.float64))
    margin = float(desc.prune_margin)
    slack = v.astype(np.float64) - (lb - margin)
    assert slack.min() >= 0.0, slack.min()
    inr = min(h) if desc.kind == nat.PVB_KIND_BOX else (float(desc.radius) if desc.kind == nat.PVB_KIND_SPHERE
                                                         else min(float(desc.radius), h[2]))
    assert desc.flags & nat.PVB_GRID_PRUNE_OK and inr <= margin <= inr + 2e-5
    # tight inside: the centre sits exactly on the bound up to the slack
    c, _ = _sim_eval(desc, np.zeros((1, 3), np.float32), fn)
    assert c[0] == -np.float32(inr)


def test_serial_sphere_bound_with_primitive_links():
    """rs_link_consts / rs_sphere_centre / rs_sphere_lb (robot_serial_kernel) read only the box, the margin and
    PVB_GRID_PRUNE_OK: with primitive descriptors the bound stays below the value under random rigid transforms."""
    import workloads
    g = np.random.default_rng(5)
    tm = workloads.random_rigid(16, seed=9, t_range=0.3).numpy()
    for name, desc, fn in _prims():
        pts = g.uniform(-0.6, 0.6, (20_000, 3)).astype(np.float32)
        for m in tm:
            xf = np.ascontiguousarray(m, dtype=np.float32)
            lb = np.empty(len(pts), np.float32)
            vm = ctypes.c_float()
            _simlib().simprim_sphere_lb(ctypes.byref(desc), _p(xf), _p(pts), ctypes.c_longlong(len(pts)), _p(lb),
                                        ctypes.byref(vm))
            local = (pts.astype(np.float64) @ m[:3, :3].T.astype(np.float64) + m[:3, 3]).astype(np.float32)
            v, _ = _sim_eval(desc, local, fn)
            assert (lb <= v).all(), (name, float((lb - v).max()))
            assert vm.value == np.float32(desc.prune_margin)
            assert (lb > v - 0.5).mean() > 0.2          # not vacuous


# ---------------------------------------------------------------- composition with the extension flag
def _mixed():
    from pytorch_volumetric_b200 import sdf as S
    from pytorch_volumetric_b200.voxel import GridView
    z = golden("ref_cachedsdf_probe")
    shape = tuple(int(s) for s in z["table_shape"])
    ranges = [tuple(r) for r in z["ranges"]]
    keep, out = [], {}
    for interp in ("nearest", "trilinear"):
        c = object.__new__(S.CachedSDF)
        c.ranges = ranges
        val = torch.from_numpy(z["table_val"]).reshape(shape)
        c.voxels = GridView(val, ranges, invalid_value=None)
        c.voxels_grad = torch.from_numpy(z["table_grad"])
        c._table = torch.cat([val.reshape(-1, 1), c.voxels_grad], 1).contiguous()
        c.bb = torch.as_tensor(np.asarray(z["bb"]))
        c._cdev = torch.device("cpu")
        c.out_of_bounds_strategy = S.OutOfBoundsStrategy.BOUNDING_BOX
        c.interpolation = interp
        out[interp] = c._make_desc()
        keep.append(c)
    p = {n: d for n, d, _ in _prims()}
    return z, out, p, keep


def _set(kind):
    z, grids, p, keep = _mixed()
    if kind == "mixed":
        return z, [grids["nearest"], p["box"], grids["trilinear"], p["cylinder"], p["sphere"], p["disc"]], keep
    return z, [grids["trilinear"], p["box"], p["cylinder"], p["sphere"], p["cube"]], keep


def _unpruned(descs):
    out = []
    for d in descs:
        c = d.copy()
        c.flags &= ~nat.PVB_GRID_PRUNE_OK
        out.append(c)
    return out


def _xforms(S, A, seed):
    import workloads
    return workloads.random_rigid(S * A, seed=seed, t_range=0.08).numpy()


def _points(z, n, seed):
    bb = np.asarray(z["bb"], dtype=np.float64)
    c, h = bb.mean(1), (bb[:, 1] - bb[:, 0]) / 2 + 0.15
    return (c + np.random.default_rng(seed).uniform(-1, 1, (n, 3)) * h).astype(np.float32)


@pytest.mark.parametrize("kind", ["mixed", "analytic"])
def test_composed_extension_independent_of_pruning_and_order(kind):
    z, descs, keep = _set(kind)
    S, A = len(descs), 6
    xf = _xforms(S, A, 21)
    q = _points(z, 4000, 22)
    ref = _sim_composed(descs, xf, A, q, order=range(S))
    rng = np.random.default_rng(3)
    for order in (list(range(S))[::-1], hs.bit_reversed_order(S), list(rng.permutation(S))):
        got = _sim_composed(descs, xf, A, q, order=order)
        assert all(np.array_equal(a, b) for a, b in zip(ref, got)), (kind, order)
    for order in (range(S), list(rng.permutation(S))):
        got = _sim_composed(_unpruned(descs), xf, A, q, order=order)
        assert all(np.array_equal(a, b) for a, b in zip(ref, got)), (kind, "unpruned", order)
    # every sub-SDF alone (nothing to prune), argmin in numpy: first index on ties, like torch
    per = [_sim_composed([descs[s]], xf[s * A:(s + 1) * A], A, q) for s in range(S)]
    vals = np.stack([p[0] for p in per])
    assert np.array_equal(ref[2], vals.argmin(0).astype(np.int32)) and np.array_equal(ref[0], vals.min(0))
    assert len(set(ref[2].tolist())) == S            # every sub-SDF wins somewhere


def test_composed_extension_vs_fp64_composition():
    z, descs, keep = _set("analytic")
    S, A = len(descs), 6
    xf = _xforms(S, A, 31)
    q = _points(z, 4000, 32)
    P = len(q)
    shape = tuple(int(s) for s in z["table_shape"])
    table = torch.from_numpy(z["table_val"]).reshape(shape)
    ranges = [tuple(r) for r in z["ranges"]]
    mats = xf.astype(np.float64).reshape(S, A, 4, 4)
    vals = np.empty((S, A, P))
    grads = np.empty((S, A, P, 3))
    for s in range(S):
        for a in range(A):
            local = q.astype(np.float64) @ mats[s, a, :3, :3].T + mats[s, a, :3, 3]
            if s == 0:
                rv, rg, _ = port.trilinear_lookup_port(table, ranges, z["bb"], torch.from_numpy(local))
                vals[s, a], grads[s, a] = rv.numpy(), rg.numpy()
            else:
                vals[s, a], grads[s, a] = pr.primitive_ref(descs[s], local)
    v, gr, w = _sim_composed(descs, xf, A, q)
    v, gr, w = v.reshape(A, P), gr.reshape(A, P, 3), w.reshape(A, P)
    which = vals.argmin(0)
    assert np.abs(v - vals.min(0)).max() < 5e-6
    differ = w != which
    assert differ.mean() < 1e-3
    a_idx, p_idx = np.nonzero(differ)          # argmin disagreements only at fp32 near-ties of the restated values
    assert (np.abs(vals[w[differ], a_idx, p_idx] - vals[which[differ], a_idx, p_idx]) < 1e-5).all()
    # gradients of the analytic winners, rotated back (g @ R), away from near-ties of the inside rules
    same = ~differ & (which > 0)
    a_i, p_i = np.nonzero(same)
    s_i = which[same]
    g_obj = np.einsum("nj,njk->nk", grads[s_i, a_i, p_i], mats[s_i, a_i, :3, :3])
    local = np.einsum("njk,nk->nj", mats[s_i, a_i, :3, :3], q[p_i].astype(np.float64)) + mats[s_i, a_i, :3, 3]
    gaps = np.array([pr.second_gap(descs[s], local[i:i + 1])[0] for i, s in enumerate(s_i)])
    clear = gaps > 1e-5
    # the outside gradient's conditioning, as in test_primitive_eval_vs_fp64_restatement
    tol = np.maximum(2e-6, 3e-7 * np.abs(local).max(1) / np.maximum(vals[s_i, a_i, p_i], 1e-30))
    tol = np.where(vals[s_i, a_i, p_i] > 0, tol, 2e-6)
    assert clear.mean() > 0.95 and (np.abs(gr[a_i, p_i] - g_obj).max(1) <= tol)[clear].all()


# ---------------------------------------------------------------- C ABI
def test_abi_refuses_unknown_kinds(built_lib):
    """A kind outside PVB_KIND_GRID .. PVB_KIND_CYLINDER is refused (PVB_ERR_INVALID) by every entry point that takes
    descriptors, before any launch; the descriptor keeps its size."""
    assert built_lib.pvb_sizeof_sdf_desc() == 240 == ctypes.sizeof(nat.SdfDesc)
    assert built_lib.pvb_version() == 100
    _, box, _ = _prims()[0]
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    for kind in (5, -1, 99):
        bad = box.copy()
        bad.kind = kind
        arr = nat.desc_array([box, bad])
        assert built_lib.pvb_composed_query(arr, 2, 0, fake, 1, 0, 1, fake, 100, nat.PVB_MESH_DEFAULT, fake, fake,
                                            None, None) == PVB_ERR_INVALID
        assert b"unknown kind" in built_lib.pvb_last_error()
        assert built_lib.pvb_composed_query_paired(arr, 2, 0, fake, 1, 0, 1, fake, 100, nat.PVB_MESH_DEFAULT, fake,
                                                   fake, None, None) == PVB_ERR_INVALID
        tg = (nat.OutTarget * 1)(nat.OutTarget(fake.value, fake.value))
        assert built_lib.pvb_composed_query_multi(arr, 2, 0, fake, 1, 0, 1, fake, 100, nat.PVB_MESH_DEFAULT, tg, 1,
                                                  None, None) == PVB_ERR_INVALID
        assert built_lib.pvb_composed_query_multicast(arr, 2, 0, fake, 64, 0, 64, fake, 1024, nat.PVB_MESH_DEFAULT,
                                                      fake, fake, None) == PVB_ERR_INVALID
        assert built_lib.pvb_chamfer(ctypes.byref(bad), fake, 4, fake, 100, 1.0, fake, fake, None, 0,
                                     None) == PVB_ERR_INVALID
        assert b"unknown kind" in built_lib.pvb_last_error()


def test_abi_multicast_refuses_primitives_off_the_serial_kernel(built_lib):
    """Multicast accepts primitive sets only where the point-serial robot kernel runs (<= 8 sub-SDFs, >=
    PVB_ROBOT_MIN_CFG configurations); elsewhere it refuses with a message, before any launch."""
    _, box, _ = _prims()[0]
    fake = ctypes.c_void_p(1 << 12)
    for descs, n_cfg in (([box] * 2, 4), ([box] * 9, 64)):
        rc = built_lib.pvb_composed_query_multicast(nat.desc_array(descs), len(descs), 0, fake, n_cfg, 0, n_cfg, fake,
                                                    1024, nat.PVB_MESH_DEFAULT, fake, fake, None)
        assert rc == PVB_ERR_INVALID and b"primitive" in built_lib.pvb_last_error(), (len(descs), n_cfg)


# ---------------------------------------------------------------- Python
def test_primitive_sdf_arguments_and_boxes():
    import pytorch_volumetric_b200 as pv
    for bad in ([-1, 1, 1], [1, float("nan"), 1], [1, 1, float("inf")], [1, 1]):
        with pytest.raises(ValueError):
            pv.BoxSDF(bad)
    for r, l in ((-0.1, 1), (0.1, -1), (float("nan"), 1), (0.1, float("inf"))):
        with pytest.raises(ValueError):
            pv.CylinderSDF(r, l)
    b = pv.BoxSDF([0.2, 0.4, 0.6])
    assert torch.allclose(b.surface_bounding_box(), torch.tensor([[-0.1, 0.1], [-0.2, 0.2], [-0.3, 0.3]]))
    assert torch.allclose(b.surface_bounding_box(padding=0.1, padding_ratio=0.5),
                          torch.tensor([[-0.25, 0.25], [-0.4, 0.4], [-0.55, 0.55]]))
    c = pv.CylinderSDF(0.1, 0.5)
    assert torch.allclose(c.surface_bounding_box(padding=0.01), torch.tensor([[-0.11, 0.11], [-0.11, 0.11],
                                                                              [-0.26, 0.26]]))
    d = c.native_desc("cpu")
    assert d.kind == nat.PVB_KIND_CYLINDER and d.radius == np.float32(0.1) and d.bb_max[2] == np.float32(0.25)
    assert list(d.bb_min) == [-np.float32(0.1), -np.float32(0.1), -np.float32(0.25)]
    s = pv.SphereSDF(0.3).native_desc("cpu")
    assert s.kind == nat.PVB_KIND_SPHERE and s.radius == np.float32(0.3) and list(s.bb_max) == [np.float32(0.3)] * 3
    assert s.flags == nat.PVB_GRID_PRUNE_OK and 0.3 <= s.prune_margin < 0.3 + 2e-5


_URDF = """<robot name="r">
<link name="base"><visual><origin xyz="0 0 0.05" rpy="0 0 0.4"/><geometry><box size="0.2 0.3 0.1"/></geometry></visual>
</link>
<link name="l1"><visual><geometry><mesh filename="link.obj" scale="2 2 2"/></geometry></visual>
<visual><origin xyz="0.01 0.02 0.1" rpy="0.3 0.2 0.1"/><geometry><cylinder radius="0.05" length="0.2"/></geometry>
</visual></link>
<link name="l2"><visual><origin xyz="0 0 0.03"/><geometry><sphere radius="0.04"/></geometry></visual>
<visual><geometry><capsule radius="0.04" length="0.1"/></geometry></visual></link>
<joint name="j1" type="revolute"><parent link="base"/><child link="l1"/><origin xyz="0 0 0.1"/><axis xyz="0 0 1"/>
</joint>
<joint name="j2" type="revolute"><parent link="l1"/><child link="l2"/><origin xyz="0 0 0.2"/><axis xyz="0 1 0"/>
</joint>
</robot>"""


def test_robot_primitive_visuals(tmp_path, caplog):
    import pytorch_volumetric_b200 as pv
    import workloads
    from pytorch_volumetric_b200.meshio import write_obj
    v, f = workloads.fixture_mesh("probe")
    write_obj(str(tmp_path / "link.obj"), v, f)
    chain = pv.build_serial_chain_from_urdf(_URDF, "l2")
    with caplog.at_level(logging.WARNING):
        plain = pv.RobotSDF(chain, path_prefix=str(tmp_path))
    assert plain.sdf_to_link_name == ["l1"] and len(plain.sdf.sdfs) == 1
    assert isinstance(plain.sdf.sdfs[0], pv.MeshSDF)
    warned = [r.getMessage() for r in caplog.records if "non-mesh" in r.getMessage()]
    assert len(warned) == 4                      # box, cylinder, sphere and the capsule, as before

    caplog.clear()
    with caplog.at_level(logging.WARNING):
        robot = pv.RobotSDF(chain, path_prefix=str(tmp_path), primitive_visuals=True,
                            link_sdf_cls=lambda fac: pv.MeshSDF(fac))
    assert robot.sdf_to_link_name == ["base", "l1", "l1", "l2"]
    kinds = [type(s) for s in robot.sdf.sdfs]
    assert kinds == [pv.BoxSDF, pv.MeshSDF, pv.CylinderSDF, pv.SphereSDF]
    assert robot.sdf.sdfs[0].size == [0.2, 0.3, 0.1]
    assert (robot.sdf.sdfs[2].radius, robot.sdf.sdfs[2].length) == (0.05, 0.2) and robot.sdf.sdfs[3].radius == 0.04
    warned = [r.getMessage() for r in caplog.records if "non-mesh" in r.getMessage()]
    assert len(warned) == 1 and "Visual(None, None) for l2" in warned[0]     # the capsule: not a URDF primitive
    # visual offsets: the <origin> of every visual, in the same order
    off = robot.offset_transforms.get_matrix()
    assert torch.allclose(off[0, :3, 3], torch.tensor([0, 0, 0.05])) and torch.allclose(off[1], torch.eye(4))
    assert torch.allclose(off[2, :3, 3], torch.tensor([0.01, 0.02, 0.1])) and not torch.allclose(off[2, :3, :3],
                                                                                                torch.eye(3))
    assert torch.allclose(off[3, :3, 3], torch.tensor([0, 0, 0.03]))
    # the link boxes follow the primitives
    boxes = robot.link_bounding_boxes()
    assert boxes.shape == (4, 8, 3)


def test_robot_primitive_bad_size_raises():
    import pytorch_volumetric_b200 as pv
    urdf = _URDF.replace('<box size="0.2 0.3 0.1"/>', '<box size="0.2 -0.3 0.1"/>')
    chain = pv.build_serial_chain_from_urdf(urdf, "l2")
    with pytest.raises(ValueError):
        pv.RobotSDF(chain, primitive_visuals=True, link_sdf_cls=lambda fac: None)


def test_sphere_sets_bit_identical_on_the_extension_path():
    """Sets containing SphereSDF moved from the nearest-voxel instantiations (spheres never pruned) to the extension
    ones (spheres pruned by their bound): values, gradients and argmin are bit-identical."""
    z, grids, p, keep = _mixed()
    zc = golden("ref_composed")
    S, A = int(zc["S"]), int(zc["A"])
    sph = hs.sphere_desc(float(zc["sphere_radius"]))
    near = grids["nearest"]
    for descs in ([near, near, sph, near], [sph, near, near, sph], [p["sphere"], sph, near, near]):
        old = hs.composed(descs, zc["tmat"], A, zc["q"])               # composed_consider<kMesh, kExt = false>
        new = _sim_composed(descs, zc["tmat"], A, zc["q"])             # composed_consider<false, kExt = true>
        assert all(np.array_equal(a, b) for a, b in zip(old, new))
