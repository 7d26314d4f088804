"""CPU tier for trilinear CachedSDF links in the fused composed kernels (CachedSDF(interpolation="trilinear") inside
ComposedSDF / RobotSDF).

1. The pruning bound every fused kernel relies on -- a sub-SDF is skipped when dist(q, bb) - prune_margin already
   exceeds the running minimum -- holds for the trilinear interpolant with the margin `grid_prune_margin` measures
   for the nearest-voxel rule (the interpolant is a convex combination of 8 corner values; the weighted mean
   distance of q to the corners is at most half a cell diagonal).
2. The device arithmetic (pvb_device.cuh compiled for the host by tests/hostsim/hostsim_trilinear.cpp):
   grid_trilinear_eval against the fp64 restatement oracle.port.trilinear_lookup_port, and composed_consider over
   trilinear and mixed compositions -- independent of pruning and visiting order, and equal to an fp64 restatement
   of the composition."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from helpers import golden
from oracle import port
from pytorch_volumetric_b200 import _native as nat
from pytorch_volumetric_b200.sdf import grid_prune_margin

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_trilinear.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_trilinear.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_trilinear.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
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


def _grid_desc(table_val, table_grad, ranges, bb, interpolation):
    """pvb_sdf_desc (GRID, bounding-box rule) built by the product's CachedSDF._make_desc over CPU tensors, as
    tests/hostsim_lib.grid_desc does, with the given interpolation.  Returns (desc, keepalive)."""
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
    return c._make_desc(), c


def _sim_trilinear(desc, points):
    p = np.ascontiguousarray(points, dtype=np.float32); n = len(p)
    val, grad = np.empty(n, np.float32), np.empty((n, 3), np.float32)
    _simlib().simtri_grid_trilinear(ctypes.byref(desc), _p(p), ctypes.c_longlong(n), _p(val), _p(grad))
    return val, grad


def _sim_composed(descs, xforms, n_cfg, points, order=None):
    """(val [n_cfg*P], grad [n_cfg*P,3], which [n_cfg*P]) through composed_consider<true, true>; `order` as in
    hostsim_lib.composed (default: the kernels' bit-reversed order)."""
    p = np.ascontiguousarray(points, dtype=np.float32); n = len(p); S = len(descs)
    arr = (nat.SdfDesc * S)(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    assert xf.shape == (S * n_cfg, 4, 4)
    order = hs.bit_reversed_order(S) if order is None else list(order)
    assert sorted(order) == list(range(S))
    od = np.asarray(order, dtype=np.uint8)
    val, grad = np.empty(n_cfg * n, np.float32), np.empty((n_cfg * n, 3), np.float32)
    which = np.empty(n_cfg * n, np.int32)
    _simlib().simtri_composed(arr, ctypes.c_int(S), _p(od), _p(xf), ctypes.c_int(n_cfg), _p(p), ctypes.c_longlong(n),
                              _p(val), _p(grad), _p(which))
    return val, grad, which


def _aabb_distance(q, bb):
    q = np.asarray(q, dtype=np.float64)
    bb = np.asarray(bb, dtype=np.float64)
    return np.linalg.norm(np.maximum(np.maximum(bb[:, 0] - q, q - bb[:, 1]), 0.0), axis=-1)


def _slack(table, ranges, bb, q):
    """value of the interpolant minus the pruning bound dist(q, bb) - margin (>= 0 where the bound holds)."""
    lo = [float(r[0]) for r in ranges]; hi = [float(r[1]) for r in ranges]
    margin = grid_prune_margin(table, lo, hi, bb)
    v, _, inb = port.trilinear_lookup_port(table, ranges, bb, torch.as_tensor(q))
    return v.numpy() - (_aabb_distance(q, bb) - margin), inb.numpy(), margin


def _in_and_out(lo, hi, n, seed):
    g = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    span = hi - lo
    return (lo - 0.5 * span + 2.0 * span * g.random((n, 3))).astype(np.float32)


@pytest.mark.parametrize("name", ["probe", "drill"])
def test_trilinear_values_respect_the_prune_bound(name):
    z = golden(f"ref_cachedsdf_{name}")
    shape = tuple(int(s) for s in z["table_shape"])
    table = torch.from_numpy(z["table_val"]).reshape(shape)
    ranges = [tuple(r) for r in z["ranges"]]
    bb = np.asarray(z["bb"], dtype=np.float32)         # fp32 like the cast at sdf.py:556-557
    lo = [r[0] for r in ranges]; hi = [r[1] for r in ranges]
    q = np.concatenate([_in_and_out(lo, hi, 300_000, 0), z["q"].astype(np.float32)])
    slack, inb, margin = _slack(table, ranges, bb.astype(np.float64), q)
    assert inb.mean() > 0.1 and (~inb).mean() > 0.1          # both sides of the range are exercised
    assert float(slack.min()) >= 0.0, float(slack.min())
    assert float(slack[inb].min()) < 2.5 * float(z["resolution"]) * 3 ** 0.5     # and it is not vacuous


def test_trilinear_prune_bound_on_adversarial_tables():
    """Random table contents (t measured on them) and a 3 x 3 x 3 table queried at cell centres, where every
    f_a (1 - f_a) peaks and the weighted corner distance reaches half the cell diagonal."""
    g = np.random.default_rng(1)
    ranges = [(-1.0, 1.0), (-0.5, 1.5), (-1.0, 0.6)]
    shape = (17, 21, 13)
    bb = np.array([[-0.2, 0.3], [0.1, 0.4], [-0.5, -0.1]])
    table = torch.from_numpy(g.uniform(-3.0, 3.0, shape))
    q = _in_and_out([r[0] for r in ranges], [r[1] for r in ranges], 200_000, 2)
    slack, inb, _ = _slack(table, ranges, bb, q)
    assert inb.mean() > 0.1 and float(slack.min()) >= 0.0, float(slack.min())

    # 3 x 3 x 3: tables that sit exactly on the bound at every corner (value = dist(corner, bb) - t)
    ranges = [(0.0, 2.0), (0.0, 1.0), (0.0, 4.0)]
    axes = [np.linspace(a, b, 3) for a, b in ranges]
    corners = np.stack(np.meshgrid(*axes, indexing="ij"), -1)
    centres = np.stack(np.meshgrid(*[0.5 * (a[:-1] + a[1:]) for a in axes], indexing="ij"), -1).reshape(-1, 3)
    for bb in (np.array([[0.5, 0.5], [0.25, 0.25], [1.0, 1.0]]),          # a point at a cell centre
               np.array([[0.4, 1.6], [0.3, 0.7], [-1.0, 0.2]]),
               np.array([[5.0, 6.0], [5.0, 6.0], [5.0, 6.0]])):            # far outside the range
        for t in (0.0, 0.7):
            table = torch.from_numpy(_aabb_distance(corners.reshape(-1, 3), bb).reshape(3, 3, 3) - t)
            slack, inb, _ = _slack(table, ranges, bb, centres.astype(np.float32))
            assert inb.all() and float(slack.min()) >= 0.0, (bb, t, float(slack.min()))


# ---------------------------------------------------------------- device arithmetic on the host
def _probe_descs():
    z = golden("ref_cachedsdf_probe")
    shape = tuple(int(s) for s in z["table_shape"])
    args = (torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"]),
            [tuple(r) for r in z["ranges"]], z["bb"])
    tri, k1 = _grid_desc(*args, interpolation="trilinear")
    near, k2 = _grid_desc(*args, interpolation="nearest")
    return z, tri, near, (k1, k2)


def test_trilinear_descriptor_keeps_the_prune_bound():
    _, tri, near, keep = _probe_descs()
    assert tri.flags & nat.PVB_GRID_TRILINEAR and tri.flags & nat.PVB_GRID_PRUNE_OK
    assert tri.prune_margin == near.prune_margin and not near.flags & nat.PVB_GRID_TRILINEAR


def test_grid_trilinear_eval_vs_its_cpu_restatement(built_lib):
    z, tri, _, keep = _probe_descs()
    ranges = [tuple(r) for r in z["ranges"]]
    shape = tuple(int(s) for s in z["table_shape"])
    lo = np.array([r[0] for r in ranges]); hi = np.array([r[1] for r in ranges])
    q = np.concatenate([z["q"].astype(np.float32), _in_and_out(lo, hi, 100_000, 3)])
    v, g = _sim_trilinear(tri, q)
    rv, rg, inb = port.trilinear_lookup_port(torch.from_numpy(z["table_val"]).reshape(shape), ranges, z["bb"],
                                             torch.from_numpy(q))
    rv, rg, inb = rv.numpy(), rg.numpy(), inb.numpy()
    assert np.abs(v - rv).max() < 2e-6
    u = (q.astype(np.float64) - lo) / ((hi - lo) / (np.array(shape) - 1))
    off_lattice = (np.abs(u - np.round(u)) > 1e-3).all(axis=1) & inb        # the gradient jumps across cell faces
    assert off_lattice.sum() > 10_000 and (~inb).sum() > 10_000
    assert np.abs(g - rg)[off_lattice].max() < 1e-4
    assert np.abs(g - rg)[~inb].max() < 1e-6


def _compositions():
    """(golden composition, [(name, descriptors)]): the golden ComposedSDF set with trilinear grids, and a mix of
    nearest and trilinear grids with the sphere."""
    z, tri, near, keep = _probe_descs()
    zc = golden("ref_composed")
    sph = hs.sphere_desc(float(zc["sphere_radius"]))
    return z, zc, [("trilinear", [tri, tri, sph, tri]), ("mixed", [near, tri, sph, tri]),
                   ("mixed2", [tri, near, near, sph])], keep


def _unpruned(descs):
    out = []
    for d in descs:
        c = d.copy()
        c.flags &= ~nat.PVB_GRID_PRUNE_OK
        out.append(c)
    return out


def test_composed_trilinear_independent_of_pruning_and_order(built_lib):
    z, zc, sets, keep = _compositions()
    S, A = int(zc["S"]), int(zc["A"])
    for name, descs in sets:
        ref = _sim_composed(descs, zc["tmat"], A, zc["q"], order=range(S))
        for order in (list(range(S))[::-1], hs.bit_reversed_order(S), [2, 0, 3, 1]):
            got = _sim_composed(descs, zc["tmat"], A, zc["q"], order=order)
            assert all(np.array_equal(a, b) for a, b in zip(ref, got)), (name, order)
        for order in (range(S), [3, 1, 2, 0]):
            got = _sim_composed(_unpruned(descs), zc["tmat"], A, zc["q"], order=order)
            assert all(np.array_equal(a, b) for a, b in zip(ref, got)), (name, "unpruned", order)
        # every sub-SDF alone (nothing to prune), argmin in numpy: first index on ties, like torch
        per = [_sim_composed([descs[s]], zc["tmat"][s * A:(s + 1) * A], A, zc["q"]) for s in range(S)]
        vals = np.stack([p[0] for p in per])
        which = vals.argmin(0)
        assert np.array_equal(ref[2], which.astype(np.int32)) and np.array_equal(ref[0], vals.min(0)), name


def test_composed_trilinear_vs_fp64_restatement(built_lib):
    z, zc, sets, keep = _compositions()
    S, A = int(zc["S"]), int(zc["A"])
    shape = tuple(int(s) for s in z["table_shape"])
    table = torch.from_numpy(z["table_val"]).reshape(shape)
    ranges = [tuple(r) for r in z["ranges"]]
    q = np.asarray(zc["q"], dtype=np.float64)
    P = len(q)
    mats = np.asarray(zc["tmat"], dtype=np.float64).reshape(S, A, 4, 4)
    v, _, w = _sim_composed(sets[0][1], zc["tmat"], A, zc["q"])
    v, w = v.reshape(A, P), w.reshape(A, P)
    vals = np.empty((S, A, P))
    for s in range(S):
        for a in range(A):
            local = q @ mats[s, a, :3, :3].T + mats[s, a, :3, 3]
            if s == 2:
                vals[s, a] = np.linalg.norm(local, axis=1) - float(zc["sphere_radius"])
            else:
                vals[s, a] = port.trilinear_lookup_port(table, ranges, z["bb"], torch.from_numpy(local))[0].numpy()
    which = vals.argmin(0)
    assert np.abs(v - vals.min(0)).max() < 5e-6
    differ = w != which
    assert differ.mean() < 1e-3
    # an argmin disagreement only where the two sub-SDFs' restated values are within 1e-5 (an fp32 near-tie)
    a_idx, p_idx = np.nonzero(differ)
    assert (np.abs(vals[w[differ], a_idx, p_idx] - vals[which[differ], a_idx, p_idx]) < 1e-5).all()


# ---------------------------------------------------------------- C ABI refusals (no kernel launch involved)
def test_abi_refuses_what_no_kernel_computes(built_lib):
    """pvb_chamfer has the nearest-voxel rule only and refuses a TRILINEAR descriptor instead of answering with it;
    multicast needs the point-serial robot kernel for trilinear sets (<= 8 links, >= PVB_ROBOT_MIN_CFG
    configurations); TRILINEAR with LOOKUP_GT_SDF is refused by the composed entry points."""
    z, tri, near, keep = _probe_descs()
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    rc = built_lib.pvb_chamfer(ctypes.byref(tri), fake, 4, fake, 100, 1.0, fake, fake, None, 0, None)
    assert rc == PVB_ERR_INVALID and b"TRILINEAR" in built_lib.pvb_last_error()
    for descs, n_cfg in (([tri] * 2, 4), ([tri] * 9, 64), ([near] * 8 + [tri], 64)):
        arr = nat.desc_array(descs)
        rc = built_lib.pvb_composed_query_multicast(arr, len(descs), 0, fake, n_cfg, 0, n_cfg, fake, 1024,
                                                    nat.PVB_MESH_DEFAULT, fake, fake, None)
        assert rc == PVB_ERR_INVALID and b"trilinear" in built_lib.pvb_last_error(), (len(descs), n_cfg)
    gt = tri.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    rc = built_lib.pvb_composed_query(nat.desc_array([near, gt]), 2, 1, fake, 1, 0, 1, fake, 100,
                                      nat.PVB_MESH_DEFAULT, fake, fake, None, None)
    assert rc == PVB_ERR_INVALID and b"bounding-box" in built_lib.pvb_last_error()
