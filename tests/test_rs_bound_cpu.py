"""CPU tier for the per-lane link bound of robot_serial_kernel (rs_link_consts, rs_sphere_centre and rs_sphere_lb of
pvb_device.cuh, compiled for the host by tests/hostsim/hostsim_rsbound.cpp): the radius term lives per link in the
kernel's constant bank and the sphere centre per (configuration, link) in shared memory.  The bound must never exceed
the true point-to-AABB distance minus the prune margin -- the kernel's pruning is exact only then -- and must never
reject a link whose transform is not an isometry or whose descriptor lacks PVB_GRID_PRUNE_OK; slots beyond n_sdf are
+inf.  The nearest-link selection over such bounds always names a real link."""
import ctypes
import os
import subprocess

import numpy as np

import hostsim_lib as hs
import workloads
from pytorch_volumetric_b200 import _native as nat

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_rsbound.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_rsbound.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_rsbound.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
                   os.path.join(root, "pytorch_volumetric_b200", "csrc", "pvb_device.cuh"),
                   os.path.join(root, "include", "pvb.h")]
        if not os.path.exists(_SIM_LIB) or any(os.path.getmtime(f) > os.path.getmtime(_SIM_LIB) for f in sources):
            os.makedirs(os.path.dirname(_SIM_LIB), exist_ok=True)
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                            "-I", _SIM_DIR, sources[0], "-o", _SIM_LIB], check=True)
        _sim = ctypes.CDLL(_SIM_LIB)
        _sim.simrs_visit_margin.restype = ctypes.c_float
    return _sim


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _box_desc(rng, prune_ok=True):
    d = nat.SdfDesc()
    d.kind = nat.PVB_KIND_GRID
    d.flags = nat.PVB_GRID_PRUNE_OK if prune_ok else 0
    lo = rng.uniform(-0.2, 0.1, 3)
    hi = lo + rng.uniform(0.005, 0.3, 3)                    # thin slabs up to near-cubes
    for k in range(3):
        d.bb_min[k], d.bb_max[k] = float(lo[k]), float(hi[k])
    d.prune_margin = float(rng.uniform(0.0, 0.03))
    return d


def _sphere_lb(descs, xforms, n_cfg, pts):
    lb = np.empty((n_cfg, len(pts), 8), np.float32)
    arr = (nat.SdfDesc * len(descs))(*descs)
    xf = np.ascontiguousarray(xforms, dtype=np.float32)
    p = np.ascontiguousarray(pts, dtype=np.float32)
    _simlib().simrs_sphere_lb(arr, len(descs), _p(xf), n_cfg, _p(p), ctypes.c_longlong(len(p)), _p(lb))
    return lb


def _aabb_dist(desc, xform, pts):
    """fp64 distance from M p to the descriptor's box, M the fp32 4x4 the kernel reads: what its visit tests."""
    m = xform.astype(np.float64)
    q = pts.astype(np.float64) @ m[:3, :3].T + m[:3, 3]
    lo, hi = np.array(desc.bb_min[:], np.float64), np.array(desc.bb_max[:], np.float64)
    return np.linalg.norm(np.clip(np.maximum(lo - q, q - hi), 0.0, None), axis=-1)


def test_sphere_bound_never_exceeds_the_aabb_distance():
    rng = np.random.default_rng(11)
    n_cfg, n_sdf = 24, 6
    descs = [_box_desc(rng) for _ in range(n_sdf)]
    xf = workloads.random_rigid(n_sdf * n_cfg, seed=5, t_range=0.6).numpy()
    # points near and inside the boxes as well as far away
    pts = np.concatenate([rng.uniform(-1.0, 1.0, (3000, 3)), rng.normal(0.0, 0.15, (3000, 3))]).astype(np.float32)
    lb = _sphere_lb(descs, xf, n_cfg, pts)
    for s, d in enumerate(descs):
        for c in range(n_cfg):
            truth = _aabb_dist(d, xf[s * n_cfg + c], pts) - d.prune_margin
            assert np.isfinite(lb[c, :, s]).all()
            assert (lb[c, :, s].astype(np.float64) <= truth).all(), (s, c)
            # and it is a useful bound: within the sphere's slack of the truth far from the box
            far = truth > 1.0
            assert (lb[c, far, s] > truth[far] - 0.6).all()
    assert np.isposinf(lb[:, :, n_sdf:]).all()          # slots beyond n_sdf: never the nearest, never visited


def test_non_isometric_and_unprunable_links_are_never_rejected():
    rng = np.random.default_rng(12)
    n_cfg, n_sdf = 8, 4
    descs = [_box_desc(rng), _box_desc(rng, prune_ok=False), _box_desc(rng), _box_desc(rng)]
    xf = workloads.random_rigid(n_sdf * n_cfg, seed=6).numpy()
    scaled = np.zeros(n_sdf * n_cfg, bool)
    scaled[2 * n_cfg:3 * n_cfg:2] = True                    # link 2: every other configuration scaled by 1.01
    xf[scaled, :3, :3] *= 1.01
    pts = rng.uniform(-1.0, 1.0, (2000, 3)).astype(np.float32)
    lb = _sphere_lb(descs, xf, n_cfg, pts)
    never = lambda a: ~(a > np.float32(-3e38))               # `lb > best` is false for every finite best
    assert never(lb[:, :, 1]).all()
    assert never(lb[0::2, :, 2]).all() and np.isfinite(lb[1::2, :, 2]).all()
    assert np.isfinite(lb[:, :, [0, 3]]).all()
    assert _simlib().simrs_visit_margin(ctypes.byref(descs[0])) == np.float32(descs[0].prune_margin)
    assert np.isposinf(_simlib().simrs_visit_margin(ctypes.byref(descs[1])))
    # the first link to visit is always a real one, whatever mix of finite, -inf, NaN and +inf bounds comes in
    rows = lb.reshape(-1, 8)
    pred = np.empty(len(rows), np.int32)
    hs.lib().sim_rs_nearest(_p(np.ascontiguousarray(rows)), ctypes.c_longlong(len(rows)), n_sdf, _p(pred))
    assert pred.min() >= 0 and pred.max() < n_sdf
