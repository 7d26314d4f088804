"""CPU tier for self-collision-cost queries (ComposedSDF.self_collision_cost / RobotSDF.self_collision_cost /
pvb_composed_query_self_collision_cost): for every configuration, the hinge cost sum max(0, m - d)^2 over every
source sub-SDF's link points against the sub-SDFs its row of `allowed` names, its twist gradient per sub-SDF (+tau to
the target, -tau to the source), and for a robot its joint gradient.

1. The device arithmetic, compiled for the host by tests/hostsim/hostsim_self_collision_cost.cpp in the order
   robot_self_collision_cost_kernel runs it, on the nearest, trilinear, mixed, drill, primitive and primitive+grid
   golden sets, with ties and duplicated points:
   - every pair the sequence evaluates below the margin has the (value, gradient, sub-SDF) of the per-point query of
     the allowed sub-composition at the posed point, bit for bit, and no pair below the margin is skipped;
   - cost and every twist component are within 1e-6 * sum|term| of the fp64 sum of the same fp32 terms;
   - rows are bit-identical under permuted configuration orders, slab splits and any forced first visit.
2. The sign convention on two spheres, with hand-computed values, and exact zeros for far-apart links and empty rows.
3. The joint gradient of a primitive chain against central differences of an fp64 restatement (fp64 forward
   kinematics and tests/primitive_ref.py SDFs), over the points whose argmin and shape rule stay put over the step.
4. The C ABI refusals and the Python shape rules, without a GPU."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import hostsim_lib as hs
from pytorch_volumetric_b200 import _native as nat
from test_paired_cpu import _sim_paired, _table_descs
from test_self_clearance_cpu import _allowed_cases, _inverse, _link_points, _masks
from test_swept_cpu import _all_sets, _trajectory

PVB_ERR_INVALID = -1        # include/pvb.h pvb_status

_SIM_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_SIM_LIB = os.path.join(_SIM_DIR, "_build", "libpvb_hostsim_self_collision_cost.so")
_sim = None


def _simlib():
    """tests/hostsim/hostsim_self_collision_cost.cpp built like tests/hostsim (g++, -ffp-contract=off), rebuilt when
    stale."""
    global _sim
    if _sim is None:
        root = os.path.dirname(os.path.dirname(_SIM_DIR))
        sources = [os.path.join(_SIM_DIR, "hostsim_self_collision_cost.cpp"), os.path.join(_SIM_DIR, "cuda_runtime.h"),
                   os.path.join(_SIM_DIR, "hostsim_robot.h"),
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


def _fused(descs, xf, inv, n_cfg, lp, allowed, margin, cfg_begin=0, cfg_count=None, lanes=32, cfg_order=0,
           shuffle_seed=0, first=-1):
    """robot_self_collision_cost_kernel on the host: (cost [C], twist [C, S, 6], and per (configuration, source,
    point): visited, value, gradient, sub-SDF, posed point, plus the number of lookups)."""
    S, K = lp.shape[:2]
    cfg_count = n_cfg - cfg_begin if cfg_count is None else cfg_count
    lp = np.ascontiguousarray(lp, dtype=np.float32)
    NP = cfg_count * S * K
    cost, twist = np.empty(cfg_count, np.float32), np.empty((cfg_count, S, 6), np.float32)
    vis, pv, pg, pw, px = np.empty(NP, np.uint8), np.empty(NP, np.float32), np.empty((NP, 3), np.float32), \
        np.empty(NP, np.int32), np.empty((NP, 3), np.float32)
    evals = ctypes.c_longlong(0)
    _simlib().simscc_fused((nat.SdfDesc * S)(*descs), ctypes.c_int(S), _p(xf), _p(inv), ctypes.c_int(n_cfg),
                           ctypes.c_int(cfg_begin), ctypes.c_int(cfg_count), _p(lp), ctypes.c_int(K),
                           _p(_masks(allowed)), ctypes.c_float(margin), ctypes.c_int(lanes), ctypes.c_int(cfg_order),
                           ctypes.c_int(shuffle_seed), ctypes.c_int(first), _p(cost), _p(twist), _p(vis), _p(pv),
                           _p(pg), _p(pw), _p(px), ctypes.byref(evals))
    sh = (cfg_count, S, K)
    return (cost, twist, vis.astype(bool).reshape(sh), pv.reshape(sh), pg.reshape(*sh, 3), pw.reshape(sh),
            px.reshape(*sh, 3), evals.value)


def _pose(inv, n_cfg, i, lp_i):
    """[n_cfg, K, 3]: link points of source i posed by W_i with composed_xform (pvb_transform_points_paired)."""
    S = len(inv) // n_cfg
    w = np.ascontiguousarray(np.asarray(inv, dtype=np.float32).reshape(S, n_cfg, 4, 4)[i])
    p = np.ascontiguousarray(lp_i, dtype=np.float32)
    out = np.empty((n_cfg, len(p), 3), np.float32)
    _simlib().simscc_pose(_p(w), ctypes.c_int(n_cfg), _p(p), ctypes.c_int(len(p)), _p(out))
    return out


def _per_point(descs, xf, inv, n_cfg, lp, allowed):
    """The definition's per-point values: for every source i with an allowed row, its points posed with W_i and the
    host build of query_paired on the composition of its allowed sub-SDFs, which mapped back.  (v, g, w, x) of shape
    [A, S, K] (+3); empty rows get +inf, 0, -1."""
    S, K = lp.shape[:2]
    tm = np.asarray(xf, dtype=np.float32).reshape(S, n_cfg, 4, 4)
    v = np.full((n_cfg, S, K), np.inf, np.float32)
    g = np.zeros((n_cfg, S, K, 3), np.float32)
    w = np.full((n_cfg, S, K), -1, np.int32)
    x = np.zeros((n_cfg, S, K, 3), np.float32)
    for i in range(S):
        js = [j for j in range(S) if allowed[i][j] and j != i]
        x[:, i] = _pose(inv, n_cfg, i, lp[i])
        if not js:
            continue
        sub_xf = np.ascontiguousarray(tm[js].reshape(len(js) * n_cfg, 4, 4))
        vi, gi, wi = _sim_paired([descs[j] for j in js], sub_xf, n_cfg, x[:, i])
        v[:, i], g[:, i] = vi.reshape(n_cfg, K), gi.reshape(n_cfg, K, 3)
        w[:, i] = np.asarray(js, np.int32)[wi.reshape(n_cfg, K)]
    return v, g, w, x


def _terms(v, g, x, m):
    """fp32 (h^2, tau [.., 6]) of every pair below m, as collision_cost_term forms them; 0 elsewhere."""
    h = np.where(v < m, np.float32(m) - v, np.float32(0)).astype(np.float32)
    t = np.float32(2) * h
    cr = np.cross(x.astype(np.float64), g.astype(np.float64))
    tau = np.concatenate([g.astype(np.float64), cr], axis=-1) * t.astype(np.float64)[..., None]
    return (h.astype(np.float64) ** 2), tau


def _fp64_sum(v, g, w, x, m, S):
    """The fp64 sums of the definition's terms: cost [A], twist [A, S, 6], and the sums of |term| per entry."""
    c, tau = _terms(v, g, x, m)
    A, _, K = v.shape
    twist = np.zeros((A, S, 6))
    abs_tw = np.zeros((A, S, 6))
    onehot = (w[..., None] == np.arange(S)).astype(np.float64)                      # [A, S_src, K, S]
    twist += np.einsum("aiks,aikq->asq", onehot, tau)
    abs_tw += np.einsum("aiks,aikq->asq", onehot, np.abs(tau))
    twist -= tau.sum(axis=2)                                                         # the source's total
    abs_tw += np.abs(tau).sum(axis=2)
    return c.sum(axis=(1, 2)), twist, c.sum(axis=(1, 2)), abs_tw


def _check_within(cost, twist, ref, what, rel=1e-6):
    rc, rt, ac, at = ref
    assert (np.abs(cost - rc) <= rel * ac + 1e-30).all(), (what, "cost", float(np.abs(cost - rc).max()))
    assert (np.abs(twist - rt) <= rel * at + 1e-30).all(), (what, "twist", float(np.abs(twist - rt).max()))


def _margin(v, allowed_pairs, q):
    return float(np.float32(np.quantile(v[allowed_pairs], q)))


# ---------------------------------------------------------------- 1. the kernel's sequence
@pytest.mark.parametrize("A", [3, 37])
def test_fused_self_collision_cost_equals_the_fp64_sum(built_lib, A):
    zc, sets, keep = _all_sets()
    S0, A0 = int(zc["S"]), int(zc["A"])
    tm = zc["tmat"] if A == A0 else _trajectory(zc["tmat"], S0, A0, A, seed=A)
    tm = np.ascontiguousarray(tm, dtype=np.float32)
    inv = _inverse(tm)
    contributed = 0
    for name, descs in sets:
        S = len(descs)
        for K in (1, 45, 130):
            lp = _link_points(zc, tm, S, A, K, seed=K + A)
            for case, allowed in _allowed_cases(S).items():
                v, g, w, x = _per_point(descs, tm, inv, A, lp, allowed)
                if case == "empty":
                    cost, twist = _fused(descs, tm, inv, A, lp, allowed, 0.05)[:2]
                    assert not cost.any() and not twist.any(), (name, K)
                    continue
                on = w >= 0
                for q in (0.05, 0.3):
                    m = _margin(v, on, q)
                    what = (name, A, K, case, m)
                    cost, twist, vis, pv, pg, pw, px, evals = _fused(descs, tm, inv, A, lp, allowed, m)
                    inside = on & (v < m)
                    contributed += int(inside.sum())
                    # no pair below the margin is skipped, and each is the per-point query's, bit for bit
                    assert vis[inside].all(), what
                    assert np.array_equal(pv[inside], v[inside]) and np.array_equal(pw[inside], w[inside]), what
                    assert np.array_equal(pg[inside], g[inside]), what
                    assert np.array_equal(px[vis], x[vis]), what
                    # an evaluated pair at or above the margin may be inexact, but is never below it
                    assert not ((pw >= 0) & ~inside & (pv < m)).any(), what
                    # empty rows are never visited
                    assert not vis[:, [i for i in range(S) if not any(allowed[i][j] for j in range(S) if j != i)]].any()
                    _check_within(cost, twist, _fp64_sum(v, g, w, x, m, S), what)
                    # configuration orders and forced first visits change nothing
                    for kw in [dict(cfg_order=1), dict(cfg_order=2, shuffle_seed=K)] + \
                            [dict(first=f, cfg_order=f % 3) for f in range(S)]:
                        c2, t2 = _fused(descs, tm, inv, A, lp, allowed, m, **kw)[:2]
                        assert np.array_equal(c2, cost) and np.array_equal(t2, twist), (what, kw)
                    # fewer lanes: another summation order, within the same bound
                    c2, t2 = _fused(descs, tm, inv, A, lp, allowed, m, lanes=5)[:2]
                    _check_within(c2, t2, _fp64_sum(v, g, w, x, m, S), (what, "lanes=5"))
    assert contributed > 1000


def test_slabs_reproduce_the_rows_of_the_full_call(built_lib):
    zc, sets, keep = _all_sets()
    S0, A0 = int(zc["S"]), int(zc["A"])
    A = 40
    tm = np.ascontiguousarray(_trajectory(zc["tmat"], S0, A0, A, seed=11), dtype=np.float32)
    inv = _inverse(tm)
    for name, descs in sets:
        S = len(descs)
        lp = _link_points(zc, tm, S, A, 70, seed=4)
        allowed = _allowed_cases(S)["full"]
        v, _, w, _ = _per_point(descs, tm, inv, A, lp, allowed)
        m = _margin(v, w >= 0, 0.2)
        cost, twist = _fused(descs, tm, inv, A, lp, allowed, m)[:2]
        assert cost.any(), name
        for begin, count in ((0, 1), (5, 32), (31, 2), (33, 7), (39, 1), (1, 39)):
            c2, t2 = _fused(descs, tm, inv, A, lp, allowed, m, cfg_begin=begin, cfg_count=count, cfg_order=2,
                            shuffle_seed=begin)[:2]
            rows = slice(begin, begin + count)
            assert np.array_equal(c2, cost[rows]) and np.array_equal(t2, twist[rows]), (name, begin, count)


def test_ties_and_duplicated_points(built_lib):
    """A sub-SDF listed twice under the same transforms (ties between targets: the first wins) and every link's
    points twice in a row (identical terms from two lanes)."""
    zc, sets, keep = _all_sets()
    S0, A0 = int(zc["S"]), int(zc["A"])
    base = _trajectory(zc["tmat"], S0, A0, 6, seed=7).reshape(S0, 6, 4, 4)
    for name, descs in sets[:3]:
        dup = [descs[0], descs[1], descs[0], descs[2]]
        tm = np.ascontiguousarray(np.concatenate([base[0:1], base[1:2], base[0:1], base[2:3]]).reshape(24, 4, 4),
                                  dtype=np.float32)
        inv = _inverse(tm)
        lp = _link_points(zc, tm, 4, 6, 50, seed=3)
        lp[2] = lp[0]
        lp = np.ascontiguousarray(np.concatenate([lp, lp], axis=1))
        allowed = [[i != j and {i, j} != {0, 2} for j in range(4)] for i in range(4)]
        v, g, w, x = _per_point(dup, tm, inv, 6, lp, allowed)
        m = _margin(v, w >= 0, 0.3)
        assert not (w == 2).any()                                    # the first of two equal targets
        cost, twist, vis, pv, pg, pw, px, evals = _fused(dup, tm, inv, 6, lp, allowed, m)
        inside = (w >= 0) & (v < m)
        assert inside.any() and vis[inside].all(), name
        assert np.array_equal(pv[inside], v[inside]) and np.array_equal(pw[inside], w[inside]), name
        assert np.array_equal(pg[inside], g[inside]), name
        _check_within(cost, twist, _fp64_sum(v, g, w, x, m, 4), name)
        # sources 0 and 2 have the same points and targets: the same terms, so the same twist on targets 1 and 3
        for kw in (dict(cfg_order=1), dict(first=3), dict(first=2, cfg_order=2, shuffle_seed=1)):
            c2, t2 = _fused(dup, tm, inv, 6, lp, allowed, m, **kw)[:2]
            assert np.array_equal(c2, cost) and np.array_equal(t2, twist), (name, kw)


# ---------------------------------------------------------------- 2. signs and zeros
def _translate(t):
    m = np.eye(4, dtype=np.float32)
    m[:3, 3] = t
    return m


def test_sign_convention_on_two_spheres(built_lib):
    """Sphere 0 (r = 0.1) at c0 = (0, -0.1, 0), sphere 1 (r = 0.1) at c1 = (0.2, 0.2, 0); only the points of sphere 1
    are tested, against sphere 0.  One point lies within the margin: x = c1 + (-0.1, 0, 0) = (0.1, 0.2, 0), at
    d = |x - c0| - 0.1 = sqrt(0.1) - 0.1 < m = 0.3 with g = (x - c0) / |x - c0|; the other is beyond it."""
    descs = [hs.sphere_desc(0.1), hs.sphere_desc(0.1)]
    c0, c1 = np.array([0.0, -0.1, 0.0]), np.array([0.2, 0.2, 0.0])
    xf = np.ascontiguousarray(np.stack([_translate(-c0), _translate(-c1)]), dtype=np.float32)     # object -> sub
    inv = np.ascontiguousarray(np.stack([_translate(c0), _translate(c1)]), dtype=np.float32)
    lp = np.zeros((2, 2, 3), np.float32)
    lp[1, 0] = (-0.1, 0.0, 0.0)
    lp[1, 1] = (0.1, 0.0, 0.0)                                    # |x - c0| = sqrt(0.18): d = 0.324 > m = 0.3
    lp[0] = (0.1, 0.0, 0.0)                                       # row 0 is empty: never tested
    allowed = [[False, False], [True, False]]
    m = 0.3
    cost, twist, vis, pv, pg, pw, px, evals = _fused(descs, xf, inv, 1, lp, allowed, m)
    x = np.array([0.1, 0.2, 0.0])
    r = x - c0
    d = np.linalg.norm(r) - 0.1
    g = r / np.linalg.norm(r)
    h = m - d
    assert 0 < h < m
    tau = 2 * h * np.concatenate([g, np.cross(x, g)])
    assert abs(tau[5]) > 1e-3                                     # a moment about the origin, not only a force
    assert cost[0] == pytest.approx(h * h, rel=1e-5)
    assert np.allclose(twist[0, 0], tau, rtol=1e-5, atol=1e-7)   # the target moves: +tau
    assert np.array_equal(twist[0, 1], -twist[0, 0])              # the source moves: -tau, exactly
    assert pw[0, 1, 0] == 0 and not vis[0, 0].any()
    # the twist is the derivative of the cost: moving sphere 0 towards x raises it, moving sphere 1 away lowers it
    def cost_at(dc0, dx):
        return max(m - (np.linalg.norm(x + dx - (c0 + dc0)) - 0.1), 0.0) ** 2
    eps = 1e-6
    for k in range(3):
        dv = np.zeros(3)
        dv[k] = eps
        # sphere 0 translated: its centre moves; sphere 1 translated: its point moves with it
        fd0 = (cost_at(dv, 0 * dv) - cost_at(-dv, 0 * dv)) / (2 * eps)
        fd1 = (cost_at(0 * dv, dv) - cost_at(0 * dv, -dv)) / (2 * eps)
        assert fd0 == pytest.approx(float(twist[0, 0, k]), rel=1e-4, abs=1e-7), k
        assert fd1 == pytest.approx(float(twist[0, 1, k]), rel=1e-4, abs=1e-7), k


def test_far_apart_links_and_empty_rows_cost_exactly_zero(built_lib):
    zc, sets, keep = _all_sets()
    S0, A = int(zc["S"]), int(zc["A"])
    tm = np.ascontiguousarray(zc["tmat"], dtype=np.float32)
    inv = _inverse(tm)
    for name, descs in sets:
        S = len(descs)
        lp = _link_points(zc, tm, S, A, 40, seed=2)
        # every source's points far from every link: each step is skipped by its bounds
        far = np.ascontiguousarray(lp + np.float32(50.0))
        inv_far = inv.copy()
        cost, twist, vis, pv, pg, pw, px, evals = _fused(descs, tm, inv_far, A, far, _allowed_cases(S)["full"], 0.05)
        assert not cost.any() and not twist.any() and not vis.any() and evals == 0, name
        # no allowed pair at all
        cost, twist, vis, pv, pg, pw, px, evals = _fused(descs, tm, inv, A, lp, _allowed_cases(S)["empty"], 1e3)
        assert not cost.any() and not twist.any() and not vis.any() and evals == 0, name


# ---------------------------------------------------------------- 3. the joint gradient of a serial chain
def test_joint_gradient_equals_finite_differences(tmp_path):
    from test_gpu_robot_fp64 import build_robot, joint_values
    from robot_ref import rigid_inverse
    robot, ref, text = build_robot("mixed", tmp_path, dtype=torch.float64, device="cpu")
    J, S = len(robot.joint_names), len(robot.sdf_to_link_name)
    assert J == ref.n_joints and S == len(ref.links)
    lp = robot.link_surface_points(num_points=300, seed=1).numpy()                # [S, K, 3], link frames
    allowed = robot.self_collision_pairs().numpy()
    np.fill_diagonal(allowed, False)
    assert allowed.any()
    qs = joint_values(ref, text, 6, seed=5).astype(np.float64)
    robot.set_joint_configuration(torch.from_numpy(qs))
    twists = robot.joint_twists().numpy()
    moves = robot.joint_moves_link()

    def per_point(q):
        """fp64 (v, g, w, gap, second, x) per (source, point) at joint values q [1, J]; +inf for empty rows."""
        M = ref.object_to_link(q)                                               # [S, 1, 4, 4]
        out = [np.full((S, lp.shape[1]), np.inf) for _ in range(2)]
        g = np.zeros((S, lp.shape[1], 3))
        w = np.full((S, lp.shape[1]), -1)
        gap = np.zeros((S, lp.shape[1]))
        x = np.zeros((S, lp.shape[1], 3))
        for i in range(S):
            W = rigid_inverse(M[i, 0])
            x[i] = lp[i] @ W[:3, :3].T + W[:3, 3]
            js = np.flatnonzero(allowed[i])
            if not len(js):
                continue
            per = ref.evaluate(M, x[i][None])
            vals = np.where(allowed[i][:, None], per["value"][:, 0], np.inf)          # [S, K]
            wi = vals.argmin(axis=0)
            k = np.arange(lp.shape[1])
            out[0][i] = vals[wi, k]
            out[1][i] = np.sort(vals, axis=0)[1]
            g[i] = per["grad"][wi, 0, k]
            w[i] = wi
            gap[i] = per["gap"][wi, 0, k]
        return out[0], g, w, gap, out[1], x

    m, h = None, 2.0 ** -16
    checked = 0
    for a in range(len(qs)):
        v, g, w, gap, second, x = per_point(qs[a:a + 1])
        if m is None:
            m = float(np.quantile(v[np.isfinite(v)], 0.1))
        hinge = np.maximum(m - v, 0.0)
        tau = np.concatenate([g, np.cross(x, g)], axis=-1) * (2.0 * hinge)[..., None]          # [S, K, 6]
        stable = (gap > 1e-3) & (second - v > 1e-3) & (v < m + 1e-2) & (w >= 0)
        for j in range(J):
            qp, qm = qs[a:a + 1].copy(), qs[a:a + 1].copy()
            qp[0, j] += h
            qm[0, j] -= h
            vp, _, wp, _, _, _ = per_point(qp)
            vm, _, wm, _, _, _ = per_point(qm)
            keep = stable & (wp == w) & (wm == w)
            fd = ((np.maximum(m - vp, 0) ** 2 - np.maximum(m - vm, 0) ** 2)[keep]).sum() / (2 * h)
            # the analytic gradient over the same points: +tau to the target, -tau to the source
            tk = np.where(keep[..., None], tau, 0.0)
            tw = np.zeros((S, 6))
            for s in range(S):
                tw[s] = tk[w == s].sum(0) - tk[s].sum(0)
            an = robot.joint_gradient(torch.from_numpy(tw[None]), torch.from_numpy(twists[a:a + 1]),
                                      moves).numpy()[0, j]
            scale = np.abs(tk).sum() * 2 * (1.0 + np.abs(twists[a, j]).max()) + 1e-12
            assert abs(fd - an) <= 1e-5 * scale, (a, j, fd, an, scale)
            checked += int(keep.sum())
    assert checked > 200


# ---------------------------------------------------------------- 4. C ABI refusals and Python rules (no device)
def test_abi_refuses_invalid_self_collision_cost_queries(built_lib):
    near, tri, keep = _table_descs("probe")
    fake = ctypes.c_void_p(1 << 12)           # never dereferenced: every call below fails its argument checks
    L = built_lib
    arr = nat.desc_array([near, near, tri])
    rows3 = (ctypes.c_uint8 * 3)(0b110, 0b101, 0b011)

    def call(descs=arr, n_sdf=3, xf=fake, inv=fake, n_cfg=4, begin=0, count=4, pts=fake, K=100, allowed=rows3,
             margin=0.05, cost=fake, twist=fake):
        return L.pvb_composed_query_self_collision_cost(descs, n_sdf, xf, inv, n_cfg, begin, count, pts, K, allowed,
                                                        margin, cost, twist, None)

    gt = near.copy()
    gt.flags |= nat.PVB_GRID_OOB_GT
    mesh = near.copy()
    mesh.kind = nat.PVB_KIND_MESH
    bad_kind = near.copy()
    bad_kind.kind = 7
    nine = (ctypes.c_uint8 * 9)()
    cases = [dict(descs=None), dict(xf=None), dict(inv=None), dict(pts=None), dict(cost=None), dict(twist=None),
             dict(allowed=None), dict(n_sdf=0), dict(n_cfg=0), dict(begin=-1), dict(count=-1), dict(count=0),
             dict(begin=2, count=3), dict(K=0), dict(K=-1), dict(K=1 << 24),
             dict(allowed=(ctypes.c_uint8 * 3)(0b1110, 0, 0)), dict(allowed=(ctypes.c_uint8 * 3)(0, 0, 0x80)),
             dict(margin=float("nan")), dict(margin=float("inf")), dict(margin=-float("inf")),
             dict(descs=nat.desc_array([near] * 9), n_sdf=9, allowed=nine),
             dict(descs=nat.desc_array([near] * 129), n_sdf=129),
             dict(descs=nat.desc_array([near, mesh, near])), dict(descs=nat.desc_array([near, gt, near])),
             dict(descs=nat.desc_array([near, bad_kind, near]))]
    for kw in cases:
        rc = call(**kw)
        msg = L.pvb_last_error()
        assert rc == PVB_ERR_INVALID and msg.startswith(b"pvb_composed_query_self_collision_cost"), (kw, msg)
    assert b"2^24" in (call(K=1 << 24), L.pvb_last_error())[1]
    assert b"finite" in (call(margin=float("nan")), L.pvb_last_error())[1]
    assert b"empty configuration slab" in (call(count=0), L.pvb_last_error())[1]
    assert b"beyond n_sdf" in (call(allowed=(ctypes.c_uint8 * 3)(0b1000, 0, 0)), L.pvb_last_error())[1]
    assert b"at most 8" in (call(descs=nat.desc_array([near] * 9), n_sdf=9, allowed=nine), L.pvb_last_error())[1]
    assert b"no mesh" in (call(descs=nat.desc_array([near, mesh, near])), L.pvb_last_error())[1]
    assert b"no mesh" in (call(descs=nat.desc_array([near, gt, near])), L.pvb_last_error())[1]


def test_self_collision_cost_shape_rules_raise_before_device_work(monkeypatch):
    import pytorch_volumetric_b200 as pv

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(nat, "compute_device", no_device)
    monkeypatch.setattr(nat, "as_f32_points", no_device)
    comp = pv.ComposedSDF([pv.SphereSDF(0.1), pv.SphereSDF(0.2), pv.SphereSDF(0.3)],
                          pv.Transform3d(matrix=torch.eye(4).repeat(6, 1, 1)))
    ok = torch.ones(3, 3, dtype=torch.bool)
    for shape in ((3, 4), (2, 4, 3), (4, 4, 3), (3, 0, 3), (3, 4, 2), (1, 3, 4, 3), (3, 1 << 24, 3)):
        lp = torch.zeros(1).expand(*shape)
        with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
            comp.query_self_collision_cost(lp, ok, 0.1)
        with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
            comp.self_collision_cost(lp, ok, 0.1)
    lp = torch.zeros(3, 5, 3)
    for bad in (torch.ones(3, 3), torch.ones(3, 4, dtype=torch.bool), np.ones((3, 3), dtype=np.int64)):
        with pytest.raises(ValueError, match="bool matrix"):
            comp.query_self_collision_cost(lp, bad, 0.1)
        with pytest.raises(ValueError, match="bool matrix"):
            comp.self_collision_cost(lp, bad, 0.1)
    for margin in (float("nan"), float("inf"), -math.inf, "x", None, torch.tensor([0.1, 0.2])):
        with pytest.raises(ValueError, match="margin"):
            comp.query_self_collision_cost(lp, ok, margin)
        with pytest.raises(ValueError, match="margin"):
            comp.self_collision_cost(lp, ok, margin)
    for begin, count in ((0, 0), (2, 0), (1, 2), (-1, 1), (0, -1)):
        with pytest.raises(ValueError, match="slab"):
            comp.query_self_collision_cost(lp, ok, 0.1, cfg_begin=begin, cfg_count=count)
    with pytest.raises(ValueError, match="slab"):
        comp.query_self_collision_cost(lp, ok, 0.1, cfg_begin=2)
    # RobotSDF delegates
    from pytorch_volumetric_b200.model_to_sdf import RobotSDF
    robot = RobotSDF.__new__(RobotSDF)
    robot.sdf = comp
    with pytest.raises(ValueError, match=r"\[S, K, 3\]"):
        robot.self_collision_cost(0.1, torch.zeros(2, 5, 3), ok)
    with pytest.raises(ValueError, match="bool matrix"):
        robot.self_collision_cost(0.1, lp, ok.int())
    with pytest.raises(ValueError, match="margin"):
        robot.self_collision_cost(float("nan"), lp, ok)
