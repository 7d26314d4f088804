"""CPU tier for compositions of many sub-SDFs: 17-128 of them (the MAXS = 128 instantiations of the composed kernels,
transforms past the 64 the point-major kernel keeps in shared memory, the mesh nearest-bound-first loop at and past
32) and more than 128 (the generic per-sub-SDF path of ComposedSDF).

1. The visiting order: hostsim_lib.bit_reversed_order is a permutation for every count 1..128 and follows the rule
   of fill_order (pvb_kernels.cu).
2. The device arithmetic compiled for the host -- composed_consider in the visiting loop of the composed kernels and
   composed_point (the per-pair body of the paired, swept and clearance kernels), with and without the
   nearest-bound-first order -- over grid, mixed grid / primitive and closed-mesh sets, against the fp64 composition of
   tests/composed_ref.py up to classified flips and ties, and bit-identical under the bit-reversed and the index
   order.  Every set holds duplicated sub-SDFs, so the first-index tie rule decides some pairs.
3. ComposedSDF with more than 128 descriptor-bearing sub-SDFs takes the generic path instead of raising, and its
   composition routes walk the slab in chunks of 64 configurations and reduce them as the fused kernels do."""
import contextlib

import numpy as np
import pytest
import torch

import composed_ref as cr
import hostsim_lib as hs
import workloads
from helpers import classify_composed, clearance_reduce, golden, grid_spec, swept_reduce
from oracle import port
from pytorch_volumetric_b200 import _native as nat

COUNTS = [17, 32, 33, 64, 65, 127, 128]
TOL = 1e-5
DUPS = ((0, 2), (1, 3))         # (original, copy): the copy has the original's descriptor and transforms


# ---------------------------------------------------------------- 1. visiting order
def _fill_order_rule(n):
    """fill_order: the indices 0..n-1 sorted by their bit reversal over ceil(log2 n) bits."""
    bits = max(0, (n - 1).bit_length())
    return sorted(range(n), key=lambda s: int(format(s, f"0{bits}b")[::-1], 2) if bits else 0)


@pytest.mark.parametrize("n", range(1, 129))
def test_bit_reversed_order_is_the_fill_order_permutation(n):
    order = hs.bit_reversed_order(n)
    assert sorted(order) == list(range(n))
    assert order == _fill_order_rule(n)
    assert order[0] == 0
    if n & (n - 1) == 0:        # a power of two: the bit-reversal permutation itself, its own inverse
        assert [order[s] for s in order] == list(range(n))


# ---------------------------------------------------------------- 2. host build of the device arithmetic
_SHARED = {}


def _parts():
    """Descriptors (host memory) and fp64 specs of the sub-SDF kinds, and one interior point of each (its frame)."""
    if _SHARED:
        return _SHARED
    import pytorch_volumetric_b200 as pv
    z = golden("ref_cachedsdf_probe")
    shape = tuple(int(s) for s in z["table_shape"])
    grid, (cached,) = hs.grid_desc(torch.from_numpy(z["table_val"]).reshape(shape), torch.from_numpy(z["table_grad"]),
                                   [tuple(r) for r in z["ranges"]], z["bb"])
    gs = grid_spec(cached)
    k = np.unravel_index(np.argmin(gs["val"]), gs["val"].shape)
    g_inside = gs["lo"] + np.array(k) * (gs["hi"] - gs["lo"]) / (np.array(gs["val"].shape) - 1)
    prims = [pv.SphereSDF(0.012), pv.BoxSDF([0.03, 0.012, 0.02]), pv.CylinderSDF(0.01, 0.035)]
    v, f = workloads.bumpy_sphere(16, 9, radius=0.02)
    obj = pv.MeshObjectFactory("bumpy", mesh=(v, f))
    assert obj.is_closed
    mesh, keep = hs.mesh_desc(obj)
    _SHARED.update(
        grid=(grid, gs, g_inside), keep=(cached, keep, prims),
        # interior points off the centres, where a gradient is well defined (one nearest face, off the axis)
        prims=[(p.native_desc("cpu"), cr.primitive_spec(p.native_desc("cpu")), np.array(c)) for p, c in
               zip(prims, [(0.004, 0.002, 0.001), (0.002, 0.003, 0.001), (0.004, 0.002, 0.003)])],
        mesh=(mesh, cr.mesh_spec(port.MeshPort(vertices=v, faces=f)), np.array([0.003, 0.002, 0.001])))
    return _SHARED


def _set(kind, S):
    """[(desc, spec, interior point)] * S of one kind: 'grid' (the golden probe table), 'mixed' (the probe with a
    sphere, a box and a cylinder in turn) or 'mesh' (a closed bumpy sphere)."""
    p = _parts()
    cycle = {"grid": [p["grid"]], "mixed": [p["grid"]] + p["prims"], "mesh": [p["mesh"]]}[kind]
    members = [cycle[s % len(cycle)] for s in range(S)]
    for a, b in DUPS:
        if b < S:
            members[b] = members[a]
    return members


def _transforms(S, A, seed):
    """(S, A, 4, 4) fp32 object->sub-frame transforms, distinct per (sub-SDF, configuration), with the DUPS copies."""
    tm = workloads.random_rigid(S * A, seed=seed, t_range=0.06).numpy().reshape(S, A, 4, 4)
    for a, b in DUPS:
        tm[b] = tm[a]
    return tm


def _points(members, tm, n, seed):
    """A uniform cloud around the set and, for every sub-SDF, its interior point under configuration 0's transform,
    so that every sub-SDF that is not a copy wins somewhere."""
    cloud = np.random.default_rng(seed).uniform(-0.1, 0.1, (n, 3))
    inner = [np.linalg.solve(tm[s, 0].astype(np.float64), np.append(c, 1.0))[:3] for s, (_d, _sp, c) in
             enumerate(members)]
    return np.concatenate([cloud, np.array(inner)]).astype(np.float32)


def _assert_matches_fp64(v, g, w, members, tm, pts, ref, what):
    rv, rg, rw, allv, _allg = ref
    S, A = tm.shape[:2]
    P = len(pts)
    v, g, w = v.reshape(A, P), g.reshape(A, P, 3), w.reshape(A, P)
    specs = [sp for _d, sp, _c in members]
    if specs[0]["kind"] == "mesh":
        bad_v, bad_g, bad_w, rep = cr.mesh_mismatch(v, g, w, ref, TOL, coord_scale=0.2)
        assert bad_v == 0 and bad_g == 0 and bad_w == 0, (what, rep)
        exceed = np.zeros((A, P), bool)
    else:
        n_ex, n_un, rep = classify_composed(v, g, rv, rg, specs, tm, pts, TOL)
        assert n_un == 0, (what, rep)
        assert n_ex <= 5e-3 * A * P, (what, rep)
        exceed = (np.abs(v - rv) > TOL) | (np.abs(g - rg).max(-1) > TOL)
    # `which` names an argmin within the tolerance (flips aside), and the first of the sub-SDFs attaining its value
    wv = np.take_along_axis(allv, w[None].astype(np.int64), 0)[0]
    assert ((np.abs(wv - rv) <= TOL) | exceed).all(), what
    for a, b in DUPS:
        assert not (w == b).any(), (what, "copy", b)
    assert (w[~exceed] == rw[~exceed]).mean() > 0.999, what


@pytest.mark.parametrize("kind", ["grid", "mixed", "mesh"])
@pytest.mark.parametrize("S", COUNTS)
def test_host_composition_equals_fp64_in_any_order(S, kind, oracle_lib):
    A = 2
    members = _set(kind, S)
    descs = [d for d, _s, _c in members]
    tm = _transforms(S, A, seed=S)
    pts = _points(members, tm, 300 if kind == "mesh" else 600, seed=S)
    P = len(pts)
    xf = tm.reshape(S * A, 4, 4)
    ref = cr.compose([sp for _d, sp, _c in members], tm, pts, per_sub=True)
    # the fp64 argmin covers nearly every sub-SDF but the copies, among them the last one visited in either order and
    # sub-SDF 31 (the last bit of the nearest-bound-first loop's mask): each one decides some pairs
    won = set(np.unique(ref[2]).tolist())
    assert not won & {b for _a, b in DUPS} and len(won) >= 0.9 * (S - len(DUPS)), (kind, len(won))
    assert {hs.bit_reversed_order(S)[-1], S - 1, min(31, S - 1)} <= won, (kind, won)

    # composed_consider in the visiting loop of the composed kernels (kMesh, kExt instantiation), bit-reversed order
    got = hs.composed(descs, xf, A, pts, ext=True)
    _assert_matches_fp64(*got, members, tm, pts, ref, (S, kind, "composed"))
    runs = {"index order": hs.composed(descs, xf, A, pts, order=range(S), ext=True)}
    if kind != "mixed":        # the kMesh, non-kExt instantiation takes grids and meshes only
        runs["hostsim"] = hs.composed(descs, xf, A, pts)
    # composed_point (paired host build) on the same points for every configuration: the fixed order, and the
    # nearest-bound-first loop where it applies (n_sdf <= 32; past that the fixed order runs)
    shared = np.broadcast_to(pts, (A, P, 3))
    for nearest_first in (1, 0):
        for name, order in (("bit-reversed", None), ("index order", range(S))):
            runs[f"composed_point {name} nf={nearest_first}"] = hs.sim_paired(descs, xf, A, shared, order=order,
                                                                              nearest_first=nearest_first)
    for name, r in runs.items():
        for a, b, part in zip(r, got, ("val", "grad", "which")):
            assert np.array_equal(a, b), (S, kind, name, part, int((a != b).reshape(len(a), -1).any(-1).sum()))


@pytest.mark.parametrize("kind", ["grid", "mixed", "mesh"])
@pytest.mark.parametrize("S", [17, 33, 65, 128])
def test_identical_copies_report_the_first(S, kind):
    """S copies of one sub-SDF at one pose: every pair reports sub-SDF 0, with the value of the single sub-SDF."""
    members = _set(kind, 1) * S
    descs = [d for d, _s, _c in members]
    tm = np.repeat(workloads.random_rigid(1, seed=5, t_range=0.06).numpy()[:, None], S, axis=0)
    pts = _points(members[:1], tm[:1], 200, seed=1)
    one = hs.composed(descs[:1], tm[0], 1, pts, ext=True)
    for nearest_first in (1, 0):
        for order in (None, range(S)[::-1]):
            for got in (hs.composed(descs, tm.reshape(S, 4, 4), 1, pts, order=order, ext=True),
                        hs.sim_paired(descs, tm.reshape(S, 4, 4), 1, pts[None], order=order,
                                      nearest_first=nearest_first)):
                assert (got[2] == 0).all(), (S, kind, nearest_first)
                assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1]), (S, kind, nearest_first)


# ---------------------------------------------------------------- 3. more than 128 sub-SDFs: the generic path
def test_more_than_128_sub_sdfs_take_the_generic_path(monkeypatch):
    import pytorch_volumetric_b200 as pv
    # no device: the route is decided before any device work, and the generic path itself is recorded, not run
    monkeypatch.setattr(nat, "compute_device", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    for S, generic in ((128, False), (129, True), (200, True)):
        comp = pv.ComposedSDF([pv.SphereSDF(0.01 + 0.001 * s) for s in range(S)],
                              pv.Transform3d(matrix=workloads.random_rigid(S * 3, seed=S)))
        arr, needs_mesh = comp._native_descs(None)
        assert (arr is None) == generic and not needs_mesh, S
        if not generic:
            continue
        calls = []

        def fake(p, cfg_begin, cfg_count, n_cfg, return_which, paired=False, _calls=calls):
            _calls.append((cfg_begin, cfg_count, n_cfg, paired))
            P = p.shape[0] // cfg_count if paired else p.shape[0]
            out = (torch.zeros(cfg_count * P), torch.zeros(cfg_count * P, 3), torch.zeros(cfg_count * P, dtype=torch.int32))
            return out if return_which else out[:2]
        monkeypatch.setattr(comp, "_generic_query", fake)
        pts = torch.zeros(2, 5, 3)
        assert comp(pts)[0].shape == (3, 2, 5)
        assert comp.swept(pts)[0].shape == (2, 5)
        assert comp.clearance(pts)[0].shape == (3, 2)
        assert comp.paired(torch.zeros(3, 5, 3))[0].shape == (3, 5)
        assert comp.paired_clearance(torch.zeros(3, 2, 5, 3))[0].shape == (3, 2)
        assert comp.collision_cost(pts, 0.1)[1].shape == (3, 2, S, 6)
        assert comp.paired_collision_cost(torch.zeros(3, 2, 5, 3), 0.1)[1].shape == (3, 2, S, 6)
        assert calls == [(0, 3, 3, False)] * 3 + [(0, 3, 3, True)] * 2 + [(0, 3, 3, False), (0, 3, 3, True)], \
            (S, calls)
        with pytest.raises(NotImplementedError, match="128"):
            comp.query_into(pts, [(torch.zeros(30), torch.zeros(30, 3))])


def _quarters(rng, lo, hi, shape):
    return torch.from_numpy(rng.integers(lo, hi, shape) / 4).float()


@pytest.mark.parametrize("n_cfg, slabs", [(1, [(0, 1)]), (63, [(0, 63)]), (64, [(0, 64)]), (65, [(0, 65), (1, 63)]),
                                          (129, [(0, 129), (30, 70), (64, 65)])])
def test_generic_composition_chunks_and_reductions(monkeypatch, n_cfg, slabs):
    """The composition routes of a set the fused kernels do not take, with `_generic_query` faked on the CPU: each
    form's chunks of 64 configurations of its slab, in ascending order, and its reduction of the chunks' results.
    The fake's results come from seeded tables, one for the shared cloud and one for the paired blocks: values from
    nine multiples of 1/4, some zeros negative, so that the minima over configurations and over points meet ties;
    gradients and points are multiples of 1/4 too, so every fp64 hinge term and sum below is exact."""
    import pytorch_volumetric_b200 as pv
    monkeypatch.setattr(nat, "compute_device", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    S, n_seg, N, m = 129, 3, 4, 1.0
    comp = pv.ComposedSDF([pv.SphereSDF(0.01) for _ in range(S)], None)
    comp.set_transforms(pv.Transform3d(matrix=workloads.random_rigid(S * n_cfg, seed=n_cfg)), batch_dim=(n_cfg,))
    rng = np.random.default_rng(n_cfg)
    tables = {}
    for paired in (False, True):
        v = _quarters(rng, -3, 6, (n_cfg, n_seg * N))
        v[(v == 0) & torch.from_numpy(rng.random(v.shape) < 0.5)] = -0.0
        tables[paired] = (v, _quarters(rng, -4, 5, (n_cfg, n_seg * N, 3)),
                          torch.from_numpy(rng.integers(0, S, (n_cfg, n_seg * N))).int())
    calls = []

    def fake(p, cfg_begin, cfg_count, n_cfg_, return_which, paired=False):
        calls.append((cfg_begin, cfg_count, n_cfg_, paired))
        P = p.shape[0] // cfg_count if paired else p.shape[0]
        assert return_which
        return tuple(t[cfg_begin:cfg_begin + cfg_count, :P].flatten(0, 1) for t in tables[paired])
    monkeypatch.setattr(comp, "_generic_query", fake)

    for begin, count in slabs:
        rows = slice(begin, begin + count)
        chunks = [(c0, min(64, begin + count - c0), n_cfg) for c0 in range(begin, begin + count, 64)]
        cloud = _quarters(rng, -4, 5, (n_seg, N, 3))
        own = _quarters(rng, -4, 5, (count, n_seg, N, 3))
        flat = {paired: tuple(t[rows].flatten(0, 1) for t in tables[paired]) for paired in (False, True)}

        def run(fn, *args):
            calls.clear()
            out = fn(*args, cfg_begin=begin, cfg_count=count)
            return out, list(calls)

        out, got = run(lambda p, **kw: comp.query_swept(p, return_which=True, **kw), cloud.reshape(-1, 3))
        assert got == [(*c, False) for c in chunks], (begin, count, got)
        for a, b in zip(out, swept_reduce(*flat[False], count, begin)):
            assert torch.equal(a, b), (begin, count, "swept")
        for paired, pts in ((False, cloud), (True, own)):
            fn = comp.query_paired_clearance if paired else comp.query_clearance
            out, got = run(lambda p, **kw: fn(p, return_which=True, **kw), pts)
            assert got == [(*c, paired) for c in chunks], (begin, count, paired, got)
            for a, b in zip(out, clearance_reduce(*flat[paired], count, n_seg)):
                assert torch.equal(a, b), (begin, count, paired, "clearance")

            fn = comp.query_paired_collision_cost if paired else comp.query_collision_cost
            (cost, twist), got = run(fn, pts, m)
            assert got == [(*c, paired) for c in chunks], (begin, count, paired, got)
            v, g, w = (t.double().numpy().reshape(count, n_seg, N, -1) for t in flat[paired])
            x = np.broadcast_to(pts.double().numpy(), (count, n_seg, N, 3))
            ref_cost = np.zeros((count, n_seg))
            ref_twist = np.zeros((count, n_seg, S, 6))
            for a, b, k in np.ndindex(count, n_seg, N):
                h = max(m - v[a, b, k, 0], 0.0)
                ref_cost[a, b] += h * h
                ref_twist[a, b, int(w[a, b, k, 0])] += 2 * h * np.concatenate([g[a, b, k], np.cross(x[a, b, k],
                                                                                                    g[a, b, k])])
            assert torch.equal(cost, torch.from_numpy(ref_cost).float().reshape(-1)), (begin, count, paired)
            assert torch.equal(twist, torch.from_numpy(ref_twist).float().reshape(-1, S, 6)), (begin, count, paired)
