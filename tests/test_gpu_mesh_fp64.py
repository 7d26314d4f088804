"""GPU: MeshSDF / ObjectFactory.object_frame_closest_point and the LOOKUP_GT_SDF grid lookup against the fp64 mesh
(tests/mesh_ref.py) on every launch route -- unbinned, binned (sort_hist / sort_scan / sort_scatter, the walk over
binned records, unpermute), the winding pass, the chunked host pipeline and the grid kernels' tree walk -- for every
output: closest point, signed distance, gradient and normal.  Every difference beyond the bounds of mesh_ref must fall
in a class it names (closest-feature tie, shell edge, sign margin); binned results equal unbinned ones bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mesh_ref as mr
import workloads
from helpers import cached_from_golden, golden, pv_factory

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (1, 3, 32767, 32768, 32769, 100003)          # binning starts at 2^15 points
BIG = (1 << 21) + 3
SEED = 5
# (mesh, mode): parity and winding on every closed mesh, the diagonal ray on closed meshes (axis_ray_when_closed=False),
# the open mesh's own diagonal ray
CONFIGS = [("probe", "parity"), ("probe", "winding"), ("probe", "ray"), ("wrench", "parity"),
           ("drill", "parity"), ("drill", "winding"), ("drill", "ray"), ("scene_overlap", "parity"),
           ("scene_overlap", "winding"), ("bumpy10k", "parity"), ("bumpy10k", "winding")]
FULL = ("probe", "wrench", "scene_overlap")          # checked on every point; the others on a fixed subset
_CACHE = {}


def mesh_obj(name, mode="parity"):
    import pytorch_volumetric_b200 as pv
    if name == "bumpy10k":
        v, f = workloads.bumpy_sphere(100, 51)
        obj = pv.MeshObjectFactory(name, mesh=(v, f), ray_seed=SEED)
    else:
        obj = pv_factory(name, ray_seed=SEED)
    obj.sign_mode = "winding" if mode == "winding" else "parity"
    obj.axis_ray_when_closed = mode != "ray"
    return obj


def mesh_points(name):
    """(points [N, 3] fp32, cluster mask): the mixed set of mesh_ref.mixed_points; every size is a prefix, so a
    point's index in the call -- the seed of its ray -- is the same in every size.  The open mesh also gets points
    whose ray grazes its boundary."""
    key = ("pts", name)
    if key not in _CACHE:
        obj = mesh_obj(name)
        v, f = obj._mesh.vertices, obj._mesh.triangles
        extra = None if obj.is_closed else mr.grazing_points(obj, 4000, seed=3)
        _CACHE[key] = mr.mixed_points(v, f, BIG if name == "bumpy10k" else SIZES[-1], seed=17, extra=extra)
    return _CACHE[key]


def subset(name, n, cluster):
    """Rows of a size-n call compared with fp64: all of them for the small meshes; otherwise the first and last 2 000,
    a stride of about 250 rows and every cluster member (one distinct point)."""
    if name in FULL:
        return np.arange(n)
    rows = np.concatenate([np.arange(min(n, 2000)), np.arange(max(0, n - 2000), n),
                           np.arange(0, n, max(1, n // 250)), np.nonzero(cluster[:n])[0]])
    return np.unique(rows)


def sizes(name):
    return SIZES + ((BIG,) if name == "bumpy10k" else ())


def reference(name, mode):
    """(rows, fp64 query of those rows) for the union of every size's subset."""
    key = ("ref", name, mode)
    if key not in _CACHE:
        pts, cluster = mesh_points(name)
        rows = np.unique(np.concatenate([subset(name, n, cluster) for n in sizes(name) if n <= len(pts)]))
        gkey = ("geo", name)
        ref_obj = _CACHE.setdefault(("mesh_ref", name), mr.MeshRef(mesh_obj(name)))
        if gkey not in _CACHE:
            _CACHE[gkey] = ref_obj.geometry(pts[rows], winding=ref_obj.closed)
        sign = "winding" if mode == "winding" else "parity"
        _CACHE[key] = rows, ref_obj.query(pts[rows], sign=sign, idx=rows, geo=_CACHE[gkey])
    return _CACHE[key]


def run(obj, pts):
    import pytorch_volumetric_b200 as pv
    q = obj.object_frame_closest_point(pts, compute_normal=True)
    v, g = pv.MeshSDF(obj)(pts)
    assert torch.equal(v, q.distance) and torch.equal(g, q.gradient)       # the call without the closest point
    return [t.cpu().numpy() for t in (q.closest, q.distance, q.gradient, q.normal)]


def check_fp64(name, mode, out, n, report):
    rows, ref = reference(name, mode)
    pts, cluster = mesh_points(name)
    want = subset(name, n, cluster)
    pos = np.searchsorted(rows, want)
    assert np.array_equal(rows[pos], want)
    c, d, g, nr = (x[want] for x in out)
    excuse = None
    if mode == "ray":        # a closed mesh's diagonal ray: its edge margin where a sign differs
        ref_obj = _CACHE[("mesh_ref", name)]
        excuse = lambda r: ref_obj.ray_grazes(pts[want[r]], want[r])
    rep, bad = mr.compare(ref, c, d, g, nr, sub=pos, sign_excuse=excuse)
    assert all(len(b) == 0 for b in bad.values()), (name, mode, n, {k: want[b[:8]] for k, b in bad.items() if len(b)},
                                                    rep)
    report.append((name, mode, n, rep))


def _print(report):
    for name, mode, n, rep in report:
        print(f"{name:14s} {mode:8s} n={n:8d} err/bound value {rep['value']:.3f} closest {rep.get('closest', 0):.3f} "
              f"grad {rep['grad']:.3f}  excused {rep['classes']}")


@pytest.mark.parametrize("name,mode", CONFIGS)
def test_every_output_vs_fp64_on_every_route(name, mode):
    """Every size from 1 point to past the binning threshold (and 2^21 + 3 on the 10k-face sphere), forward and
    reversed: each output against fp64, and the reversed call against the forward one -- bit for bit where the answer
    does not depend on the point's index (closed meshes with the axis walk, the winding number), on |d|, the closest
    point and the normal where the ray is seeded by it."""
    obj = mesh_obj(name, mode)
    pts, _ = mesh_points(name)
    seeded = mode == "ray" or not obj.is_closed
    report = []
    for n in sizes(name):
        p = torch.from_numpy(pts[:n]).cuda()
        out = run(obj, p)
        check_fp64(name, mode, out, n, report)
        rev = run(obj, p.flip(0))
        back = [x[::-1] for x in rev]
        if seeded:
            assert np.array_equal(np.abs(back[1]), np.abs(out[1]))
            assert np.array_equal(back[0], out[0]) and np.array_equal(back[3], out[3])
        else:
            for a, b in zip(back, out):
                assert np.array_equal(a, b)
    _print(report)


_CHILD = """
import sys, numpy as np, torch
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_mesh_fp64 as t
out = {{}}
for name, mode in t.CONFIGS:
    pts, _ = t.mesh_points(name)
    obj = t.mesh_obj(name, mode)
    for n in (32768, len(pts)):
        out[(name, mode, n)] = t.run(obj, torch.from_numpy(pts[:n]).cuda())
torch.save(out, {out!r})
"""


@pytest.mark.parametrize("env", [{"PVB_SORT_QUERIES": "0"}, {"PVB_SORT_BITS": "4"}], ids=["unbinned", "bits4"])
def test_binned_equals_unbinned_bit_for_bit(env, tmp_path):
    """Every output of every configuration at 2^15 and the largest size equals, bit for bit, the result of a process
    that does not bin (PVB_SORT_QUERIES=0) or bins into 16^3 cells (PVB_SORT_BITS=4: 4 096 cells, one uint4 per scan
    thread).  The knobs are read once per process, hence the child."""
    res = str(tmp_path / "out.pt")
    flags = ["-s"] if sys.flags.no_user_site else []
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), out=res)
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    other = torch.load(res, weights_only=False)
    for (name, mode, n), outs in other.items():
        pts, _ = mesh_points(name)
        mine = run(mesh_obj(name, mode), torch.from_numpy(pts[:n]).cuda())
        for k, (a, b) in enumerate(zip(mine, outs)):
            assert np.array_equal(a, b), (name, mode, n, k, np.argwhere(a != b)[:5])


@pytest.mark.parametrize("name", ["probe", "drill"])
def test_host_pipeline_equals_device_call_and_fp64(name, monkeypatch):
    """A host fp32 batch of 100 003 points streamed in chunks of 40 000 (two binned chunks, an unbinned tail of
    20 003) and of 32 768 (three binned chunks, a tail of 1 699): the same bits as the device call, with and without
    the normal and through MeshSDF.__call__, and within the fp64 bounds.  Every query is answered per point, so a
    chunk launched over more rows than it holds (stale rows of an earlier chunk) would leave those outputs unchanged:
    the lengths the chunks are launched with are checked directly."""
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import _native as nat
    obj = mesh_obj(name)
    pts, _ = mesh_points(name)
    host = torch.from_numpy(pts)
    dev = obj.object_frame_closest_point(host.cuda(), compute_normal=True)
    dev = [t.cpu() for t in dev]
    L = nat.lib()
    launches = []
    native_query = L.pvb_mesh_query

    def counted(desc, p, n, *rest):
        launches.append(int(n))
        return native_query(desc, p, n, *rest)

    monkeypatch.setattr(L, "pvb_mesh_query", counted)
    report = []
    try:
        obj.host_pipeline_min_points = 1000
        for chunk in (40000, 32768):
            obj.host_pipeline_chunk = chunk
            full = [chunk] * (len(pts) // chunk) + [len(pts) % chunk]     # [40000, 40000, 20003], [32768 x 3, 1699]
            launches.clear()
            q = obj.object_frame_closest_point(host, compute_normal=True)
            assert launches == full, (chunk, launches)
            assert q.distance.is_pinned()
            for a, b in zip(dev, q):
                assert torch.equal(a, b)
            launches.clear()
            q0 = obj.object_frame_closest_point(host)
            assert launches == full, (chunk, launches)
            assert q0.normal is None
            for a, b in zip(dev[:3], q0[:3]):
                assert torch.equal(a, b)
            launches.clear()
            v, g = pv.MeshSDF(obj)(host)
            assert launches == full, (chunk, launches)
            assert torch.equal(v, dev[1]) and torch.equal(g, dev[2])
            check_fp64(name, "parity", [t.numpy() for t in q], len(pts), report)
        assert obj._pipe_state is not None
    finally:
        del obj.host_pipeline_min_points, obj.host_pipeline_chunk
    _print(report)


# ------------------------------------------------------------------ LOOKUP_GT_SDF grids
def _gt_grid(name, tmp_path):
    import pytorch_volumetric_b200 as pv
    if name == "probe":
        c = cached_from_golden(golden("ref_cachedsdf_probe"), "probe", tmp_path,
                               out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    else:
        obj = mesh_obj(name)
        c = pv.CachedSDF(name, 0.002, obj.bounding_box(padding=0.006), pv.MeshSDF(obj), device="cuda",
                         cache_path=str(tmp_path / "wrench.pkl"), clean_cache=True,
                         out_of_bounds_strategy=pv.OutOfBoundsStrategy.LOOKUP_GT_SDF)
    assert c.native_desc("cuda").flags & 2                  # PVB_GRID_OOB_GT: the tree walk runs in the kernel
    assert not c.native_desc("cuda").flags & 1              # fp64 index arithmetic (numpy range)
    return c


def _keys(c, p):
    """The reference's nearest-voxel key (round((p - min) / res) in fp64), -1 out of range."""
    shape = np.array(c.voxels.shape)
    lo = np.array([float(min(r)) for r in c.ranges])
    hi = np.array([float(max(r)) for r in c.ranges])
    res = (hi - lo) / (shape - 1)
    p = p.astype(np.float64)
    inb = np.all((p >= lo) & (p <= hi), axis=1)
    k = np.clip(np.rint((p - lo) / res), 0, shape - 1).astype(np.int64)
    return np.where(inb, (k[:, 0] * shape[1] + k[:, 1]) * shape[2] + k[:, 2], -1)


@pytest.mark.parametrize("name", ["probe", "wrench"])
def test_lookup_gt_grid_vs_table_and_fp64(name, tmp_path):
    """n = 0..3 (mod 4), as an aligned tensor (grid_lookup_vec4_kernel<true> plus the scalar tail) and as a view one
    point into a buffer (grid_lookup_scalar_kernel<true> for every point): in-range points are exact gathers of the
    table, out-of-range ones the fp64 mesh with the ray seeded by the point's index in the call; outside_surface and
    voxel_keys follow the same keys.  The wrench set includes points whose ray grazes its open boundary."""
    c = _gt_grid(name, tmp_path)
    table = c._table.cpu().numpy()
    obj = c.gt_sdf.obj_factory
    ref_obj = mr.MeshRef(obj)
    lo = np.array([float(min(r)) for r in c.ranges])
    hi = np.array([float(max(r)) for r in c.ranges])
    rng = np.random.default_rng(4)
    base = rng.uniform(lo - 0.5 * (hi - lo), hi + 0.5 * (hi - lo), (6004, 3)).astype(np.float32)
    if not obj.is_closed:
        base[1::3] = mr.grazing_points(obj, len(base[1::3]), seed=9, t_range=(0.02, 0.05))
    inb_all = _keys(c, base) >= 0
    oob_all = np.nonzero(~inb_all)[0]
    ref_all = ref_obj.query(base[oob_all], idx=oob_all)        # every size is a prefix: the same index in the call
    report = []
    for n in (6001, 6002, 6003, 6004):
        for offset in (0, 1):
            buf = torch.zeros(n + offset, 3, device="cuda")
            buf[offset:] = torch.from_numpy(base[:n]).cuda()
            p = buf[offset:]
            assert (p.data_ptr() % 16 == 0) == (offset == 0)
            val, grad = (t.cpu().numpy() for t in c(p))
            keys = c.voxel_keys(p).cpu().numpy()
            outside = c.outside_surface(p).cpu().numpy()
            want = _keys(c, base[:n])
            assert np.array_equal(keys, want)
            inb = want >= 0
            assert np.array_equal(val[inb], table[want[inb], 0]) and np.array_equal(grad[inb], table[want[inb], 1:])
            oob = np.nonzero(~inb)[0]
            rep, bad = mr.compare(ref_all, None, val[oob], grad[oob], sub=np.searchsorted(oob_all, oob))
            assert all(len(b) == 0 for b in bad.values()), (n, offset, {k: oob[b[:8]] for k, b in bad.items()}, rep)
            report.append((name, f"grid+{offset}", n, rep))
            assert np.array_equal(outside, np.where(inb, val > 0, True))
    _print(report)
