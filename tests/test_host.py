"""CPU: host-side logic of the product -- C ABI surface, BVH builder invariants, API mirrors, sharding."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import workloads
from robot_ref import MIXED_URDF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_c_abi_exports_every_declared_symbol(built_lib):
    from pytorch_volumetric_b200 import _native
    header = open(os.path.join(ROOT, "include", "pvb.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(pvb_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    raw = ctypes.CDLL(_native.LIB_PATH)
    for sym in declared:
        assert hasattr(raw, sym), f"{sym} declared in include/pvb.h but not exported by libpvb.so"
    assert declared == set(_native.EXPORTED_SYMBOLS)
    assert built_lib.pvb_sizeof_sdf_desc() == ctypes.sizeof(_native.SdfDesc)
    assert built_lib.pvb_sizeof_bvh4_node() == 128
    assert built_lib.pvb_version() == 100


def test_c_abi_argument_validation_without_gpu(built_lib):
    from pytorch_volumetric_b200 import _native
    d = _native.SdfDesc()
    rc = built_lib.pvb_mesh_query(ctypes.byref(d), None, 10, 3, None, None, None, None, None, None, 0, None)
    assert rc == -1 and b"null" in built_lib.pvb_last_error()
    rc = built_lib.pvb_grid_lookup(ctypes.byref(d), ctypes.c_void_p(16), 10, None, None, None, 0.0, None, None)
    assert rc == -1 and b"empty" in built_lib.pvb_last_error()
    v = np.zeros((3, 3), np.float32)
    f = np.array([[0, 1, 5]], np.int32)
    with pytest.raises(_native.NativeLibraryError, match="out of range"):
        _native.bvh_build(v, f)


def test_no_cpu_fallback_without_gpu():
    """The product path must fail loudly, not fall back, when there is no CUDA device."""
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200._native import NativeLibraryError
    v, f = workloads.fixture_mesh("probe")
    obj = pv.MeshObjectFactory("probe", mesh=(v, f))
    with pytest.raises(NativeLibraryError, match="no CPU fallback"):
        pv.MeshSDF(obj)(torch.zeros(4, 3))
    with pytest.raises(NativeLibraryError):
        pv.SphereSDF(1.0)(torch.zeros(4, 3))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "pytorch_volumetric_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), fn
                assert "liborc_geom" not in src, fn


def _check_bvh(v32, f):
    """Structural invariants of pvb_bvh_build's output: every face once, BFS layout, boxes nest and contain their
    triangles, every node reachable exactly once, traversal stack bound."""
    from pytorch_volumetric_b200 import _native
    nodes_raw, tris, depth = _native.bvh_build(v32, f)
    nodes = nodes_raw.view(np.float32).reshape(-1, 32)
    child = nodes_raw.view(np.int32).reshape(-1, 32)[:, 24:28]
    n_nodes = len(nodes)
    assert n_nodes >= 1
    assert 3 * depth + 2 <= 64
    face_of = tris.view(np.int32)[:, 3]
    assert np.array_equal(np.sort(face_of), np.arange(len(f)))        # a permutation of the faces
    assert np.array_equal(tris[:, [0, 1, 2, 4, 5, 6, 8, 9, 10]].reshape(-1, 3, 3), v32[f[face_of]])
    seen_tri = np.zeros(len(f), dtype=int)
    seen_node = np.zeros(n_nodes, dtype=int)
    seen_node[0] = 1

    def box(node, k):
        return nodes[node, [0 + k, 4 + k, 8 + k]], nodes[node, [12 + k, 16 + k, 20 + k]]

    def node_bounds(i):
        los, his = [], []
        for k in range(4):
            if child[i, k] != -2 ** 31:
                lo, hi = box(i, k)
                los.append(lo); his.append(hi)
        return np.min(los, axis=0), np.max(his, axis=0)

    for i in range(n_nodes):
        for k in range(4):
            c = int(child[i, k])
            if c == -2 ** 31:
                continue
            lo, hi = box(i, k)
            if c >= 0:
                assert c > i, "BFS layout: children come after their parent"
                seen_node[c] += 1
                clo, chi = node_bounds(c)
                assert (clo >= lo).all() and (chi <= hi).all()
            else:
                code = ~c
                first, cnt = code >> 2, (code & 3) + 1
                seen_tri[first:first + cnt] += 1
                tv = tris[first:first + cnt][:, [0, 1, 2, 4, 5, 6, 8, 9, 10]].reshape(-1, 3)
                assert (tv >= lo).all() and (tv <= hi).all()
    assert (seen_tri == 1).all() and (seen_node == 1).all()
    return n_nodes, depth


@pytest.mark.parametrize("name", ["probe", "wrench", "drill"])
def test_bvh_builder_invariants(name, built_lib):
    v, f = workloads.fixture_mesh(name)
    _check_bvh(v.astype(np.float32), f)


def test_bvh_builder_degenerate_inputs(built_lib):
    """Inputs that break naive SAH builders: a single triangle, many coincident triangles (zero-extent centroid
    boxes: no split plane exists), zero-area triangles, a flat sheet (one axis has no extent), a strongly skewed
    size distribution, and a large random soup (depth bound of the wide tree)."""
    rng = np.random.default_rng(0)
    tri = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float32)
    one = np.array([[0, 1, 2]], dtype=np.int32)
    assert _check_bvh(tri, one)[0] == 1
    _check_bvh(tri, np.repeat(one, 1000, axis=0))                                   # 1000 identical triangles
    pts = np.zeros((3, 3), dtype=np.float32)
    _check_bvh(pts, np.repeat(one, 37, axis=0))                                     # all vertices at one point
    line = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2], [3, 3, 3]], dtype=np.float32)
    _check_bvh(line, np.array([[0, 1, 2], [1, 2, 3], [0, 2, 3]], dtype=np.int32))   # zero-area (collinear)
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), indexing="ij"), -1).reshape(-1, 2)
    sheet = np.concatenate([g, np.zeros((len(g), 1))], 1).astype(np.float32)        # flat in z
    idx = np.arange(40 * 40).reshape(40, 40)
    quads = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 4)
    _check_bvh(sheet, np.concatenate([quads[:, [0, 1, 2]], quads[:, [0, 2, 3]]]).astype(np.int32))
    v = rng.normal(size=(3000, 3)).astype(np.float32)
    v[:10] *= 1e4                                                                   # a few huge triangles over many tiny
    _check_bvh(v, rng.integers(0, 3000, size=(5000, 3)).astype(np.int32))
    v = rng.uniform(-1, 1, size=(60_000, 3)).astype(np.float32)
    c = rng.integers(0, 60_000, size=120_000)
    f = np.stack([c, (c + 1) % 60_000, (c + 2) % 60_000], 1).astype(np.int32)
    n_nodes, depth = _check_bvh(v, f)
    assert depth <= 20


def test_grid_helpers_match_port():
    import pytorch_volumetric_b200 as pv
    from oracle import port
    rng = np.array([[-0.067981, 0.095006], [-0.041332, 0.081863], [-0.003716, 0.183718]])
    rng[:, 0] -= 0.1; rng[:, 1] += 0.1
    for res in (0.005, 0.01, 0.02):
        a = pv.get_divisible_range_by_resolution(res, rng)
        b = port.divisible_range(res, rng)
        assert a == b
        ca, pa = pv.get_coordinates_and_points_in_grid(res, a)
        cb, pb = port.grid_coords_and_points(res, b)
        assert all(torch.equal(x, y) for x, y in zip(ca, cb)) and torch.equal(pa, pb)
    assert [len(c) for c in pv.get_coordinates_and_points_in_grid(0.005, pv.get_divisible_range_by_resolution(0.005, rng))[0]] == [74, 66, 78]


def test_transform3d_and_kinematics_match_oracle_restatement(tmp_path):
    import pytorch_volumetric_b200 as pv
    from oracle import tp_pytorch_kinematics as opk
    m = workloads.random_rigid(7, seed=2)
    a, b = pv.Transform3d(matrix=m), opk.Transform3d(matrix=m)
    p = torch.randn(50, 3)
    assert torch.allclose(a.transform_points(p), b.transform_points(p), atol=1e-6)
    assert torch.allclose(a.inverse().get_matrix(), b.inverse().get_matrix(), atol=1e-6)
    assert torch.allclose(a.transform_normals(p), b.transform_normals(p), atol=1e-5)
    assert torch.allclose(a[2:5].get_matrix(), b[2:5].get_matrix())
    assert torch.allclose(a.compose(a.inverse()).get_matrix(), torch.eye(4).repeat(7, 1, 1), atol=1e-6)
    assert a[0].transform_points(p).shape == (50, 3) and a.transform_points(p).shape == (7, 50, 3)
    t = pv.Translate(0.1, 0, 0).stack(pv.Translate(-0.2, 0, 0.2))
    assert len(t) == 2 and torch.allclose(t.get_matrix()[1, :3, 3], torch.tensor([-0.2, 0.0, 0.2]))
    urdf, end = workloads.write_arm(str(tmp_path))
    data = open(urdf).read()
    c1 = pv.build_serial_chain_from_urdf(data, end)
    c2 = opk.build_serial_chain_from_urdf(data, end)
    assert c1.get_joint_parameter_names() == c2.get_joint_parameter_names()
    assert c1.get_frame_names(exclude_fixed=False) == c2.get_frame_names(exclude_fixed=False)
    th = workloads.arm_configurations(6)
    f1 = c1.forward_kinematics(th, end_only=False)
    f2 = c2.forward_kinematics(th, end_only=False)
    for k in f2:
        assert torch.allclose(f1[k].get_matrix(), f2[k].get_matrix(), atol=2e-6), k
    vis = c1.find_frame("link_3").link.visuals[0]
    assert vis.geom_type == "mesh" and vis.geom_param[0] == "link.obj" and vis.geom_param[1] == [3.0, 3.0, 3.0]


def test_mesh_factory_host_side(tmp_path):
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200.meshio import write_obj
    from oracle import port
    v, f = workloads.fixture_mesh("probe")
    path = str(tmp_path / "probe.obj")
    write_obj(path, v, f)
    kw = dict(scale=2.0, vis_frame_pos=(0.01, 0.02, 0.03), vis_frame_rot=(0.1, 0.2, 0.3, 0.9))
    obj = pv.MeshObjectFactory(path, **kw)
    ref = port.MeshPort(path, **kw)
    np.testing.assert_allclose(obj._mesh.vertices, ref.mesh.vertices, atol=1e-15)
    np.testing.assert_allclose(obj.bounding_box(0.1, 0.05), ref.bounding_box(0.1, 0.05), atol=1e-15)
    np.testing.assert_allclose(obj._face_normals, ref.face_normals, atol=1e-12)
    np.testing.assert_allclose(obj.center(), ref.mesh.get_center(), atol=1e-15)
    with pytest.raises(RuntimeError, match="does not exist"):
        pv.MeshObjectFactory(str(tmp_path / "missing.obj"))
    pre = pv.MeshObjectFactory("package://probe.obj", path_prefix=str(tmp_path))
    assert pre.get_mesh_resource_filename() == path
    import pickle
    again = pickle.loads(pickle.dumps(obj))
    np.testing.assert_array_equal(again._mesh.vertices, obj._mesh.vertices)
    assert pv.MeshSDF(obj).surface_bounding_box(padding=0.1).shape == (3, 2)


def test_shard_range_and_gather_single_process():
    from pytorch_volumetric_b200.distributed import shard_range, all_gather_slabs
    for n in (0, 1, 7, 200, 100003):
        for world in (1, 2, 3, 8):
            spans = [shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1
    x = torch.arange(6.).reshape(3, 2)
    assert all_gather_slabs(x, [3]) is x


def _gloo_worker(rank, world, port_no, tmpdir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from pytorch_volumetric_b200 import distributed as pd

    class Sphere:                      # CPU stand-in for an ObjectFrameSDF (host logic only)
        def __call__(self, p):
            r = p.norm(dim=-1)
            return r - 1.0, p / r.unsqueeze(-1)

    pts = torch.randn(2, 103, 3, generator=torch.Generator().manual_seed(0))
    v, g = pd.sharded_query(Sphere(), pts, gather=True)
    v_ref, g_ref = Sphere()(pts)
    ok1 = torch.equal(v, v_ref) and torch.equal(g, g_ref)

    class FakeComposed:                # the configuration-slab contract of ComposedSDF.query
        tsf_batch = (5,)

        def query(self, points, cfg_begin=0, cfg_count=None):
            P = points.reshape(-1, 3).shape[0]
            cfg = torch.arange(cfg_begin, cfg_begin + cfg_count, dtype=torch.float32)
            val = (cfg[:, None] * 1000 + torch.arange(P)[None]).reshape(-1)
            return val, val[:, None].repeat(1, 3)

    class FakeRobot:
        sdf = FakeComposed()

    rv, rg = pd.sharded_robot_query(FakeRobot(), pts[0], gather=True)
    exp = torch.arange(5.)[:, None] * 1000 + torch.arange(103.)[None]
    ok2 = torch.equal(rv, exp) and rg.shape == (5, 103, 3)
    lv, lg, (b, e) = pd.sharded_robot_query(FakeRobot(), pts[0], gather=False)
    ok3 = (b, e) == pd.shard_range(5, rank, world) and lv.shape == (e - b, 103)
    ragged = pd.all_gather_slabs(torch.full((rank + 1, 2), float(rank)), [1, 2])
    ok4 = torch.equal(ragged, torch.tensor([[0., 0.], [1., 1.], [1., 1.]]))
    with open(os.path.join(tmpdir, f"ok{rank}"), "w") as fh:
        fh.write(str(int(ok1 and ok2 and ok3 and ok4)))
    dist.destroy_process_group()


def test_sharding_world_size_2_gloo(tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port_no = s.getsockname()[1]; s.close()
    mp.spawn(_gloo_worker, args=(2, port_no, str(tmp_path)), nprocs=2, join=True)
    assert [open(tmp_path / f"ok{r}").read() for r in range(2)] == ["1", "1"]


def test_bvh_builder_rejects_bad_meshes(built_lib):
    from pytorch_volumetric_b200 import _native
    v = np.zeros((3, 3), np.float32)
    for faces in (np.zeros((0, 3), np.int32), np.array([[0, 1, 5]], np.int32), np.array([[0, -1, 2]], np.int32)):
        with pytest.raises(_native.NativeLibraryError):
            _native.bvh_build(v, faces)


def test_mesh_readers_edge_cases(tmp_path):
    """OBJ: indentation, CRLF, comments, v/vt/vn corner syntax, negative (relative) indices, quads and n-gons as
    fans, vertex colours; binary and ASCII STL; error behaviour."""
    import struct
    from pytorch_volumetric_b200 import meshio
    obj = tmp_path / "m.obj"
    obj.write_text("# comment\r\n"
                   "mtllib x.mtl\r\n"
                   "  v 0 0 0 1.0 0.5 0.25\r\n"
                   "v 1 0 0\r\n"
                   "\tv 1 1 0\r\n"
                   "v 0 1 0\r\n"
                   "vn 0 0 1\r\nvt 0.5 0.5\r\n"
                   "v 0.5 0.5 1\r\n"
                   "g part\r\ns off\r\n"
                   "f 1/1/1 2/1/1 3/1/1 4/1/1\r\n"          # quad -> 2 triangles
                   "f -5//1 -4//1 -1//1\r\n"                # relative indices
                   "f 1 2 3 4 5\r\n")                       # pentagon -> 3 triangles
    v, f = meshio.read_obj(str(obj))
    assert v.shape == (5, 3) and v.dtype == np.float64
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 4], [0, 1, 2], [0, 2, 3], [0, 3, 4]]
    bad = tmp_path / "bad.obj"
    bad.write_text("v 0 0 0\nv 1 0 0\nf 1 2 7\n")
    with pytest.raises(RuntimeError):
        meshio.read_obj(str(bad))
    empty = tmp_path / "empty.obj"
    empty.write_text("v 0 0 0\n")
    with pytest.raises(RuntimeError):
        meshio.read_triangle_mesh(str(empty))
    with pytest.raises(RuntimeError):
        meshio.read_triangle_mesh(str(tmp_path / "mesh.ply"))
    # STL, both encodings, same triangles
    tri = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 0, 1], [1, 0, 1], [0, 1, 1]]], dtype=np.float32)
    b = tmp_path / "b.stl"
    with open(b, "wb") as fh:
        fh.write(b"binary stl".ljust(80, b" ")); fh.write(struct.pack("<I", len(tri)))
        for t in tri:
            fh.write(struct.pack("<3f", 0, 0, 1)); fh.write(t.tobytes()); fh.write(b"\x00\x00")
    a = tmp_path / "a.stl"
    a.write_text("solid s\n" + "".join(
        "facet normal 0 0 1\n outer loop\n" + "".join(f"  vertex {p[0]} {p[1]} {p[2]}\n" for p in t) +
        " endloop\nendfacet\n" for t in tri) + "endsolid s\n")
    for path in (a, b):
        v, f = meshio.read_triangle_mesh(str(path))
        assert np.array_equal(v[f], tri.astype(np.float64))
    # write_obj round trip keeps every bit of the fp64 positions
    vv = np.random.default_rng(0).normal(size=(7, 3))
    ff = np.array([[0, 1, 2], [3, 4, 5], [6, 0, 3]], dtype=np.int32)
    meshio.write_obj(str(tmp_path / "rt.obj"), vv, ff)
    v2, f2 = meshio.read_obj(str(tmp_path / "rt.obj"))
    assert np.array_equal(v2, vv) and np.array_equal(f2, ff)


def test_urdf_chain_mixed_joint_types_match_oracle_restatement():
    """Fixed / revolute / prismatic / continuous joints, rotated origins, non-axis-aligned and unnormalised axes,
    links without visuals, non-mesh visuals, a side branch off the serial path: names, visuals and batched FK agree
    with the oracle's restatement of pytorch_kinematics."""
    import pytorch_volumetric_b200 as pv
    from oracle import tp_pytorch_kinematics as opk
    c1 = pv.build_serial_chain_from_urdf(MIXED_URDF, "tool")
    c2 = opk.build_serial_chain_from_urdf(MIXED_URDF, "tool")
    assert c1.get_joint_parameter_names() == c2.get_joint_parameter_names() == ["j_rev", "j_pris", "j_cont"]
    names = c1.get_frame_names(exclude_fixed=False)
    assert names == c2.get_frame_names(exclude_fixed=False)
    assert not any("side" in n for n in names)
    for n in names:
        v1, v2 = c1.find_frame(n).link.visuals, c2.find_frame(n).link.visuals
        assert [(v.geom_type, v.geom_param) for v in v1] == [(v.geom_type, v.geom_param) for v in v2], n
        for a, b in zip(v1, v2):
            assert torch.allclose(a.offset.get_matrix(), b.offset.get_matrix(), atol=1e-7)
    g = torch.Generator().manual_seed(0)
    th = torch.randn(9, 3, generator=g)
    f1, f2 = c1.forward_kinematics(th, end_only=False), c2.forward_kinematics(th, end_only=False)
    assert set(f1) == set(f2)
    for k in f2:
        assert f1[k].get_matrix().shape == (9, 4, 4)
        assert torch.allclose(f1[k].get_matrix(), f2[k].get_matrix(), atol=2e-6), k
    one1, one2 = c1.forward_kinematics(th[0], end_only=False), c2.forward_kinematics(th[0], end_only=False)
    for k in one2:
        assert torch.allclose(one1[k].get_matrix(), one2[k].get_matrix(), atol=2e-6), k
    assert torch.allclose(c1.forward_kinematics(th, end_only=True).get_matrix(),
                          c2.forward_kinematics(th, end_only=True).get_matrix(), atol=2e-6)


def test_grid_descriptor_from_reference_table_without_gpu():
    """CachedSDF._make_desc (the host half of pvb_grid_lookup's contract) on the reference-built golden table, with
    CPU tensors standing in for device memory: lattice, dtype mode, in-range bounds, index band, pruning margin."""
    from helpers import golden
    from pytorch_volumetric_b200 import sdf as S, _native as nat
    from pytorch_volumetric_b200.voxel import GridView
    z = golden("ref_cachedsdf_probe")
    shape = tuple(int(s) for s in z["table_shape"])
    for ranges, fp32_mode in (([tuple(r) for r in z["ranges"]], False),
                              ([tuple(float(x) for x in r) for r in z["ranges"]], True)):
        c = object.__new__(S.CachedSDF)
        c.ranges = ranges
        val = torch.from_numpy(z["table_val"]).reshape(shape)
        c.voxels = GridView(val, ranges, invalid_value=None)
        c.voxels_grad = torch.from_numpy(z["table_grad"])
        c._table = torch.cat([val.reshape(-1, 1), c.voxels_grad], 1).contiguous()
        c.bb = torch.from_numpy(z["bb"])
        c._cdev = torch.device("cpu")
        c.out_of_bounds_strategy = S.OutOfBoundsStrategy.BOUNDING_BOX
        c.interpolation = "nearest"
        d = c._make_desc()
        assert d.kind == nat.PVB_KIND_GRID and list(d.dims) == list(shape) and d.table == c._table.data_ptr()
        assert bool(d.flags & nat.PVB_GRID_INDEX_FP32) == fp32_mode      # numpy scalars -> fp64 index arithmetic
        assert d.flags & nat.PVB_GRID_PRUNE_OK and not d.flags & nat.PVB_GRID_OOB_GT
        for k in range(3):
            lo, hi = float(ranges[k][0]), float(ranges[k][1])
            assert d.min64[k] == lo and abs(d.res64[k] - (hi - lo) / (shape[k] - 1)) < 1e-15
            assert d.valid_lo[k] >= lo - 1e-7 and d.valid_hi[k] <= hi + 1e-7
            if not fp32_mode:       # fp32 bounds equivalent to the fp64 comparison: never outside the fp64 range
                assert float(d.valid_lo[k]) >= lo and float(d.valid_hi[k]) <= hi
            assert (d.inv_res32[k], d.idx_certain[k]) == tuple(np.float32(x) for x in S.fast_index_band(lo, hi, shape[k]))
            assert d.bb_min[k] == np.float32(z["bb"][k, 0]) and d.bb_max[k] == np.float32(z["bb"][k, 1])
        want = S.grid_prune_margin(val, [r[0] for r in ranges], [r[1] for r in ranges], z["bb"].astype(np.float32))
        assert abs(d.prune_margin - want) < 1e-7


def test_cpulist_parser_and_numa_binding_is_a_noop_without_gpu():
    from pytorch_volumetric_b200 import distributed as pd
    assert pd._parse_cpulist("0-3,8,10-11\n") == {0, 1, 2, 3, 8, 10, 11}
    assert pd._parse_cpulist("") == set()
    assert pd._parse_cpulist("5") == {5}
    # no GPU here: nothing is known about the PCIe root, and the affinity is left alone
    before = os.sched_getaffinity(0) if hasattr(os, "sched_getaffinity") else None
    assert pd.gpu_numa_node(0) is None
    assert pd.bind_to_gpu_numa_node(0) is None
    if before is not None:
        assert os.sched_getaffinity(0) == before


def test_every_declared_symbol_is_documented_in_integration_md():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "pvb.h")).read()
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    names = sorted(set(re.findall(r"\b(pvb_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 31
    missing = [n for n in names if n not in doc]
    assert not missing, missing
