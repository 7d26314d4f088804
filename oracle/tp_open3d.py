"""Restatement of the slice of Open3D that the reference's SDF path calls.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Open3D is a third-party dependency of the reference that is NOT vendored under
the reference and is unpinned (pyproject.toml:54-61, "open3d").  The
published behaviour of the calls made at the sites below is restated; nothing
here was checked against a real Open3D build ("parity unpinned" at this
boundary, see DESIGN.md):

  o3d.io.read_triangle_mesh                      src/pytorch_volumetric/sdf.py:103
  TriangleMesh.transform / rotate / translate    sdf.py:107-113
  o3d.geometry.get_rotation_matrix_from_quaternion   sdf.py:111
  o3d.t.geometry.TriangleMesh.from_legacy        sdf.py:116
  o3d.t.geometry.RaycastingScene.add_triangles / compute_closest_points /
      count_intersections                        sdf.py:117-118, 134, 153
  TriangleMesh.compute_triangle_normals / triangle_normals   sdf.py:119-120
  TriangleMesh.get_axis_aligned_bounding_box     sdf.py:81-83
  TriangleMesh.get_center                        sdf.py:95
  TriangleMesh.sample_points_uniformly           sdf.py:654
  o3d.utility.random.seed                        sdf.py:646
"""
import os
import struct
import types

import numpy as np

from oracle import _geom

# 'brute' (parity checker) or 'bvh' (timed CPU baseline); see geom.c
QUERY_METHOD = "brute"

_global_seed = [None]


def _seed(s):
    _global_seed[0] = int(s)
    _engine[0] = None


_engine = [None]


def _uniform_doubles(n):
    """std::uniform_real_distribution<double>(0,1) over a std::mt19937 engine
    (libstdc++ generate_canonical: two 32-bit draws per double), which is what
    Open3D's utility::random::UniformRealGenerator<double> wraps."""
    if _engine[0] is None:
        seed = _global_seed[0]
        if seed is None:
            seed = int.from_bytes(os.urandom(4), "little")
        # RandomState(int) seeds with init_genrand(seed) == std::mt19937(seed)
        _engine[0] = np.random.RandomState(seed)
    raw = _engine[0]._bit_generator.random_raw(2 * n).astype(np.float64)
    r = (raw[0::2] + raw[1::2] * 4294967296.0) / 18446744073709551616.0
    r[r >= 1.0] = np.nextafter(1.0, 0.0)
    return r


class _AABB:
    def __init__(self, lo, hi):
        self._lo, self._hi = lo, hi

    def get_min_bound(self):
        return self._lo.copy()

    def get_max_bound(self):
        return self._hi.copy()


class _PointCloud:
    def __init__(self, points=None):
        self.points = points
        self.normals = None


class TriangleMesh:
    """Legacy (fp64 vertices, int triangles) triangle mesh."""

    def __init__(self, vertices=None, triangles=None):
        self.vertices = np.zeros((0, 3)) if vertices is None else np.array(vertices, dtype=np.float64)
        self.triangles = np.zeros((0, 3), np.int32) if triangles is None else np.array(triangles, dtype=np.int32)
        self.triangle_normals = np.zeros((0, 3))

    def transform(self, m):
        m = np.asarray(m, dtype=np.float64)
        v = self.vertices @ m[:3, :3].T + m[:3, 3]
        self.vertices = v
        return self

    def rotate(self, R, center):
        c = np.asarray(center, dtype=np.float64)
        self.vertices = (self.vertices - c) @ np.asarray(R, dtype=np.float64).T + c
        return self

    def translate(self, t):
        self.vertices = self.vertices + np.asarray(t, dtype=np.float64)
        return self

    def compute_triangle_normals(self, normalized=True):
        v = self.vertices
        f = self.triangles
        n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        if normalized:
            with np.errstate(invalid="ignore", divide="ignore"):
                n = n / np.linalg.norm(n, axis=1, keepdims=True)
            bad = np.isnan(n[:, 0])
            n[bad] = np.array([0.0, 0.0, 1.0])
        self.triangle_normals = n
        return self

    def get_axis_aligned_bounding_box(self):
        return _AABB(self.vertices.min(axis=0), self.vertices.max(axis=0))

    def get_center(self):
        return self.vertices.mean(axis=0)

    def get_surface_area_per_triangle(self):
        v = self.vertices
        f = self.triangles
        return 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1)

    def sample_points_uniformly(self, number_of_points=100, use_triangle_normal=False):
        """Open3D TriangleMesh::SamplePointsUniformlyImpl: triangle t receives
        round(cumulative_area_fraction(t) * n) - (points so far) samples, each
        (1-sqrt(r1)) v0 + sqrt(r1)(1-r2) v1 + sqrt(r1) r2 v2, walking the
        triangles in index order (hence "not dispersed", sdf.py:648)."""
        areas = self.get_surface_area_per_triangle()
        cum = np.cumsum(areas / areas.sum())
        # std::round = half away from zero; values are >= 0
        upto = np.floor(cum * number_of_points + 0.5).astype(np.int64)
        upto = np.minimum(upto, number_of_points)
        counts = np.diff(np.concatenate([[0], upto]))
        counts = np.maximum(counts, 0)
        tri_of_point = np.repeat(np.arange(len(areas)), counts)
        n = len(tri_of_point)
        r = _uniform_doubles(2 * n)
        r1, r2 = r[0::2], r[1::2]
        s = np.sqrt(r1)
        a, b, c = (1 - s), s * (1 - r2), s * r2
        v = self.vertices
        f = self.triangles[tri_of_point]
        pts = a[:, None] * v[f[:, 0]] + b[:, None] * v[f[:, 1]] + c[:, None] * v[f[:, 2]]
        return _PointCloud(pts)


def _parse_obj(path):
    """Wavefront OBJ: 'v x y z' positions, 'f' polygons triangulated as a fan
    (tinyobjloader with triangulate=true on convex polygons); vt/vn ignored;
    1-based and negative (relative) indices."""
    verts, tris = [], []
    with open(path, "r", errors="ignore") as fh:
        for line in fh:
            if line.startswith("v "):
                p = line.split()
                verts.append((float(p[1]), float(p[2]), float(p[3])))
            elif line.startswith("f "):
                idx = []
                for tok in line.split()[1:]:
                    i = int(tok.split("/")[0])
                    idx.append(i - 1 if i > 0 else len(verts) + i)
                for k in range(1, len(idx) - 1):
                    tris.append((idx[0], idx[k], idx[k + 1]))
    return np.array(verts, dtype=np.float64).reshape(-1, 3), np.array(tris, dtype=np.int32).reshape(-1, 3)


def _parse_stl(path):
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:5] == b"solid" and b"facet" in data[:1000]:
        vs = []
        for line in data.decode(errors="ignore").splitlines():
            line = line.strip()
            if line.startswith("vertex"):
                p = line.split()
                vs.append((float(p[1]), float(p[2]), float(p[3])))
        v = np.array(vs, dtype=np.float64).reshape(-1, 3)
    else:
        n = struct.unpack("<I", data[80:84])[0]
        rec = np.frombuffer(data, dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", 9), ("a", "<u2")]), count=n, offset=84)
        v = rec["v"].reshape(-1, 3).astype(np.float64)
    f = np.arange(len(v), dtype=np.int32).reshape(-1, 3)
    return v, f


def read_triangle_mesh(path):
    if path.lower().endswith(".stl"):
        v, f = _parse_stl(path)
    else:
        v, f = _parse_obj(path)
    return TriangleMesh(v, f)


def get_rotation_matrix_from_quaternion(q):
    w, x, y, z = (float(c) for c in q)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
    ])


class _T:
    """Minimal stand-in for open3d.core.Tensor (only .numpy() is used)."""

    def __init__(self, a):
        self._a = a

    def numpy(self):
        return self._a


class _TMesh:
    def __init__(self, v32, f):
        self.v32, self.f = v32, f

    @staticmethod
    def from_legacy(mesh):
        # t.geometry.TriangleMesh.from_legacy defaults to float32 positions
        return _TMesh(mesh.vertices.astype(np.float32), mesh.triangles.astype(np.int32))


class RaycastingScene:
    def __init__(self):
        self._soup = None

    def add_triangles(self, mesht):
        self._soup = _geom.TriangleSoup(mesht.v32, mesht.f)
        return 0

    def compute_closest_points(self, query_points):
        q = np.ascontiguousarray(query_points, dtype=np.float32)
        shape = q.shape[:-1]
        closest, _d2, face = self._soup.closest_points(q.reshape(-1, 3), method=QUERY_METHOD)
        return {"points": _T(closest.reshape(*shape, 3)),
                "primitive_ids": _T(face.astype(np.uint32).reshape(shape)),
                "geometry_ids": _T(np.zeros(shape, np.uint32))}

    def count_intersections(self, rays):
        r = np.ascontiguousarray(rays, dtype=np.float32)
        shape = r.shape[:-1]
        return _T(self._soup.count_intersections(r.reshape(-1, 6), method=QUERY_METHOD).reshape(shape))


# --- module layout mirroring `import open3d as o3d` -------------------------
io = types.SimpleNamespace(read_triangle_mesh=read_triangle_mesh)
geometry = types.SimpleNamespace(TriangleMesh=TriangleMesh, PointCloud=_PointCloud,
                                 get_rotation_matrix_from_quaternion=get_rotation_matrix_from_quaternion)
t = types.SimpleNamespace(geometry=types.SimpleNamespace(TriangleMesh=_TMesh, RaycastingScene=RaycastingScene))
utility = types.SimpleNamespace(random=types.SimpleNamespace(seed=_seed))
