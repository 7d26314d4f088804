"""Synthetic workloads shared by bench.py and tests/ (BASELINE.json configs made concrete, SURVEY.md section 8d).

Nothing here reads the reference project: the reference's test meshes come from tests/golden/meshes.npz (written by
oracle/make_golden.py in the build container), everything else is procedural and seeded.
"""
import math
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(ROOT, "tests", "golden")

_mesh_cache = {}


def fixture_mesh(name):
    """(vertices fp64 [V,3], faces int32 [F,3]) of one of the reference's test meshes:
    probe | wrench | drill | scene_overlap | scene_separated."""
    if not _mesh_cache:
        with np.load(os.path.join(GOLDEN, "meshes.npz")) as z:
            for k in z.files:
                _mesh_cache[k] = z[k]
    return _mesh_cache[name + "_v"].copy(), _mesh_cache[name + "_f"].copy()


def bumpy_sphere(n_lon, n_lat, radius=0.1, bump=0.25):
    """Closed genus-0 non-convex mesh with exactly 2*n_lon*(n_lat-1) triangles:
    r(theta, phi) = radius * (1 + bump * sin(5 theta) * sin(4 phi)); n_lon=100, n_lat=51 -> 10 000 triangles,
    n_lon=250, n_lat=101 -> 50 000 triangles (SURVEY.md 8d, north-star target mesh)."""
    verts = [(0.0, 0.0, radius)]
    for i in range(1, n_lat):
        phi = math.pi * i / n_lat
        for j in range(n_lon):
            th = 2 * math.pi * j / n_lon
            r = radius * (1 + bump * math.sin(5 * th) * math.sin(4 * phi))
            verts.append((r * math.sin(phi) * math.cos(th), r * math.sin(phi) * math.sin(th), r * math.cos(phi)))
    verts.append((0.0, 0.0, -radius))
    south = len(verts) - 1

    def vid(i, j):
        return 1 + (i - 1) * n_lon + (j % n_lon)

    faces = []
    for j in range(n_lon):
        faces.append((0, vid(1, j), vid(1, j + 1)))
    for i in range(1, n_lat - 1):
        for j in range(n_lon):
            a, b, c, d = vid(i, j), vid(i, j + 1), vid(i + 1, j), vid(i + 1, j + 1)
            faces.append((a, c, d))
            faces.append((a, d, b))
    for j in range(n_lon):
        faces.append((south, vid(n_lat - 1, j + 1), vid(n_lat - 1, j)))
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    f = np.asarray(faces, dtype=np.int32)
    assert len(f) == 2 * n_lon * (n_lat - 1)
    return v, f


def uniform_points(n, lo, hi, seed, device="cpu", dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed)
    lo = torch.as_tensor(lo, dtype=torch.float64)
    hi = torch.as_tensor(hi, dtype=torch.float64)
    chunks = []
    left = n
    while left > 0:        # chunked so that 10^7-point clouds do not need a 240 MB fp64 temporary
        m = min(left, 2_000_000)
        chunks.append((lo + (hi - lo) * torch.rand(m, 3, generator=g, dtype=torch.float64)).to(dtype))
        left -= m
    return torch.cat(chunks).to(device)


def random_rigid(n, seed, t_range=0.5, dtype=torch.float32):
    """n rigid 4x4: translation U[-t_range, t_range]^3, rotation from a normalised 4-D Gaussian quaternion."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).reshape(n, 3, 3)
    m = torch.eye(4, dtype=torch.float64).repeat(n, 1, 1)
    m[:, :3, :3] = R
    m[:, :3, 3] = (torch.rand(n, 3, generator=g, dtype=torch.float64) - 0.5) * 2 * t_range
    return m.to(dtype)


# --------------------------------------------------------------------------- C4: synthetic 7-DOF arm
# pybullet_data's KUKA iiwa is not available offline: an "iiwa-like" serial chain with 8 links (base + 7
# revolute joints), alternating z / y axes, link meshes = the reference's probe mesh scaled to ~0.2 m.
ARM_JOINTS = [
    # (xyz of the joint origin in the parent link frame, axis)
    ((0.0, 0.0, 0.1575), (0, 0, 1)),
    ((0.0, 0.0, 0.2025), (0, 1, 0)),
    ((0.0, 0.0, 0.2045), (0, 0, 1)),
    ((0.0, 0.0, 0.2155), (0, -1, 0)),
    ((0.0, 0.0, 0.1845), (0, 0, 1)),
    ((0.0, 0.0, 0.2155), (0, 1, 0)),
    ((0.0, 0.0, 0.0810), (0, 0, 1)),
]
ARM_NOMINAL = [0.0, -math.pi / 4.0, 0.0, math.pi / 2.0, 0.0, math.pi / 4.0, 0.0]


def write_arm(dirname, mesh_scale=3.0):
    """Writes link.obj (probe mesh) + arm.urdf into `dirname`; returns the URDF path and end link name."""
    from pytorch_volumetric_b200.meshio import write_obj
    os.makedirs(dirname, exist_ok=True)
    v, f = fixture_mesh("probe")
    write_obj(os.path.join(dirname, "link.obj"), v, f)
    parts = ['<robot name="arm7">']
    for i in range(8):
        parts.append(f'<link name="link_{i}"><visual><origin xyz="0 0 0.02" rpy="0 0 {0.3 * i:.3f}"/><geometry>'
                     f'<mesh filename="link.obj" scale="{mesh_scale} {mesh_scale} {mesh_scale}"/></geometry></visual>'
                     f'</link>')
    for i, (xyz, axis) in enumerate(ARM_JOINTS):
        parts.append(f'<joint name="joint_{i + 1}" type="revolute"><parent link="link_{i}"/>'
                     f'<child link="link_{i + 1}"/><origin xyz="{xyz[0]} {xyz[1]} {xyz[2]}" rpy="0 0 0"/>'
                     f'<axis xyz="{axis[0]} {axis[1]} {axis[2]}"/></joint>')
    parts.append("</robot>")
    path = os.path.join(dirname, "arm.urdf")
    with open(path, "w") as fh:
        fh.write("\n".join(parts))
    return path, "link_7"


def arm_configurations(n, seed=3, dtype=torch.float32):
    """nominal pose + 0.1 * randn perturbations stacked under it (README.md:166-170 of the reference)."""
    g = torch.Generator().manual_seed(seed)
    th = torch.tensor(ARM_NOMINAL, dtype=dtype)
    if n == 1:
        return th.view(1, -1)
    return torch.cat((th.view(1, -1), torch.randn(n - 1, 7, generator=g, dtype=dtype) * 0.1 + th))


ARM_QUERY_RANGE = ((-1.0, 0.5), (-0.5, 0.5), (-0.2, 0.8))     # README.md:86-90 of the reference
