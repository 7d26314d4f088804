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


# The same chain with every link an analytic URDF primitive (RobotSDF(..., primitive_visuals=True)): a box base, then
# cylinders and boxes of about 0.2 m and a sphere at the end, each placed by an <origin> with a non-trivial rpy.
PRIMITIVE_ARM_LINKS = [
    # (geometry element, origin xyz, origin rpy)
    ('<box size="0.24 0.2 0.15"/>', "0 0 0.075", "0 0 0.3"),
    ('<cylinder radius="0.065" length="0.2"/>', "0 0 0.1", "0.2 0 0"),
    ('<box size="0.1 0.12 0.21"/>', "0 0 0.1", "0 0.15 0.6"),
    ('<cylinder radius="0.06" length="0.22"/>', "0 0 0.11", "0.1 -0.1 0.9"),
    ('<box size="0.09 0.11 0.19"/>', "0 0 0.09", "-0.2 0 1.2"),
    ('<cylinder radius="0.055" length="0.21"/>', "0 0 0.1", "0 0.25 1.5"),
    ('<box size="0.08 0.09 0.1"/>', "0 0 0.04", "0.3 0.2 0.1"),
    ('<sphere radius="0.05"/>', "0 0 0.05", "0 0 0"),
]
# links of the mixed arm that are the probe mesh (as in write_arm) instead of their primitive
MIXED_ARM_MESH_LINKS = (1, 4, 6)


def write_primitive_arm(dirname, mesh_links=(), mesh_scale=3.0):
    """Writes arm.urdf (+ link.obj when `mesh_links` is not empty) into `dirname`: the chain of write_arm with link i
    the primitive PRIMITIVE_ARM_LINKS[i], or the probe mesh of write_arm for i in `mesh_links`
    (MIXED_ARM_MESH_LINKS: the mixed arm).  Returns the URDF path and end link name."""
    from pytorch_volumetric_b200.meshio import write_obj
    os.makedirs(dirname, exist_ok=True)
    if mesh_links:
        v, f = fixture_mesh("probe")
        write_obj(os.path.join(dirname, "link.obj"), v, f)
    parts = ['<robot name="arm7_primitive">']
    for i, (geom, xyz, rpy) in enumerate(PRIMITIVE_ARM_LINKS):
        if i in mesh_links:
            xyz, rpy = "0 0 0.02", f"0 0 {0.3 * i:.3f}"
            geom = f'<mesh filename="link.obj" scale="{mesh_scale} {mesh_scale} {mesh_scale}"/>'
        parts.append(f'<link name="link_{i}"><visual><origin xyz="{xyz}" rpy="{rpy}"/><geometry>{geom}</geometry>'
                     f'</visual></link>')
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


# --------------------------------------------------------------------------- kinematic trees
# Two branching robots for RobotSDF's tree path (build_chain_from_urdf).  Every joint carries a <limit>, which
# tree_configurations samples within.  Joints are written in depth-first pre-order, so the document order of the
# movable joints is the column order of q.
def _tree_urdf(dirname, name, links, joints, meshes):
    """Writes <name>.urdf (+ link.obj, the probe mesh, with `meshes`): links [(name, [(kind, dims, xyz, rpy)])],
    joints [(name, type, parent, child, xyz, rpy, axis, (lower, upper))].  With `meshes` every visual is the probe mesh
    scaled to the primitive's extents.  Returns the URDF path."""
    from pytorch_volumetric_b200.meshio import write_obj
    os.makedirs(dirname, exist_ok=True)
    if meshes:
        v, f = fixture_mesh("probe")
        write_obj(os.path.join(dirname, "link.obj"), v, f)
        span = v.max(0) - v.min(0)

    def geometry(kind, dims):
        if meshes:
            size = dims if kind == "box" else (2 * dims[0], 2 * dims[0], dims[1] if kind == "cylinder" else 2 * dims[0])
            return f'<mesh filename="link.obj" scale="{" ".join(f"{s / e:.6f}" for s, e in zip(size, span))}"/>'
        if kind == "box":
            return f'<box size="{dims[0]} {dims[1]} {dims[2]}"/>'
        if kind == "cylinder":
            return f'<cylinder radius="{dims[0]}" length="{dims[1]}"/>'
        return f'<sphere radius="{dims[0]}"/>'

    parts = [f'<robot name="{name}">']
    for link, visuals in links:
        vis = "".join(f'<visual><origin xyz="{xyz}" rpy="{rpy}"/><geometry>{geometry(k, d)}</geometry></visual>'
                      for k, d, xyz, rpy in visuals)
        parts.append(f'<link name="{link}">{vis}</link>')
    for jn, jt, parent, child, xyz, rpy, axis, (lo, hi) in joints:
        ax = f'<axis xyz="{axis}"/>' if axis else ""
        parts.append(f'<joint name="{jn}" type="{jt}"><parent link="{parent}"/><child link="{child}"/>'
                     f'<origin xyz="{xyz}" rpy="{rpy}"/>{ax}<limit lower="{lo}" upper="{hi}"/></joint>')
    parts.append("</robot>")
    path = os.path.join(dirname, name + ".urdf")
    with open(path, "w") as fh:
        fh.write("\n".join(parts))
    return path


HAND_FINGERS = 4


def write_hand(dirname, meshes=False):
    """A hand on a two-joint wrist: forearm (root) -> wrist -> palm; four fingers off the palm, each an abduction joint
    and three flexion joints (knuckle without a visual, then proximal, middle and distal segments); a thumb mounted
    through a fixed joint with a rotated origin, then three revolute joints.  23 links, 18 of them with a box,
    cylinder or sphere visual (the probe mesh with `meshes`), 21 movable joints.  Returns the URDF path."""
    links = [("forearm", [("cylinder", (0.035, 0.2), "0 0 -0.1", "0 0 0")]), ("wrist", []),
             ("palm", [("box", (0.09, 0.03, 0.1), "0 0 0.05", "0 0 0")])]
    joints = [("wrist_pitch", "revolute", "forearm", "wrist", "0 0 0.02", "0 0 0", "0 1 0", (-1.0, 1.0)),
              ("wrist_roll", "revolute", "wrist", "palm", "0 0 0.03", "0 0 0", "1 0 0", (-1.0, 1.0))]
    for i in range(HAND_FINGERS):
        f, k = f"finger{i}", 1.0 - 0.08 * abs(i - 1.5)           # the middle fingers are the longest
        x = -0.033 + 0.022 * i
        links += [(f"{f}_knuckle", []),
                  (f"{f}_proximal", [("cylinder", (0.009, 0.045 * k), f"0 0 {0.0225 * k:.5f}", "0 0 0")]),
                  (f"{f}_middle", [("cylinder", (0.008, 0.03 * k), f"0 0 {0.015 * k:.5f}", "0 0 0")]),
                  (f"{f}_distal", [("box", (0.014, 0.013, 0.025 * k), f"0 0 {0.0125 * k:.5f}", "0 0 0.1")])]
        joints += [(f"{f}_abduct", "revolute", "palm", f"{f}_knuckle", f"{x:.3f} 0 0.1", "0 0 0", "0 1 0", (-0.3, 0.3)),
                   (f"{f}_flex1", "revolute", f"{f}_knuckle", f"{f}_proximal", "0 0 0.002", "0 0 0", "1 0 0",
                    (-0.2, 1.5)),
                   (f"{f}_flex2", "revolute", f"{f}_proximal", f"{f}_middle", f"0 0 {0.045 * k:.5f}", "0 0 0",
                    "1 0 0", (0.0, 1.6)),
                   (f"{f}_flex3", "revolute", f"{f}_middle", f"{f}_distal", f"0 0 {0.03 * k:.5f}", "0 0 0", "1 0 0",
                    (0.0, 1.4))]
    links += [("thumb_base", [("sphere", (0.013,), "0 0 0", "0 0 0")]),
              ("thumb_proximal", [("cylinder", (0.01, 0.035), "0 0 0.0175", "0 0 0")]),
              ("thumb_middle", [("cylinder", (0.009, 0.03), "0 0 0.015", "0 0 0")]),
              ("thumb_distal", [("sphere", (0.01,), "0 0 0.01", "0 0 0")])]
    joints += [("thumb_mount", "fixed", "palm", "thumb_base", "0.05 0 0.03", "0.2 0.9 0.3", None, (0.0, 0.0)),
               ("thumb_flex1", "revolute", "thumb_base", "thumb_proximal", "0 0 0.012", "0 0 0", "1 0 0", (-0.5, 1.2)),
               ("thumb_flex2", "revolute", "thumb_proximal", "thumb_middle", "0 0 0.035", "0 0 0", "1 0 0",
                (0.0, 1.2)),
               ("thumb_flex3", "revolute", "thumb_middle", "thumb_distal", "0 0 0.03", "0 0 0", "1 0 0", (0.0, 1.2))]
    return _tree_urdf(dirname, "hand_mesh" if meshes else "hand", links, joints, meshes)


def write_gripper_tree(dirname):
    """A short arm with a two-finger gripper: base (root) -> three revolute joints -> palm, then one prismatic finger
    (with a fingertip through a fixed joint with a rotated origin) and one revolute finger of two segments.  8 links,
    every one with a box, cylinder or sphere visual, so the fused cost and self-clearance kernels run on it; 6 movable
    joints.  Returns the URDF path."""
    links = [("base", [("box", (0.12, 0.12, 0.06), "0 0 0.03", "0 0 0.2")]),
             ("link1", [("cylinder", (0.04, 0.2), "0 0 0.1", "0 0 0")]),
             ("link2", [("cylinder", (0.035, 0.18), "0 0 0.09", "0.1 0 0")]),
             ("palm", [("box", (0.1, 0.04, 0.04), "0 0 0.02", "0 0 0")]),
             ("finger_a", [("box", (0.015, 0.02, 0.06), "0 0 0.03", "0 0 0")]),
             ("finger_a_tip", [("sphere", (0.01,), "0 0 0.005", "0 0 0")]),
             ("finger_b1", [("box", (0.015, 0.02, 0.05), "0 0 0.025", "0 0 0")]),
             ("finger_b2", [("cylinder", (0.008, 0.04), "0 0 0.02", "0 0 0")])]
    joints = [("j1", "revolute", "base", "link1", "0 0 0.06", "0 0 0", "0 0 1", (-3.0, 3.0)),
              ("j2", "revolute", "link1", "link2", "0 0 0.2", "0 0 0", "0 1 0", (-1.5, 1.5)),
              ("j3", "revolute", "link2", "palm", "0 0 0.18", "0 0 0", "0 0 1", (-3.0, 3.0)),
              ("finger_a_slide", "prismatic", "palm", "finger_a", "-0.03 0 0.04", "0 0 0", "1 0 0", (-0.025, 0.0)),
              ("finger_a_tip_mount", "fixed", "finger_a", "finger_a_tip", "0 0 0.06", "0 0.3 0", None, (0.0, 0.0)),
              ("finger_b_base", "revolute", "palm", "finger_b1", "0.03 0 0.04", "0 0 0", "0 1 0", (-0.6, 0.3)),
              ("finger_b_tip", "revolute", "finger_b1", "finger_b2", "0 0 0.05", "0 0 0", "0 1 0", (-0.8, 0.8))]
    return _tree_urdf(dirname, "gripper_tree", links, joints, False)


def tree_configurations(urdf_path, n, seed=5, dtype=torch.float32):
    """[n, J] joint values of a URDF written by write_hand / write_gripper_tree: configuration 0 all zeros (clamped
    into the limits), the others uniform within every movable joint's <limit>; J in document order."""
    import xml.etree.ElementTree as ET
    joints = [j for j in ET.parse(urdf_path).getroot().findall("joint") if j.get("type") != "fixed"]
    lo = torch.tensor([float(j.find("limit").get("lower")) for j in joints], dtype=torch.float64)
    hi = torch.tensor([float(j.find("limit").get("upper")) for j in joints], dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    q = lo + (hi - lo) * torch.rand(n, len(joints), generator=g, dtype=torch.float64)
    q[0] = torch.zeros(len(joints), dtype=torch.float64).clamp(lo, hi)
    return q.to(dtype)


# ---------------------------------------------------------------- depth images of box scenes (depth_occupancy)
# The tabletop scene of scripts/c4bench.scene_points as solid boxes (lo_x, lo_y, lo_z, size_x, size_y, size_z): the
# table, 5 cm thick with its top at z = -0.2, and the six boxes standing on it or above it.
TABLETOP_BOXES = ((-1.0, -0.5, -0.25, 1.5, 1.0, 0.05), (-0.9, -0.45, -0.2, 0.3, 0.25, 0.35),
                  (0.2, -0.45, -0.2, 0.25, 0.2, 0.6), (-0.4, 0.3, -0.2, 0.5, 0.15, 0.25),
                  (0.3, 0.25, -0.2, 0.15, 0.2, 0.9), (-0.95, 0.2, 0.4, 0.2, 0.25, 0.3),
                  (-0.3, -0.5, 0.5, 0.6, 0.05, 0.3))
TABLETOP_RANGE = ((-1.1, 0.7), (-0.6, 0.6), (-0.35, 1.0))


def look_at(eye, target, up=(0.0, 0.0, 1.0)):
    """fp64 [4, 4] camera-to-world transform of an OpenCV camera (x right, y down, z forward) at eye looking at
    target."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, np.asarray(up, np.float64))
    x /= np.linalg.norm(x)
    m = np.eye(4)
    m[:3, :3] = np.stack([x, np.cross(z, x), z], axis=1)
    m[:3, 3] = eye
    return m


def camera_ring(n, target, radius, height, f, H=480, W=640, seed=0):
    """(K fp64 [3, 3], cam_to_world fp64 [n, 4, 4]): n pinhole cameras of focal length f pixels (principal point at
    the image centre) evenly spaced on a horizontal circle of the given radius about target, `height` above it, all
    looking at target; the seed turns the ring by a random angle."""
    K = np.array([[f, 0.0, (W - 1) / 2], [0.0, f, (H - 1) / 2], [0.0, 0.0, 1.0]])
    phase = np.random.default_rng(seed).uniform(0.0, 2 * math.pi)
    target = np.asarray(target, np.float64)
    poses = []
    for k in range(n):
        a = phase + 2 * math.pi * k / n
        poses.append(look_at(target + [radius * math.cos(a), radius * math.sin(a), height], target))
    return K, np.stack(poses)


def render_depth(boxes, K, cam_to_world, H=480, W=640, noise=0.0, seed=0):
    """float32 [V, H, W] z-depth images of solid axis-aligned boxes (lo_x, lo_y, lo_z, size_x, size_y, size_z), in
    fp64 by ray-slab intersection: pixel (i, j) looks along ((j - cx) / fx, (i - cy) / fy, 1) in the camera, so the
    ray parameter of the first hit is its z-depth.  A pixel that hits nothing reads 0 (no return); noise > 0 adds
    seeded Gaussian noise of that standard deviation (metres) to every hit."""
    K = np.asarray(K, np.float64)
    poses = np.asarray(cam_to_world, np.float64)
    K = np.broadcast_to(K, (len(poses), 3, 3))
    b = np.asarray(boxes, np.float64)
    lo, hi = b[:, :3], b[:, :3] + b[:, 3:]
    i, j = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    g = np.random.default_rng(seed)
    out = np.zeros((len(poses), H, W), np.float32)
    for v, (k, m) in enumerate(zip(K, poses)):
        d_cam = np.stack([(j - k[0, 2]) / k[0, 0], (i - k[1, 2]) / k[1, 1], np.ones_like(i)], -1).reshape(-1, 3)
        d = d_cam @ m[:3, :3].T
        o = m[:3, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            t0 = (lo[None] - o) / d[:, None]                    # [rays, boxes, 3]
            t1 = (hi[None] - o) / d[:, None]
        near = np.fmax.reduce(np.minimum(t0, t1), axis=2)
        far = np.fmin.reduce(np.maximum(t0, t1), axis=2)
        hit = (near <= far) & (near > 0)
        t = np.where(hit, near, np.inf).min(axis=1)
        depth = np.where(np.isfinite(t), t, 0.0)
        if noise > 0:
            depth = np.where(depth > 0, depth + g.normal(0.0, noise, depth.shape), 0.0)
        out[v] = depth.reshape(H, W)
    return out


def tabletop_views(n, H=480, W=640, f=800.0, seed=0):
    """(depth float32 [n, H, W], K fp64 [3, 3], cam_to_world fp64 [n, 4, 4]): the tabletop boxes seen by a ring of n
    cameras 2.2 m from the scene's centre and 1.3 m above it (about 2.5 m away)."""
    K, poses = camera_ring(n, (-0.25, 0.0, 0.2), 2.2, 1.3, f, H, W, seed)
    return render_depth(TABLETOP_BOXES, K, poses, H, W), K, poses


# ---------------------------------------------------------------- LiDAR scans of box scenes (ray_occupancy)
def render_lidar(boxes, origin, beams, columns, elevation=(-0.4, 0.4), max_range=10.0, noise=0.0, seed=0):
    """float32 [beams * columns, 3] world returns of a spinning LiDAR at `origin` among solid axis-aligned boxes
    (lo_x, lo_y, lo_z, size_x, size_y, size_z), in fp64 by ray-slab intersection as render_depth does.  Beam b looks
    at elevation lo + (hi - lo) b / (beams - 1) radians, column c at azimuth 2 pi c / columns, rows beam-major.  The
    first hit along a ray at range t <= max_range gives o + t d; a ray that hits nothing within max_range reads NaN
    (no return).  noise > 0 adds seeded Gaussian noise of that standard deviation (metres) to every hit's range."""
    o = np.asarray(origin, np.float64)
    b = np.asarray(boxes, np.float64)
    lo, hi = b[:, :3], b[:, :3] + b[:, 3:]
    el = np.linspace(elevation[0], elevation[1], beams) if beams > 1 else np.array([elevation[0]], np.float64)
    az = 2 * math.pi * np.arange(columns, dtype=np.float64) / columns
    e, a = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (lo[None] - o) / d[:, None]
        t1 = (hi[None] - o) / d[:, None]
    near = np.fmax.reduce(np.minimum(t0, t1), axis=2)
    far = np.fmin.reduce(np.maximum(t0, t1), axis=2)
    t = np.where((near <= far) & (near > 0), near, np.inf).min(axis=1)
    if noise > 0:
        t = t + np.random.default_rng(seed).normal(0.0, noise, t.shape)
    hit = np.isfinite(t) & (t <= max_range)
    return np.where(hit[:, None], o + np.where(hit, t, 0.0)[:, None] * d, np.nan).astype(np.float32)


# The tabletop boxes in a room: a floor 0.45 m below the table's top and four walls 3 m from the scene's centre.
TABLETOP_ROOM = TABLETOP_BOXES + ((-3.25, -3.0, -0.75, 6.0, 6.0, 0.1), (-3.35, -3.0, -0.75, 0.1, 6.0, 3.0),
                                  (2.75, -3.0, -0.75, 0.1, 6.0, 3.0), (-3.25, -3.1, -0.75, 6.0, 0.1, 3.0),
                                  (-3.25, 3.0, -0.75, 6.0, 0.1, 3.0))

# Sensor positions about the tabletop: even ones inside TABLETOP_RANGE (above the table, clear of every box), odd
# ones outside it on a ring, so that rays both start inside the grid and enter it from outside.
TABLETOP_LIDAR_INSIDE = ((-0.25, 0.0, 0.3), (-0.5, 0.1, 0.25), (0.0, -0.1, 0.45), (-0.6, -0.2, 0.35))


def tabletop_lidar(n, beams=64, columns=1024, max_range=6.0, noise=0.0, seed=0, boxes=TABLETOP_ROOM):
    """(points float32 [n, beams * columns, 3], origins float32 [n, 3]): n LiDAR scans of the tabletop room, the
    sensors alternately inside TABLETOP_RANGE (TABLETOP_LIDAR_INSIDE in turn) and outside it (on a circle 1.8 m from
    the scene's centre, 1.2 m above it, at seeded angles), elevations -0.6..0.3 rad inside and -0.7..0.1 outside."""
    g = np.random.default_rng(seed)
    pts, origins = [], []
    for k in range(n):
        if k % 2 == 0:
            o = np.asarray(TABLETOP_LIDAR_INSIDE[(k // 2) % len(TABLETOP_LIDAR_INSIDE)], np.float64)
            elevation = (-0.6, 0.3)
        else:
            a = g.uniform(0.0, 2 * math.pi)
            o = np.array([-0.25 + 1.8 * math.cos(a), 1.8 * math.sin(a), 1.4])
            elevation = (-0.7, 0.1)
        pts.append(render_lidar(boxes, o, beams, columns, elevation, max_range, noise, seed + k))
        origins.append(o)
    return np.stack(pts), np.asarray(origins, np.float32)
