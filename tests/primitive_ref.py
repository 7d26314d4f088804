"""fp64 restatements of the analytic primitive SDFs (BoxSDF, CylinderSDF, SphereSDF; pvb_device.cuh box_eval /
cylinder_eval / sphere_eval) with the tie rules their docstrings state, for the CPU and GPU tiers.  Each takes fp64
points [n, 3] in the primitive's frame and returns (value [n], gradient [n, 3])."""
import numpy as np


def _sign(x):
    return np.where(x >= 0, 1.0, -1.0)          # -0 counts as +


def box_ref(half, q):
    """half: the three half extents (bb_max of the descriptor)."""
    q = np.asarray(q, dtype=np.float64)
    e = np.abs(q) - np.asarray(half, dtype=np.float64)
    w = np.maximum(e, 0.0)
    n = np.linalg.norm(w, axis=1)
    out = n > 0
    k = e.argmax(axis=1)                         # first axis on ties
    val = np.where(out, n, e.max(axis=1))
    g_in = np.zeros_like(q)
    g_in[np.arange(len(q)), k] = _sign(q[np.arange(len(q)), k])
    with np.errstate(invalid="ignore", divide="ignore"):
        g_out = _sign(q) * w / n[:, None]
    return val, np.where(out[:, None], g_out, g_in)


def cylinder_ref(radius, half_length, q):
    q = np.asarray(q, dtype=np.float64)
    rho = np.hypot(q[:, 0], q[:, 1])
    on_axis = rho == 0
    with np.errstate(invalid="ignore", divide="ignore"):
        ux = np.where(on_axis, 1.0, q[:, 0] / rho)
        uy = np.where(on_axis, 0.0, q[:, 1] / rho)
    sz = _sign(q[:, 2])
    dr, dz = rho - radius, np.abs(q[:, 2]) - half_length
    wr, wz = np.maximum(dr, 0.0), np.maximum(dz, 0.0)
    n = np.hypot(wr, wz)
    out = n > 0
    radial = dr >= dz                            # radial wins ties
    val = np.where(out, n, np.maximum(dr, dz))
    with np.errstate(invalid="ignore", divide="ignore"):
        g_out = np.stack([wr * ux / n, wr * uy / n, wz * sz / n], axis=1)
    g_in = np.where(radial[:, None], np.stack([ux, uy, np.zeros_like(ux)], 1),
                    np.stack([np.zeros_like(ux), np.zeros_like(ux), sz], 1))
    return val, np.where(out[:, None], g_out, g_in)


def sphere_ref(radius, q):
    q = np.asarray(q, dtype=np.float64)
    r = np.linalg.norm(q, axis=1)
    return r - radius, q / (r + 1e-12)[:, None]


def primitive_ref(desc, q):
    """The restatement for a pvb_sdf_desc of kind SPHERE / BOX / CYLINDER (its fp32 fields)."""
    from pytorch_volumetric_b200 import _native as nat
    h = [float(desc.bb_max[k]) for k in range(3)]
    if desc.kind == nat.PVB_KIND_BOX:
        return box_ref(h, q)
    if desc.kind == nat.PVB_KIND_CYLINDER:
        return cylinder_ref(float(desc.radius), h[2], q)
    assert desc.kind == nat.PVB_KIND_SPHERE
    return sphere_ref(float(desc.radius), q)


def second_gap(desc, q):
    """Distance between the two largest per-axis terms of the inside rule (box: |q_k| - h_k; cylinder: rho - r and
    |z| - h), fp64: where it is tiny, fp32 rounding may pick the other axis, so a gradient comparison there is a
    near-tie, not an error.  +inf for spheres."""
    from pytorch_volumetric_b200 import _native as nat
    q = np.asarray(q, dtype=np.float64)
    h = np.array([float(desc.bb_max[k]) for k in range(3)])
    if desc.kind == nat.PVB_KIND_BOX:
        e = np.sort(np.abs(q) - h, axis=1)
        return e[:, 2] - e[:, 1]
    if desc.kind == nat.PVB_KIND_CYLINDER:
        return np.abs(np.hypot(q[:, 0], q[:, 1]) - float(desc.radius) - (np.abs(q[:, 2]) - h[2]))
    return np.full(len(q), np.inf)
