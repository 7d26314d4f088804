"""Host-side model of tile-level culling for the C4 / RobotSDF kernel (next-round candidate, DESIGN section 8):
Morton-sort the shared point set, take tiles of 32 points, and per (configuration, tile) reject links with ONE
bounding-sphere test before any per-point work.  Counts, per (configuration, point) pair: link bound tests and table
lookups, against today's per-point scheme (8 object-frame sphere tests + bit-reversed visiting order).  CPU only
(oracle port for the true values, the product's grid_prune_margin for the bounds)."""
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import workloads  # noqa: E402
from oracle import port, tp_open3d  # noqa: E402
from oracle import tp_pytorch_kinematics as opk  # noqa: E402
from pytorch_volumetric_b200.sdf import grid_prune_margin  # noqa: E402


def morton_order(p, lo, hi, bits=10):
    g = ((p - lo) / (hi - lo) * ((1 << bits) - 1)).astype(np.int64).clip(0, (1 << bits) - 1)
    code = np.zeros(len(p), dtype=np.int64)
    for b in range(bits):
        for a in range(3):
            code |= ((g[:, a] >> b) & 1) << (3 * b + a)
    return np.argsort(code, kind="stable")


def main(n_cfg=16, n_pts=100_000, tile=32):
    tp_open3d.QUERY_METHOD = "bvh"
    d = tempfile.mkdtemp(prefix="pvb_arm_cpu_")
    urdf, end = workloads.write_arm(d)
    chain = opk.build_serial_chain_from_urdf(open(urdf).read(), end)
    robot = port.RobotSDFPort(chain, path_prefix=d, link_sdf_factory=port.cache_link_sdf_factory_port(0.02, 1.0))
    robot.set_joint_configuration(workloads.arm_configurations(n_cfg))
    lo = np.array([r[0] for r in workloads.ARM_QUERY_RANGE]); hi = np.array([r[1] for r in workloads.ARM_QUERY_RANGE])
    pts = workloads.uniform_points(n_pts, lo, hi, seed=4).numpy()
    pts = pts[morton_order(pts, lo, hi)]
    pts = pts[:(len(pts) // tile) * tile]
    P, S = len(pts), len(robot.sdf.sdfs)
    T = P // tile
    M = robot.object_to_link.get_matrix().reshape(S, n_cfg, 4, 4).numpy().astype(np.float64)
    V = np.empty((n_cfg, P, S)); LB = np.empty((n_cfg, P, S)); LBT = np.empty((n_cfg, T, S))
    cen = pts.reshape(T, tile, 3).mean(1)
    rad = np.linalg.norm(pts.reshape(T, tile, 3) - cen[:, None], axis=-1).max(1)
    for s, link in enumerate(robot.sdf.sdfs):
        bb = np.asarray(link.bb, dtype=np.float64)
        rl = [float(r[0]) for r in link.ranges]; rh = [float(r[1]) for r in link.ranges]
        margin = grid_prune_margin(link.voxels.raw_data.reshape(tuple(link.voxels.shape)), rl, rh, bb.astype(np.float32))
        q = np.einsum("cij,pj->cpi", M[s, :, :3, :3], pts) + M[s, :, None, :3, 3]
        v, _ = link(torch.from_numpy(q.reshape(-1, 3)).float())
        V[:, :, s] = v.reshape(n_cfg, P).numpy()
        LB[:, :, s] = np.linalg.norm(np.clip(np.maximum(bb[:, 0] - q, q - bb[:, 1]), 0, None), axis=-1) - margin
        qc = np.einsum("cij,tj->cti", M[s, :, :3, :3], cen) + M[s, :, None, :3, 3]
        LBT[:, :, s] = np.linalg.norm(np.clip(np.maximum(bb[:, 0] - qc, qc - bb[:, 1]), 0, None), axis=-1) - rad - margin
    order = [0, 4, 2, 6, 1, 5, 3, 7][:S]

    def per_point(allowed):           # allowed: (cfg, P, S) bool -- links not culled at tile level
        best = np.full((n_cfg, P), np.inf); looks = np.zeros((n_cfg, P)); tests = np.zeros((n_cfg, P))
        for s in order:
            tests += allowed[:, :, s]
            ev = allowed[:, :, s] & (LB[:, :, s] <= best)
            looks += ev
            best = np.where(ev, np.minimum(best, V[:, :, s]), best)
        return tests.mean(), looks.mean(), best

    t0, l0, b0 = per_point(np.ones((n_cfg, P, S), bool))
    assert np.array_equal(b0, V.min(-1))
    print(f"pairs {n_cfg * P}, tiles of {tile} Morton-ordered points: mean tile radius {rad.mean():.3f} m")
    print(f"today        : {t0:.2f} per-point link tests + {l0:.2f} lookups per pair")
    # tile culling: evaluate the link with the smallest tile bound for all 32 points, cull links whose tile bound
    # exceeds the largest of those 32 values, then the per-point scheme on the survivors
    first = LBT.argmin(-1)                                                     # (cfg, T)
    vf = np.take_along_axis(V.reshape(n_cfg, T, tile, S), first[:, :, None, None], -1)[..., 0]    # (cfg, T, tile)
    ub = vf.max(-1)                                                            # (cfg, T)
    keep = LBT <= ub[:, :, None]                                               # (cfg, T, S)
    allowed = np.repeat(keep, tile, axis=1)
    t1, l1, b1 = per_point(allowed)
    assert np.array_equal(b1, V.min(-1)), "tile culling must be exact"
    print(f"tile culling : {S / tile:.2f} tile tests + {t1:.2f} per-point link tests + {l1:.2f} lookups per pair; "
          f"{keep.sum(-1).mean():.2f} of {S} links survive per tile")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:]))
