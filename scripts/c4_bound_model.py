"""Host-side model of the per-lane link bounds of robot_serial_kernel on the C4 arm: per (point, 32-configuration warp
step), how many warp-level link visits, lane-level table lookups and wasted visits (the warp visits a link, but no lane
passes the exact AABB test after the transform) does each candidate bound cost?  The model follows the kernel: lanes
are 32 consecutive configurations of one point; the first visit goes to lane 0's link with the smallest bound and
every lane looks it up; a later link is visited when some lane's bound is <= its running minimum, and inside the
visit a lane looks up only when dist(q, AABB) - prune_margin <= its running minimum.  Bounds (all minus prune_margin,
in fp64: the kernel's fp32 slack only lowers them further):
  sphere : |p - c_obj| - r           (the sphere around the link AABB, centre carried to the object frame)
  slab   : |n.p + t - c| - h         (the link-frame row of the AABB's thinnest axis: centre c, half-extent h)
  max    : max(sphere, slab)
  aabb   : the exact dist(q, AABB) itself (floor: no wasted visit)
Asserts that every bound is exact (the same minimum as evaluating all links).  CPU only (oracle port for the true
values, the product's grid_prune_margin for the margins)."""
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


def simulate(V, EX, LB, lanes=32):
    """V, EX, LB: (cfg, P, S) values, exact AABB bounds, candidate pre-bounds.  Returns the mean warp visits, lane
    lookups and wasted visits per warp step (point x `lanes` configurations) and the per-pair minimum."""
    C, P, S = V.shape
    W = C // lanes
    V, EX, LB = (a[:W * lanes].reshape(W, lanes, P, S) for a in (V, EX, LB))
    first = LB[:, 0].argmin(-1)                                           # (W, P): lane 0's nearest-bound link
    take = lambda a: np.take_along_axis(a, first[:, None, :, None], -1)[..., 0]
    best = take(V)                                                        # every lane looks the first link up
    visits = np.ones((W, P)); looks = np.full((W, P), float(lanes)); wasted = np.zeros((W, P))
    for s in range(S):
        nf = first != s
        want = nf[:, None] & (LB[..., s] <= best)                         # lanes whose pre-bound passes
        vis = want.any(1)
        look = want & (EX[..., s] <= best)                                # lanes that pass the exact test too
        visits += vis; looks += look.sum(1); wasted += vis & ~look.any(1)
        best = np.where(look, np.minimum(best, V[..., s]), best)
    return visits.mean(), looks.mean(), wasted.mean(), best.reshape(W * lanes, P)


def main(n_cfg=64, n_pts=20_000):
    tp_open3d.QUERY_METHOD = "bvh"
    d = tempfile.mkdtemp(prefix="pvb_arm_cpu_")
    urdf, end = workloads.write_arm(d)
    chain = opk.build_serial_chain_from_urdf(open(urdf).read(), end)
    robot = port.RobotSDFPort(chain, path_prefix=d, link_sdf_factory=port.cache_link_sdf_factory_port(0.02, 1.0))
    robot.set_joint_configuration(workloads.arm_configurations(n_cfg))
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    pts = workloads.uniform_points(n_pts, lo, hi, seed=4).numpy().astype(np.float64)
    S = len(robot.sdf.sdfs)
    M = robot.object_to_link.get_matrix().reshape(S, n_cfg, 4, 4).numpy().astype(np.float64)
    V, EX = np.empty((n_cfg, n_pts, S)), np.empty((n_cfg, n_pts, S))
    LBS, LBL = np.empty((n_cfg, n_pts, S)), np.empty((n_cfg, n_pts, S))
    for s, link in enumerate(robot.sdf.sdfs):
        bb = np.asarray(link.bb, dtype=np.float64)
        rl = [float(r[0]) for r in link.ranges]; rh = [float(r[1]) for r in link.ranges]
        margin = grid_prune_margin(link.voxels.raw_data.reshape(tuple(link.voxels.shape)), rl, rh, bb.astype(np.float32))
        R, t = M[s, :, :3, :3], M[s, :, :3, 3]
        q = np.einsum("cij,pj->cpi", R, pts) + t[:, None]
        v, _ = link(torch.from_numpy(q.reshape(-1, 3)).float())
        V[:, :, s] = v.reshape(n_cfg, n_pts).numpy()
        EX[:, :, s] = np.linalg.norm(np.clip(np.maximum(bb[:, 0] - q, q - bb[:, 1]), 0, None), axis=-1) - margin
        cen, hl = 0.5 * (bb[:, 0] + bb[:, 1]), 0.5 * (bb[:, 1] - bb[:, 0])
        c_obj = np.einsum("cji,cj->ci", R, cen - t)                       # R^T (c - t)
        LBS[:, :, s] = np.linalg.norm(pts[None] - c_obj[:, None], axis=-1) - np.linalg.norm(hl) - margin
        a = int(np.argmin(hl))
        LBL[:, :, s] = np.abs(q[..., a] - cen[a]) - hl[a] - margin
        if s == 0:
            print(f"link AABB {2 * hl.round(4)} m, sphere radius {np.linalg.norm(hl):.3f} m, thin axis {a}, "
                  f"prune_margin {margin:.4f} m")
    ref = V.min(-1)
    print(f"{n_cfg} configurations x {n_pts} points, {S} links; per (point, 32-configuration warp step):")
    print(f"{'bound':8s} {'visits':>7s} {'lookups/lane':>13s} {'wasted':>7s}")
    for name, lb in (("sphere", LBS), ("slab", LBL), ("max", np.maximum(LBS, LBL)), ("aabb", EX)):
        vis, looks, wasted, best = simulate(V, EX, lb)
        assert np.array_equal(best, ref[:best.shape[0]]), f"{name}: pruning must be exact"
        print(f"{name:8s} {vis:7.3f} {looks / 32:13.3f} {wasted:7.3f}")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:]))
