"""Host-side model of the C4 pruning: how many link lookups per (configuration, point) pair does a visiting order
cost?  Uses the oracle port (CPU) for the true per-link values and the same bounds as the kernels
(dist(q, link AABB) - prune_margin).  Prints the count for index order, bit-reversed order, the best static order
found by greedy construction, per-pair best-first (needs an extra bound pass) and the floor (only links whose bound
is below the final minimum)."""
import itertools
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


def main(n_cfg=24, n_pts=4000):
    tp_open3d.QUERY_METHOD = "bvh"
    d = tempfile.mkdtemp(prefix="pvb_arm_cpu_")
    urdf, end = workloads.write_arm(d)
    chain = opk.build_serial_chain_from_urdf(open(urdf).read(), end)
    robot = port.RobotSDFPort(chain, path_prefix=d, link_sdf_factory=port.cache_link_sdf_factory_port(0.02, 1.0))
    robot.set_joint_configuration(workloads.arm_configurations(n_cfg))
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    pts = workloads.uniform_points(n_pts, lo, hi, seed=4)
    S = len(robot.sdf.sdfs)
    M = robot.object_to_link.get_matrix().reshape(S, n_cfg, 4, 4)
    vals, lbs = [], []
    for s, link in enumerate(robot.sdf.sdfs):
        q = pts @ M[s, :, :3, :3].transpose(-1, -2) + M[s, :, :3, 3].unsqueeze(1)         # (cfg, P, 3)
        v, _ = link(q.reshape(-1, 3))
        bb = np.asarray(link.bb, dtype=np.float64)
        rl = [float(r[0]) for r in link.ranges]; rh = [float(r[1]) for r in link.ranges]
        margin = grid_prune_margin(link.voxels.raw_data.reshape(tuple(link.voxels.shape)), rl, rh, bb.astype(np.float32))
        dist = torch.clamp(torch.maximum(torch.as_tensor(bb[:, 0]) - q.double(), q.double() - torch.as_tensor(bb[:, 1])),
                           min=0).norm(dim=-1)
        vals.append(v.reshape(n_cfg, n_pts).double()); lbs.append(dist - margin)
    V = torch.stack(vals, -1).reshape(-1, S).numpy(); LB = torch.stack(lbs, -1).reshape(-1, S).numpy()

    def cost(order):
        best = np.full(len(V), np.inf); n = np.zeros(len(V))
        for s in order:
            ev = LB[:, s] <= best
            n += ev
            best = np.where(ev, np.minimum(best, V[:, s]), best)
        return n.mean()

    def bitrev(n):
        bits = max(1, (n - 1).bit_length())
        return [r for r in (int(format(i, f"0{bits}b")[::-1], 2) for i in range(1 << bits)) if r < n]

    print("links", S, "pairs", len(V))
    print("index order      ", round(cost(range(S)), 3))
    print("bit-reversed     ", round(cost(bitrev(S)), 3), bitrev(S))
    # greedy static order: next = the link that minimises the cost of the prefix
    order, rest = [], list(range(S))
    while rest:
        c = {s: cost(order + [s] + [r for r in rest if r != s]) for s in rest}
        nxt = min(c, key=c.get); order.append(nxt); rest.remove(nxt)
    print("greedy static    ", round(cost(order), 3), order)
    if S <= 8:
        best = min(itertools.permutations(range(S)), key=lambda o: cost(o)) if len(V) <= 20000 else None
        if best is not None:
            print("optimal static   ", round(cost(best), 3), list(best))
    first = LB.argmin(1)
    bf = np.take_along_axis(V, first[:, None], 1)[:, 0]
    print("per-pair best-first then index", round(1 + ((LB <= bf[:, None]).sum(1) - 1).mean(), 3), "(upper bound)")
    print("floor            ", round((LB <= V.min(1)[:, None]).sum(1).mean(), 3))
    w = V.argmin(1)
    print("argmin histogram ", np.bincount(w, minlength=S).tolist())


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:]))
