"""Clearance queries: RobotSDF.clearance(points) -- for every configuration, the first point of every segment
attaining the minimum over the segment, with its value and gradient -- against today's way to get it,
robot(points) followed by the same first-index reduction over the points in torch, on the 8-link arm.

    python scripts/bench_c4clearance.py [--steps K] [--warmup W] [--rounds R]

Shapes: C4 (8 links x 200 configurations x 10^5 points uniform in ARM_QUERY_RANGE) with nearest, trilinear and
primitive links; the same with a scene-like cloud (points on a table plane and on the shells of boxes around the arm,
most of them away from it); 200 configurations x 1000 segments x 1000 points (batched environments); and 4096 x 10^6
with the clearance arm only (the cross product, 65.5 GB, does not fit beside anything else on an 80 GB card; the
baseline is reported as not run).  Both arms are asserted to give identical values, gradients and point indices at
every shape where both run.  Device time per step from CUDA events around K steps after W warm-up steps, the two arms
alternating for R rounds; pairs/s = |A| * (points) / time.  Prints one JSON line per shape with the card's name and
power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import workloads  # noqa: E402
from bench_c4swept import make_robot  # noqa: E402
from bench_c4tri import card, timed  # noqa: E402


def reduce_cross_product(robot, pts):
    """robot(pts) [A, *B, N], then the first point attaining the minimum of every (configuration, segment)."""
    v, g = robot(pts)
    N = v.shape[-1]
    v, g = v.reshape(-1, N), g.reshape(-1, N, 3)
    i = (v == v.amin(dim=-1, keepdim=True)).int().argmax(dim=-1, keepdim=True)
    return v.gather(-1, i)[:, 0], g.gather(-2, i[..., None].expand(-1, 1, 3))[:, 0], i[:, 0]


def scene_points(n, seed):
    """A tabletop scene around the arm: a third of the points on the table plane z = -0.2, the rest on the shells of
    six boxes (shelves, bins, a wall) placed around the workspace; few of them near any configuration."""
    g = torch.Generator().manual_seed(seed)
    n_table = n // 3
    table = torch.rand(n_table, 3, generator=g) * torch.tensor([1.5, 1.0, 0.0]) + torch.tensor([-1.0, -0.5, -0.2])
    boxes = torch.tensor([[-0.9, -0.45, -0.2, 0.3, 0.25, 0.35], [0.2, -0.45, -0.2, 0.25, 0.2, 0.6],
                          [-0.4, 0.3, -0.2, 0.5, 0.15, 0.25], [0.3, 0.25, -0.2, 0.15, 0.2, 0.9],
                          [-0.95, 0.2, 0.4, 0.2, 0.25, 0.3], [-0.3, -0.5, 0.5, 0.6, 0.05, 0.3]])
    m = n - n_table
    k = torch.randint(0, len(boxes), (m,), generator=g)
    lo, size = boxes[k, :3], boxes[k, 3:]
    u = torch.rand(m, 3, generator=g)
    face = torch.randint(0, 6, (m,), generator=g)               # pin one coordinate to a face of the box
    axis, side = face % 3, (face // 3).float()
    u[torch.arange(m), axis] = side
    shell = lo + u * size
    return torch.cat([table, shell])[torch.randperm(n, generator=g)].contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_c4clearance.py needs a CUDA device")
    gpu = card()
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    tmp = tempfile.mkdtemp(prefix="pvb_c4clearance_")
    try:
        robots = {k: make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        uniform = lambda n, s: workloads.uniform_points(n, lo, hi, seed=s)   # noqa: E731
        shapes = [("c4", "nearest", 200, uniform, (100_000,), True),
                  ("c4_trilinear", "trilinear", 200, uniform, (100_000,), True),
                  ("c4_primitive", "primitive", 200, uniform, (100_000,), True),
                  ("c4_scene", "nearest", 200, scene_points, (100_000,), True),
                  ("c4_scene_trilinear", "trilinear", 200, scene_points, (100_000,), True),
                  ("c4_scene_primitive", "primitive", 200, scene_points, (100_000,), True),
                  ("a200_seg1000_n1000", "nearest", 200, uniform, (1000, 1000), True),
                  ("a4096_n1e6", "nearest", 4096, uniform, (1_000_000,), False)]
        for name, kind, A, cloud, seg_shape, baseline in shapes:
            robot = robots[kind]
            robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
            n = 1
            for s in seg_shape:
                n *= s
            bufs = [cloud(n, 200 + i).reshape(*seg_shape, 3).cuda() for i in range(2)]
            arms = {"clearance": lambda i, r=robot: r.clearance(bufs[i % 2], return_argmin=True)}
            identical = None
            if baseline:
                arms["cross_product_then_min"] = lambda i, r=robot: reduce_cross_product(r, bufs[i % 2])
                cv, cg, ci, _ = robot.clearance(bufs[0], return_argmin=True)
                rv, rg, ri = reduce_cross_product(robot, bufs[0])
                identical = bool(torch.equal(cv.reshape(-1), rv) and torch.equal(cg.reshape(-1, 3), rg)
                                 and torch.equal(ci.reshape(-1), ri))
                assert identical, name
                del cv, cg, ci, rv, rg, ri
            rounds = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, step in arms.items():
                    rounds[k].append(timed(step, args.steps, args.warmup))
                    torch.cuda.empty_cache()
            ms = {k: statistics.median(v) for k, v in rounds.items()}
            pairs = A * n
            line = {"shape": name, "links": kind, "cloud": "scene" if cloud is scene_points else "uniform",
                    "n_cfg": A, "points": list(seg_shape),
                    "clearance_ms": ms["clearance"], "clearance_pairs_per_s": pairs / (ms["clearance"] * 1e-3),
                    "baseline_ms": ms.get("cross_product_then_min"),
                    "baseline_pairs_per_s": (pairs / (ms["cross_product_then_min"] * 1e-3)) if baseline else None,
                    "speedup": (ms["cross_product_then_min"] / ms["clearance"]) if baseline else None,
                    "baseline_note": None if baseline else "not run: the cross product needs 16 * A * N bytes",
                    "outputs_identical": identical, "rounds_ms": rounds, "steps": args.steps,
                    "warmup": args.warmup, "gpu": gpu}
            print(json.dumps(line), flush=True)
            del bufs, arms
            torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
