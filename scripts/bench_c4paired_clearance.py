"""Paired clearance queries: RobotSDF.paired_clearance(points) -- every configuration against its own cloud, the first
point of every segment attaining the minimum, with its value and gradient -- against today's way to get it,
robot.paired(points) followed by the same first-index reduction over the points in torch, on the 8-link arm.

    python scripts/bench_c4paired_clearance.py [--steps K] [--warmup W] [--rounds R]

Shapes (A configurations x points per configuration): 200 x 10^4, 4096 x 2048, 65 536 x 64 and 1024 x (8 segments x
256), with nearest, trilinear and primitive links, and two clouds: uniform in ARM_QUERY_RANGE (a fresh cloud per
configuration), and the tabletop scene of bench_c4clearance.scene_points shifted per configuration by a seeded offset
(every environment differs; most points are away from the arm).  Both arms are asserted to give identical values,
gradients and point indices.  Device time per step from CUDA events around K steps after W warm-up steps, the two arms
alternating for R rounds; pairs/s = A * (points per configuration) / time.  Prints one JSON line per shape with the
card's name and power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
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
from bench_c4clearance import scene_points  # noqa: E402
from bench_c4swept import make_robot  # noqa: E402
from bench_c4tri import card, timed  # noqa: E402


def reduce_paired(robot, pts):
    """robot.paired(pts) [A, *B, N], then the first point attaining the minimum of every (configuration, segment)."""
    v, g = robot.paired(pts)
    N = v.shape[-1]
    v, g = v.reshape(-1, N), g.reshape(-1, N, 3)
    i = (v == v.amin(dim=-1, keepdim=True)).int().argmax(dim=-1, keepdim=True)
    return v.gather(-1, i)[:, 0], g.gather(-2, i[..., None].expand(-1, 1, 3))[:, 0], i[:, 0]


def clouds(kind, A, seg_shape, seed):
    """[A, *seg_shape, 3] on the GPU: a uniform cloud per configuration, or the scene moved per configuration."""
    lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
    n = 1
    for s in seg_shape:
        n *= s
    if kind == "uniform":
        pts = workloads.uniform_points(A * n, lo, hi, seed=seed).reshape(A, n, 3)
    else:
        g = torch.Generator().manual_seed(seed)
        offset = torch.randn(A, 1, 3, generator=g) * torch.tensor([0.1, 0.1, 0.03])
        pts = scene_points(n, seed)[None] + offset
    return pts.reshape(A, *seg_shape, 3).contiguous().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_c4paired_clearance.py needs a CUDA device")
    gpu = card()
    tmp = tempfile.mkdtemp(prefix="pvb_c4pclearance_")
    try:
        robots = {k: make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        shapes = [("a200_n1e4", 200, (10_000,)), ("a4096_n2048", 4096, (2048,)), ("a65536_n64", 65_536, (64,)),
                  ("a1024_seg8_n256", 1024, (8, 256))]
        for name, A, seg_shape in shapes:
            for cloud in ("uniform", "scene"):
                bufs = [clouds(cloud, A, seg_shape, 300 + i) for i in range(2)]
                for kind, robot in robots.items():
                    robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
                    arms = {"paired_clearance": lambda i, r=robot: r.paired_clearance(bufs[i % 2], return_argmin=True),
                            "paired_then_min": lambda i, r=robot: reduce_paired(r, bufs[i % 2])}
                    cv, cg, ci, _ = robot.paired_clearance(bufs[0], return_argmin=True)
                    rv, rg, ri = reduce_paired(robot, bufs[0])
                    identical = bool(torch.equal(cv.reshape(-1), rv) and torch.equal(cg.reshape(-1, 3), rg)
                                     and torch.equal(ci.reshape(-1), ri))
                    assert identical, (name, cloud, kind)
                    del cv, cg, ci, rv, rg, ri
                    rounds = {k: [] for k in arms}
                    for _ in range(args.rounds):
                        for k, step in arms.items():
                            rounds[k].append(timed(step, args.steps, args.warmup))
                    ms = {k: statistics.median(v) for k, v in rounds.items()}
                    pairs = A * bufs[0][0].numel() // 3
                    line = {"shape": name, "links": kind, "cloud": cloud, "n_cfg": A, "points": list(seg_shape),
                            "paired_clearance_ms": ms["paired_clearance"],
                            "paired_clearance_pairs_per_s": pairs / (ms["paired_clearance"] * 1e-3),
                            "baseline_ms": ms["paired_then_min"],
                            "baseline_pairs_per_s": pairs / (ms["paired_then_min"] * 1e-3),
                            "speedup": ms["paired_then_min"] / ms["paired_clearance"],
                            "outputs_identical": identical, "rounds_ms": rounds, "steps": args.steps,
                            "warmup": args.warmup, "gpu": gpu}
                    print(json.dumps(line), flush=True)
                del bufs
                torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
