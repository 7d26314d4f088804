"""Paired clearance queries: RobotSDF.paired_clearance(points) -- every configuration against its own cloud, the first
point of every segment attaining the minimum, with its value and gradient -- against today's way to get it,
robot.paired(points) followed by the same first-index reduction over the points in torch, on the 8-link arm.

    python scripts/bench_c4paired_clearance.py [--steps K] [--warmup W] [--rounds R]

Shapes (A configurations x points per configuration): 200 x 10^4, 4096 x 2048, 65 536 x 64 and 1024 x (8 segments x
256), with nearest, trilinear and primitive links, and two clouds: uniform in ARM_QUERY_RANGE (a fresh cloud per
configuration), and the tabletop scene of c4bench.scene_points shifted per configuration by a seeded offset
(every environment differs; most points are away from the arm).  Both arms are asserted to give identical values,
gradients and point indices.  Device time per step from CUDA events around K steps after W warm-up steps, the two arms
alternating for R rounds; pairs/s = A * (points per configuration) / time.  Prints one JSON line per shape with the
card's name and power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
import json

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def main():
    with c4bench.session(20, 3, 3) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        shapes = [("a200_n1e4", 200, (10_000,)), ("a4096_n2048", 4096, (2048,)), ("a65536_n64", 65_536, (64,)),
                  ("a1024_seg8_n256", 1024, (8, 256))]
        for name, A, seg_shape in shapes:
            for cloud in ("uniform", "scene"):
                bufs = [c4bench.clouds(cloud, A, seg_shape, 300 + i).cuda() for i in range(2)]
                for kind, robot in robots.items():
                    robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
                    # robot.paired(points) [A, *B, N], then the first point attaining the minimum of every
                    # (configuration, segment)
                    arms = {"paired_clearance": lambda i, r=robot: r.paired_clearance(bufs[i % 2], return_argmin=True),
                            "paired_then_min": lambda i, r=robot: c4bench.first_min(*r.paired(bufs[i % 2]))}
                    cv, cg, ci, _ = robot.paired_clearance(bufs[0], return_argmin=True)
                    rv, rg, ri = c4bench.first_min(*robot.paired(bufs[0]))
                    identical = bool(torch.equal(cv.reshape(-1), rv) and torch.equal(cg.reshape(-1, 3), rg)
                                     and torch.equal(ci.reshape(-1), ri))
                    assert identical, (name, cloud, kind)
                    del cv, cg, ci, rv, rg, ri
                    rounds, ms = c4bench.alternate(arms, args)
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


if __name__ == "__main__":
    main()
