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
import json
import math

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def main():
    with c4bench.session(20, 3, 3) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        uniform, scene = c4bench.uniform, c4bench.scene_points
        shapes = [("c4", "nearest", 200, uniform, (100_000,), True),
                  ("c4_trilinear", "trilinear", 200, uniform, (100_000,), True),
                  ("c4_primitive", "primitive", 200, uniform, (100_000,), True),
                  ("c4_scene", "nearest", 200, scene, (100_000,), True),
                  ("c4_scene_trilinear", "trilinear", 200, scene, (100_000,), True),
                  ("c4_scene_primitive", "primitive", 200, scene, (100_000,), True),
                  ("a200_seg1000_n1000", "nearest", 200, uniform, (1000, 1000), True),
                  ("a4096_n1e6", "nearest", 4096, uniform, (1_000_000,), False)]
        for name, kind, A, cloud, seg_shape, baseline in shapes:
            robot = robots[kind]
            robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
            n = math.prod(seg_shape)
            bufs = [cloud(n, 200 + i).reshape(*seg_shape, 3).cuda() for i in range(2)]
            arms = {"clearance": lambda i, r=robot: r.clearance(bufs[i % 2], return_argmin=True)}
            identical = None
            if baseline:
                # robot(points) [A, *B, N], then the first point attaining the minimum of every (configuration, segment)
                arms["cross_product_then_min"] = lambda i, r=robot: c4bench.first_min(*r(bufs[i % 2]))
                cv, cg, ci, _ = robot.clearance(bufs[0], return_argmin=True)
                rv, rg, ri = c4bench.first_min(*robot(bufs[0]))
                identical = bool(torch.equal(cv.reshape(-1), rv) and torch.equal(cg.reshape(-1, 3), rg)
                                 and torch.equal(ci.reshape(-1), ri))
                assert identical, name
                del cv, cg, ci, rv, rg, ri
            rounds, ms = c4bench.alternate(arms, args, empty_cache=True)
            pairs = A * n
            line = {"shape": name, "links": kind, "cloud": "scene" if cloud is scene else "uniform",
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


if __name__ == "__main__":
    main()
