"""Swept queries: RobotSDF.swept(points) -- at every point the first configuration attaining the minimum over all
installed configurations, with its value and gradient -- against today's way to get it, robot(points) followed by
the same lexicographic reduction in torch (min value, first configuration), on the 8-link arm.

    python scripts/bench_c4swept.py [--steps K] [--warmup W] [--rounds R]

Shapes: C4 (8 cached nearest-voxel links x 200 configurations x 10^5 points), C4 with trilinear links, C4 with
primitive links (workloads.write_primitive_arm), 4096 x 10^5, and 4096 x 10^6 with the swept arm only (the cross
product, 65.5 GB, does not fit beside anything else on an 80 GB card; the baseline is reported as not run).
Both arms are asserted to give identical values, gradients and configuration indices at every shape where both run.
Device time per step from CUDA events around K steps after W warm-up steps, the two arms alternating for R rounds;
pairs/s = |A| * N / time.  Prints one JSON line per shape with the card's name and power limit.  Meshes and table
caches go to a temporary directory that is removed at exit."""
import json

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def reduce_cross_product(robot, pts):
    """robot(pts) [A, N], then the first configuration attaining the minimum at every point."""
    v, g = robot(pts)
    v, g = v.reshape(-1, v.shape[-1]), g.reshape(-1, g.shape[-2], 3)
    c = (v == v.amin(dim=0)).int().argmax(dim=0)
    return v.gather(0, c[None])[0], g.gather(0, c[None, :, None].expand(1, c.numel(), 3))[0], c


def main():
    with c4bench.session(20, 3, 3) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        shapes = [("c4", "nearest", 200, 100_000, True), ("c4_trilinear", "trilinear", 200, 100_000, True),
                  ("c4_primitive", "primitive", 200, 100_000, True), ("a4096_n1e5", "nearest", 4096, 100_000, True),
                  ("a4096_n1e6", "nearest", 4096, 1_000_000, False)]
        for name, kind, A, N, baseline in shapes:
            robot = robots[kind]
            robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
            bufs = [c4bench.uniform(N, seed=100 + i).cuda() for i in range(2)]
            arms = {"swept": lambda i, r=robot: r.swept(bufs[i % 2], return_argmin=True)}
            identical = None
            if baseline:
                arms["cross_product_then_min"] = lambda i, r=robot: reduce_cross_product(r, bufs[i % 2])
                sv, sg, sc, _ = robot.swept(bufs[0], return_argmin=True)
                rv, rg, rc = reduce_cross_product(robot, bufs[0])
                identical = bool(torch.equal(sv, rv) and torch.equal(sg, rg) and torch.equal(sc, rc))
                assert identical, name
                del sv, sg, sc, rv, rg, rc
            rounds, ms = c4bench.alternate(arms, args, empty_cache=True)
            line = {"shape": name, "links": kind, "n_cfg": A, "n_pts": N,
                    "swept_ms": ms["swept"], "swept_pairs_per_s": A * N / (ms["swept"] * 1e-3),
                    "baseline_ms": ms.get("cross_product_then_min"),
                    "baseline_pairs_per_s": (A * N / (ms["cross_product_then_min"] * 1e-3)) if baseline else None,
                    "speedup": (ms["cross_product_then_min"] / ms["swept"]) if baseline else None,
                    "baseline_note": None if baseline else "not run: the cross product needs 16 * A * N bytes",
                    "outputs_identical": identical, "rounds_ms": rounds, "steps": args.steps,
                    "warmup": args.warmup, "gpu": gpu}
            print(json.dumps(line), flush=True)
            del bufs, arms
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
