"""Paired RobotSDF queries: every joint configuration checked against its own points (RobotSDF.paired), on the
synthetic 7-DOF arm (8 links, per-link CachedSDF(res=0.02, padding=1.0)) -- against the two ways to get the same
numbers without a paired query, timed in rounds that alternate with it:

  loop   one query_at launch per configuration (cfg_begin=c, cfg_count=1) into one result buffer
  cross  (only at 200 x 10 000) the cross product __call__ over all A * P points, then its diagonal

    python scripts/bench_c4paired.py [--steps K] [--warmup W] [--rounds R] [--shapes 200x10000,4096x2048,65536x64]

One GPU.  Device time per step from CUDA events around K steps of each arm.  Prints one JSON line per shape
(A configurations x P points each): pairs per second per arm, whether the arms' outputs are bit-identical, and the
card's name and power limit.  Table caches go to a temporary directory that is removed at exit."""
import json
import sys

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def main():
    with c4bench.session(10, 2, 3, shapes="200x10000,4096x2048,65536x64") as (args, tmp):
        shapes = [tuple(int(x) for x in s.split("x")) for s in args.shapes.split(",")]
        info = c4bench.card()
        robot = c4bench.make_robot("nearest", tmp)
        for A, P in shapes:
            robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
            comp = robot.sdf
            own = c4bench.uniform(A * P, seed=4).cuda().reshape(A, P, 3)
            val = torch.empty(A * P, device="cuda")
            grad = torch.empty(A * P, 3, device="cuda")

            def paired(_):
                return robot.paired(own)

            def loop(_):
                for c in range(A):
                    comp.query_at(own[c], val.data_ptr(), grad.data_ptr(), cfg_begin=c, cfg_count=1)
                return val, grad

            idx = torch.arange(A, device="cuda")

            def cross(_):
                v, g = robot(own.reshape(-1, 3))               # [A, A * P]
                return v.view(A, A, P)[idx, idx], g.view(A, A, P, 3)[idx, idx]

            arms = {"paired": paired, "loop": loop}
            if (A, P) == (200, 10_000):
                arms["cross"] = cross
            ms, med = c4bench.alternate(arms, args)
            outs = {k: f(0) for k, f in arms.items()}
            ref_v, ref_g = outs["paired"]
            ref_v, ref_g = ref_v.reshape(-1), ref_g.reshape(-1, 3)
            equal = all(torch.equal(v.reshape(-1), ref_v) and torch.equal(g.reshape(-1, 3), ref_g)
                        for v, g in outs.values())
            del outs
            print(json.dumps({
                "workload": f"RobotSDF.paired, synthetic 7-DOF arm (8 links, CachedSDF res=0.02 pad=1.0) x {A} "
                            f"configurations x {P} points each, value+gradient",
                "n_cfg": A, "n_pts_per_cfg": P, "unit": "pairs/s",
                "pairs_per_s": {k: A * P / (m * 1e-3) for k, m in med.items()},
                "ms_per_step": med, "rounds_ms": ms, "arms_bit_equal": equal,
                "steps": args.steps, "warmup": args.warmup, "card": info}), flush=True)
            torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    sys.exit(main())
