"""C4 with trilinear links: RobotSDF of the synthetic 7-DOF arm (8 links, per-link
CachedSDF(res=0.02, padding=1.0, interpolation="trilinear")) x 200 joint configurations x 100 000 points, value +
gradient, on the fused kernels -- against the same query with the links wrapped in an opaque ObjectFrameSDF (the
generic per-link composition of ComposedSDF), timed in rounds alternating with the fused path.

    python scripts/bench_c4tri.py [--steps K] [--warmup W] [--rounds R] [--n-cfg 200] [--n-pts 100000]

One GPU.  Device time per step from CUDA events around K steps of the public call (3 rotating point buffers, as
bench.py's C4).  Prints one JSON line: fused `ms_per_step` / `value` (pairs per second), `generic_path_ms`, the
per-round times and the card's name and power limit.  Table caches go to a temporary directory that is removed at
exit.  The reference project has no trilinear interpolation, so there is no reference arm."""
import json
import sys

import torch

import c4bench  # first: puts the repository root on sys.path
import pytorch_volumetric_b200 as pv
import workloads


class Opaque(pv.ObjectFrameSDF):          # no native descriptor: ComposedSDF takes its generic path
    def __init__(self, inner):
        self.inner = inner

    def __call__(self, p):
        return self.inner(p)

    def surface_bounding_box(self, **kw):
        return self.inner.surface_bounding_box(**kw)


def main():
    with c4bench.session(50, 5, 3, n_cfg=200, n_pts=100_000) as (args, tmp):
        robot = c4bench.make_robot("trilinear", tmp)
        robot.set_joint_configuration(workloads.arm_configurations(args.n_cfg).cuda())
        dev = [c4bench.uniform(args.n_pts, seed=4 + b).cuda() for b in range(3)]
        generic = pv.ComposedSDF([Opaque(s) for s in robot.sdf.sdfs], robot.sdf.obj_frame_to_link_frame)
        arms = {"fused": lambda i: robot(dev[i % 3]), "generic": lambda i: generic(dev[i % 3])}
        rounds, med = c4bench.alternate(arms, args)
        # the two paths agree (values and argmin bit for bit, tests/test_gpu_trilinear_composed.py): check once here
        vf, _ = robot(dev[0])
        vg, _ = generic(dev[0])
        same_values = bool(torch.equal(vf, vg))
    ms = med["fused"]
    print(json.dumps({
        "workload": f"C4 RobotSDF synthetic 7-DOF arm (8 links, CachedSDF res=0.02 pad=1.0 interpolation='trilinear') "
                    f"x {args.n_cfg} configurations x {args.n_pts} points, value+gradient",
        "unit": "pairs/s", "value": args.n_cfg * args.n_pts / (ms * 1e-3), "ms_per_step": ms,
        "generic_path_ms": med["generic"], "generic_over_fused": med["generic"] / ms,
        "rounds": {"fused_ms_per_step": rounds["fused"], "generic_ms_per_step": rounds["generic"]},
        "steps": args.steps, "warmup": args.warmup, "fused_equals_generic_values": same_values,
        "reference_arm": None, "reference_arm_reason": "the reference has no trilinear interpolation",
        "card": c4bench.card()}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
