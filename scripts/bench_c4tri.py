"""C4 with trilinear links: RobotSDF of the synthetic 7-DOF arm (8 links, per-link
CachedSDF(res=0.02, padding=1.0, interpolation="trilinear")) x 200 joint configurations x 100 000 points, value +
gradient, on the fused kernels -- against the same query with the links wrapped in an opaque ObjectFrameSDF (the
generic per-link composition of ComposedSDF), timed in rounds alternating with the fused path.

    python scripts/bench_c4tri.py [--steps K] [--warmup W] [--rounds R] [--n-cfg 200] [--n-pts 100000]

One GPU.  Device time per step from CUDA events around K steps of the public call (3 rotating point buffers, as
bench.py's C4).  Prints one JSON line: fused `ms_per_step` / `value` (pairs per second), `generic_path_ms`, the
per-round times and the card's name and power limit.  Table caches go to a temporary directory that is removed at
exit.  The reference project has no trilinear interpolation, so there is no reference arm."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import workloads  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in out.stdout.strip().split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:          # noqa: BLE001  (the numbers stay valid without it; say why it is missing)
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "error": repr(e)[:200]}


def timed(step, steps, warmup):
    out = None
    for i in range(warmup):
        out = step(i)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
        out = step(i)
    t1.record()
    torch.cuda.synchronize()
    del out
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n-cfg", type=int, default=200)
    ap.add_argument("--n-pts", type=int, default=100_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_c4tri.py measures the GPU path and needs a CUDA device")
    import pytorch_volumetric_b200 as pv
    from pytorch_volumetric_b200 import _native
    if _native.lib_missing():
        raise SystemExit("libpvb.so is missing: build it first (python -c \"import __graft_entry__ as g; g.build()\")")

    tmp = tempfile.mkdtemp(prefix="pvb_c4tri_")
    try:
        urdf, end = workloads.write_arm(os.path.join(tmp, "arm"))
        chain = pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda")
        robot = pv.RobotSDF(chain, path_prefix=os.path.dirname(urdf),
                            link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                                   cache_path=os.path.join(tmp, "cache.pkl"),
                                                                   interpolation="trilinear"))
        robot.set_joint_configuration(workloads.arm_configurations(args.n_cfg).cuda())
        lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
        dev = [workloads.uniform_points(args.n_pts, lo, hi, seed=4 + b).cuda() for b in range(3)]

        class Opaque(pv.ObjectFrameSDF):          # no native descriptor: ComposedSDF takes its generic path
            def __init__(self, inner):
                self.inner = inner

            def __call__(self, p):
                return self.inner(p)

            def surface_bounding_box(self, **kw):
                return self.inner.surface_bounding_box(**kw)

        generic = pv.ComposedSDF([Opaque(s) for s in robot.sdf.sdfs], robot.sdf.obj_frame_to_link_frame)
        fused_ms, generic_ms = [], []
        for _ in range(args.rounds):
            fused_ms.append(timed(lambda i: robot(dev[i % 3]), args.steps, args.warmup))
            generic_ms.append(timed(lambda i: generic(dev[i % 3]), args.steps, args.warmup))
        # the two paths agree (values and argmin bit for bit, tests/test_gpu_trilinear_composed.py): check once here
        vf, _ = robot(dev[0])
        vg, _ = generic(dev[0])
        same_values = bool(torch.equal(vf, vg))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    ms = statistics.median(fused_ms)
    print(json.dumps({
        "workload": f"C4 RobotSDF synthetic 7-DOF arm (8 links, CachedSDF res=0.02 pad=1.0 interpolation='trilinear') "
                    f"x {args.n_cfg} configurations x {args.n_pts} points, value+gradient",
        "unit": "pairs/s", "value": args.n_cfg * args.n_pts / (ms * 1e-3), "ms_per_step": ms,
        "generic_path_ms": statistics.median(generic_ms), "generic_over_fused": statistics.median(generic_ms) / ms,
        "rounds": {"fused_ms_per_step": fused_ms, "generic_ms_per_step": generic_ms},
        "steps": args.steps, "warmup": args.warmup, "fused_equals_generic_values": same_values,
        "reference_arm": None, "reference_arm_reason": "the reference has no trilinear interpolation",
        "card": card()}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
