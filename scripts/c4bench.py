"""What the scripts/bench_c4*.py query-form benchmarks share: the command line, the timing, the robots, the clouds,
the first-point reduction and the error measure.

A script runs inside `session`, which parses its command line, refuses to run without a CUDA device or without
libpvb.so, and removes its temporary directory (meshes, table caches) at exit.  `alternate` times its arms in rounds:
every round runs each arm in turn, K timed steps after W warm-up steps.  The clouds are generated on the CPU from a
seed; callers move them to the GPU."""
import argparse
import contextlib
import math
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import workloads  # noqa: E402

LO = [r[0] for r in workloads.ARM_QUERY_RANGE]
HI = [r[1] for r in workloads.ARM_QUERY_RANGE]


@contextlib.contextmanager
def session(steps, warmup, rounds, **options):
    """Yield (args, tmp): the parsed --steps/--warmup/--rounds with this script's defaults, plus one option per
    keyword (n_cfg=200 gives --n-cfg, of the default's type), and a temporary directory removed at exit."""
    script = os.path.basename(sys.argv[0])
    ap = argparse.ArgumentParser(prog=script)
    ap.add_argument("--steps", type=int, default=steps, help=f"timed steps per arm and round (default: {steps})")
    ap.add_argument("--warmup", type=int, default=warmup, help=f"warm-up steps before each timed window "
                                                               f"(default: {warmup})")
    ap.add_argument("--rounds", type=int, default=rounds, help=f"alternating rounds (default: {rounds})")
    for name, default in options.items():
        ap.add_argument("--" + name.replace("_", "-"), type=type(default), default=default,
                        help=f"(default: {default})")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit(f"{script} measures the GPU path and needs a CUDA device")
    from pytorch_volumetric_b200 import _native
    if _native.lib_missing():
        sys.exit("libpvb.so is missing: build it first (python -c \"import __graft_entry__ as g; g.build()\")")
    tmp = tempfile.mkdtemp(prefix=f"pvb_{os.path.splitext(script)[0]}_")
    try:
        yield args, tmp
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


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


def alternate(arms, args, empty_cache=False):
    """Time every arm step(i) of {name: step} for args.rounds rounds, the arms in turn within a round: the per-round
    ms per step {name: [ms, ...]} and their medians {name: ms}.  empty_cache=True returns the allocator's cached blocks
    to the device after each arm.  Each script keeps the choice its published numbers were taken with: a timed step
    allocates its output while the previous step's is still alive, so after an empty cache a single warm-up step
    leaves the first timed step to allocate from the device, which shows in the median at --warmup 1.  From two
    warm-up steps on, both outputs come from the cache and the choice does not show in the times."""
    rounds = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, step in arms.items():
            rounds[k].append(timed(step, args.steps, args.warmup))
            if empty_cache:
                torch.cuda.empty_cache()
    return rounds, {k: statistics.median(v) for k, v in rounds.items()}


def make_robot(kind, tmp):
    """The 8-link arm with cached "nearest" or "trilinear" links (CachedSDF res=0.02, padding=1.0), or the primitive
    arm (workloads.write_primitive_arm) with "primitive" links, on the GPU; its files go under tmp."""
    import pytorch_volumetric_b200 as pv
    if kind == "primitive":
        urdf, end = workloads.write_primitive_arm(os.path.join(tmp, "prim"))
        return pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"),
                           primitive_visuals=True)
    d = os.path.join(tmp, kind)
    urdf, end = workloads.write_arm(d)
    return pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"), path_prefix=d,
                       link_sdf_cls=pv.cache_link_sdf_factory(resolution=0.02, padding=1.0, device="cuda",
                                                              cache_path=os.path.join(d, "cache.pkl"),
                                                              interpolation=kind))


def uniform(n, seed):
    """[n, 3] uniform in workloads.ARM_QUERY_RANGE."""
    return workloads.uniform_points(n, LO, HI, seed=seed)


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


def clouds(kind, A, seg_shape, seed):
    """[A, *seg_shape, 3]: a "uniform" cloud per configuration, or the "scene" moved per configuration by a seeded
    offset."""
    n = math.prod(seg_shape)
    if kind == "uniform":
        pts = uniform(A * n, seed).reshape(A, n, 3)
    else:
        g = torch.Generator().manual_seed(seed)
        offset = torch.randn(A, 1, 3, generator=g) * torch.tensor([0.1, 0.1, 0.03])
        pts = scene_points(n, seed)[None] + offset
    return pts.reshape(A, *seg_shape, 3).contiguous()


def crossing_configurations(A):
    """[A, 7] joint values uniform in +-pi on the GPU, seeded by A, so that the arm's links pass through one another."""
    g = torch.Generator().manual_seed(A)
    return ((torch.rand(A, 7, generator=g, dtype=torch.float64) * 2 - 1) * math.pi).float().cuda()


def first_min(v, g):
    """Values v [..., N] and gradients g [..., N, 3]: per row of v, the first point attaining the minimum over N, as
    (value [R], gradient [R, 3], index [R]) over the R rows."""
    N = v.shape[-1]
    v, g = v.reshape(-1, N), g.reshape(-1, N, 3)
    i = (v == v.amin(dim=-1, keepdim=True)).int().argmax(dim=-1, keepdim=True)
    return v.gather(-1, i)[:, 0], g.gather(-2, i[..., None].expand(-1, 1, 3))[:, 0], i[:, 0]


def rel_err(got, ref, bound):
    """Largest |got - ref| / bound over the entries, got in ref's shape."""
    return float(((got.double().reshape(ref.shape) - ref).abs() / bound.clamp_min(1e-30)).max())
