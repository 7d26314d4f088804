"""Self-clearance queries: ComposedSDF.query_self_clearance (one fused kernel and its finish) against the composition
route it is defined by, ComposedSDF._composed_self_clearance called directly (per source link: the link points posed
by pvb_transform_points_paired, query_paired_clearance on the allowed links, then the torch minimum over sources), on
the 8-link arm with the default pairs (self_collision_pairs) and link_surface_points.

    python scripts/bench_c4self_clearance.py [--steps K] [--warmup W] [--rounds R]

Shapes (A configurations x points per link): 200 x 1024, 4096 x 256 and 65 536 x 64, with nearest, trilinear and
primitive links; joint values uniform in +-pi, so that links pass through one another.  Both arms are asserted to give
identical values, gradients and indices.  Device time per step from CUDA events around K steps after W warm-up steps,
the two arms alternating for R rounds; pairs/s = A * S * (points per link) / time.  Prints one JSON line per shape with
the card's name and power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
import argparse
import json
import math
import os
import shutil
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_c4swept import make_robot  # noqa: E402
from bench_c4tri import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_c4self_clearance.py needs a CUDA device")
    gpu = card()
    tmp = tempfile.mkdtemp(prefix="pvb_c4self_")
    try:
        robots = {k: make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        for name, A, K in (("a200_k1024", 200, 1024), ("a4096_k256", 4096, 256), ("a65536_k64", 65_536, 64)):
            g = torch.Generator().manual_seed(A)
            q = ((torch.rand(A, 7, generator=g, dtype=torch.float64) * 2 - 1) * math.pi).float().cuda()
            for kind, robot in robots.items():
                robot.set_joint_configuration(q)
                comp = robot.sdf
                lp = robot.link_surface_points(num_points=K, seed=0)
                allowed = robot.self_collision_pairs()
                S = lp.shape[0]
                _, rows = comp._self_clearance_args(lp, allowed)
                p = lp.reshape(-1, 3).contiguous()
                arms = {"fused": lambda i: comp.query_self_clearance(lp, allowed, return_which=True),
                        "composition": lambda i: comp._composed_self_clearance(p, K, rows, 0, A, True)}
                got, ref = arms["fused"](0), arms["composition"](0)
                identical = all(torch.equal(a, b) for a, b in zip(got, ref))
                assert identical, (name, kind)
                negative = int((got[0] < 0).sum())
                del got, ref
                rounds = {k: [] for k in arms}
                for _ in range(args.rounds):
                    for k, step in arms.items():
                        rounds[k].append(timed(step, args.steps, args.warmup))
                ms = {k: statistics.median(v) for k, v in rounds.items()}
                pairs = A * S * K
                line = {"shape": name, "links": kind, "n_cfg": A, "points_per_link": K, "n_links": S,
                        "fused_ms": ms["fused"], "fused_pairs_per_s": pairs / (ms["fused"] * 1e-3),
                        "composition_ms": ms["composition"],
                        "composition_pairs_per_s": pairs / (ms["composition"] * 1e-3),
                        "speedup": ms["composition"] / ms["fused"], "outputs_identical": identical,
                        "configurations_in_collision": negative, "rounds_ms": rounds, "steps": args.steps,
                        "warmup": args.warmup, "gpu": gpu}
                print(json.dumps(line), flush=True)
            torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
