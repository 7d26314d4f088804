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
import json

import torch

import c4bench  # first: puts the repository root on sys.path


def main():
    with c4bench.session(20, 3, 3) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        for name, A, K in (("a200_k1024", 200, 1024), ("a4096_k256", 4096, 256), ("a65536_k64", 65_536, 64)):
            q = c4bench.crossing_configurations(A)
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
                rounds, ms = c4bench.alternate(arms, args)
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


if __name__ == "__main__":
    main()
