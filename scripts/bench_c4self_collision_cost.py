"""Self-collision-cost queries: ComposedSDF.query_self_collision_cost (one fused kernel) against the composition route
it is defined by, ComposedSDF._composed_self_collision_cost called directly (per source link and chunk of
configurations: the link points posed by pvb_transform_points_paired, query_paired on the allowed links, the hinge
terms in fp64 and one masked sum per target in torch), on the 8-link arm with the default pairs (self_collision_pairs)
and link_surface_points.

    python scripts/bench_c4self_collision_cost.py [--steps K] [--warmup W] [--rounds R]

Shapes (A configurations x points per link): 200 x 1024, 4096 x 256 and 65 536 x 64, with nearest, trilinear and
primitive links; margins 0.02 and 0.1 m; joint values uniform in +-pi, so that links pass through one another.  Before
timing, the two arms are asserted to agree within 1e-5 of the sum of |term| of every cost and twist entry.  Device
time per call from CUDA events around K calls after W warm-up calls, the two arms alternating for R rounds, median
reported; pairs/s = A * S * (points per link) / time.  Prints one JSON line per (shape, links, margin) with the card's
name and power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
import json

import torch

import c4bench  # first: puts the repository root on sys.path
import pytorch_volumetric_b200 as pv
from pytorch_volumetric_b200 import _native as nat


def abs_terms(comp, lp, rows, m, A):
    """sum|h^2| [A] and sum|tau| [A, S, 6] of every entry, from the composition route's own per-point values."""
    S, K = lp.shape[:2]
    dev = lp.device
    xf = comp._xforms_on(dev).reshape(S, A, 4, 4)
    inv = comp._inv_xforms_on(dev).reshape(S, A, 4, 4)
    ac = torch.zeros(A, dtype=torch.float64, device=dev)
    at = torch.zeros(A, S, 6, dtype=torch.float64, device=dev)
    for i in range(S):
        js = [j for j in range(S) if rows[i][j]]
        if not js:
            continue
        sub = pv.ComposedSDF([comp.sdfs[j] for j in js], None)
        sub.set_transforms(pv.Transform3d(matrix=xf[js].reshape(-1, 4, 4)), batch_dim=(A,))
        jt = torch.tensor(js, device=dev)
        for c0 in range(0, A, 8192):
            cc = min(8192, A - c0)
            w_i = inv[i, c0:c0 + cc].contiguous()
            own = lp[i].float().expand(cc, K, 3).contiguous()
            x = torch.empty(cc, K, 3, device=dev)
            nat.check(nat.lib().pvb_transform_points_paired(nat.ptr(w_i), cc, nat.ptr(own), K, nat.ptr(x),
                                                            nat.stream_ptr(dev)), "pvb_transform_points_paired")
            v, g, w = sub.query_paired(x, cfg_begin=c0, cfg_count=cc, return_which=True)
            v, g, w = v.reshape(cc, K).double(), g.reshape(cc, K, 3).double(), jt[w.long()].reshape(cc, K)
            h = (m - v).clamp_min(0.0)
            tau = (torch.cat([g, torch.linalg.cross(x.double(), g, dim=-1)], -1) * (2 * h)[..., None]).abs()
            ac[c0:c0 + cc] += (h * h).sum(-1)
            for j in js:
                at[c0:c0 + cc, j] += (tau * (w == j)[..., None]).sum(-2)
            at[c0:c0 + cc, i] += tau.sum(-2)
    return ac, at


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
                p = lp.reshape(-1, 3).float().contiguous()
                for margin in (0.02, 0.1):
                    m = comp._collision_cost_margin(margin)             # rounded to fp32, as the query does
                    arms = {"fused": lambda i: comp.query_self_collision_cost(lp, allowed, m),
                            "composition": lambda i: comp._composed_self_collision_cost(p, K, rows, m, 0, A)}
                    got, ref = arms["fused"](0), arms["composition"](0)
                    ac, at = abs_terms(comp, lp, rows, m, A)
                    err_c = float(((got[0].double() - ref[0].double()).abs() / ac.clamp_min(1e-300)).max())
                    err_t = float(((got[1].double() - ref[1].double()).abs() / at.clamp_min(1e-300)).max())
                    assert err_c <= 1e-5 and err_t <= 1e-5, (name, kind, margin, err_c, err_t)
                    contributing = int((got[0] > 0).sum())
                    del got, ref, ac, at
                    rounds, ms = c4bench.alternate(arms, args)
                    pairs = A * S * K
                    line = {"shape": name, "links": kind, "margin": margin, "n_cfg": A, "points_per_link": K,
                            "n_links": S, "fused_ms": ms["fused"], "fused_pairs_per_s": pairs / (ms["fused"] * 1e-3),
                            "composition_ms": ms["composition"],
                            "composition_pairs_per_s": pairs / (ms["composition"] * 1e-3),
                            "speedup": ms["composition"] / ms["fused"], "max_rel_err_cost": err_c,
                            "max_rel_err_twist": err_t, "configurations_with_cost": contributing,
                            "rounds_ms": rounds, "steps": args.steps, "warmup": args.warmup, "gpu": gpu}
                    print(json.dumps(line), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
