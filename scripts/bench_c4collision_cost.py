"""Collision-cost queries: RobotSDF.collision_cost(points, margin) -- for every configuration and segment, the hinge
cost sum_p max(0, m - d)^2 and its joint gradient -- against today's way to get it: the per-pair query
(robot.sdf.query(..., return_which=True), the kernel behind robot(points), plus the argmin link) followed by the
same cost, twist gradient and joint gradient in torch, on the 8-link arm.

    python scripts/bench_c4collision_cost.py [--steps K] [--warmup W] [--rounds R]

Arms: cached nearest, cached trilinear and primitive links.  Clouds: uniform in ARM_QUERY_RANGE and the tabletop scene
of c4bench.scene_points.  Margins 0.02 and 0.1 m.  Shapes: 200 x 10^5, 4096 x 10^5 and 200 x (1000 segments x 1000).
Device time per call from CUDA events around K calls after W warm-up calls, the two arms alternating for R rounds;
pairs/s = |A| * points / time.  For each arm, the largest error of its cost and joint gradient against the fp64 sum
of the same fp32 per-pair outputs, relative to the sum of |term| of each entry, and the largest difference between the
two arms on the same scale; the fused arm's error is asserted <= 1e-5.  One JSON line per shape
with the card's name and power limit.  Meshes and table caches go to a temporary directory that is removed at exit."""
import json
import math

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def per_pair_cost(robot, pts, m, dtype=torch.float32, cfg_chunk=None):
    """The per-pair query, then cost [A, n_seg], joint gradient [A, n_seg, J] and (fp64 only) the sums of |term| of
    both, in `dtype`, in chunks of cfg_chunk configurations."""
    comp = robot.sdf
    S, L = len(comp.sdfs), pts.shape[-2]
    n_cfg = robot.joint_twists().shape[0]
    p = pts.reshape(-1, L, 3).to(dtype)
    n_seg = p.shape[0]
    jt, moves = robot.joint_twists().to(dtype), robot.joint_moves_link().to(device=pts.device, dtype=dtype)
    step = cfg_chunk or n_cfg
    out = [[], [], [], []]
    for c0 in range(0, n_cfg, step):
        cc = min(step, n_cfg - c0)
        v, g, w = comp.query(pts.reshape(-1, 3), c0, cc, return_which=True)
        v, g, w = v.reshape(cc, n_seg, L).to(dtype), g.reshape(cc, n_seg, L, 3).to(dtype), w.reshape(cc, n_seg, L)
        h = (m - v).clamp_min(0.0)
        out[0].append((h * h).sum(-1))
        twist = torch.empty(cc, n_seg, S, 6, dtype=dtype, device=pts.device)
        abs_tw = torch.empty_like(twist) if dtype == torch.float64 else None
        for s in range(S):
            hs = 2 * h * (w == s)
            gv = g * hs[..., None]
            twist[:, :, s, :3] = gv.sum(-2)
            twist[:, :, s, 3:] = torch.linalg.cross(p.expand_as(gv), gv, dim=-1).sum(-2)
            if abs_tw is not None:
                abs_tw[:, :, s, :3] = gv.abs().sum(-2)
                abs_tw[:, :, s, 3:] = torch.linalg.cross(p.expand_as(gv), gv, dim=-1).abs().sum(-2)
        j = jt[c0:c0 + cc].to(pts.device)
        out[1].append(torch.einsum("absk,js,ajk->abj", twist, moves, j))
        if abs_tw is not None:
            out[2].append((h * h).sum(-1))
            out[3].append(torch.einsum("absk,js,ajk->abj", abs_tw, moves, j.abs()))
    return [torch.cat(o) if o else None for o in out]


def main():
    with c4bench.session(10, 2, 2) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        for A, seg_shape in ((200, (100_000,)), (4096, (100_000,)), (200, (1000, 1000))):
            for kind, robot in robots.items():
                robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
                for cloud in (c4bench.uniform, c4bench.scene_points):
                    n = math.prod(seg_shape)
                    pts = cloud(n, 300).reshape(*seg_shape, 3).cuda()
                    for m in (0.02, 0.1):
                        m = torch.tensor(m, dtype=torch.float32).item()     # the fp32 margin every route uses
                        arms = {"fused": lambda i, r=robot, p=pts, m=m: r.collision_cost(p, m),
                                "per_pair_then_torch": lambda i, r=robot, p=pts, m=m: per_pair_cost(r, p, m)[:2]}
                        rc, rg, ac, ag = per_pair_cost(robot, pts, m, torch.float64, cfg_chunk=256)
                        err, outs = {}, {}
                        for k, f in arms.items():
                            c, g = f(0)
                            outs[k] = (c.reshape(rc.shape).double(), g.reshape(rg.shape).double())
                            err[k] = {"cost": c4bench.rel_err(outs[k][0], rc, ac),
                                      "joint_grad": c4bench.rel_err(outs[k][1], rg, ag)}
                        (fc, fg), (bc, bg) = outs["fused"], outs["per_pair_then_torch"]
                        agree = {"cost": c4bench.rel_err(fc, bc, ac), "joint_grad": c4bench.rel_err(fg, bg, ag)}
                        # the torch arm's own fp32 cross products cancel where p is nearly parallel to g, so only the
                        # fused arm is held to the bound; the difference between the arms is reported
                        within = err["fused"]["cost"] <= 1e-5 and err["fused"]["joint_grad"] <= 1e-5
                        del outs, fc, fg, bc, bg
                        del rc, rg, ac, ag
                        torch.cuda.empty_cache()
                        rounds, ms = c4bench.alternate(arms, args, empty_cache=True)
                        pairs = A * n
                        line = {"links": kind, "cloud": "scene" if cloud is c4bench.scene_points else "uniform",
                                "n_cfg": A, "points": list(seg_shape), "margin": m,
                                "fused_ms": ms["fused"], "fused_pairs_per_s": pairs / (ms["fused"] * 1e-3),
                                "baseline_ms": ms["per_pair_then_torch"],
                                "baseline_pairs_per_s": pairs / (ms["per_pair_then_torch"] * 1e-3),
                                "speedup": ms["per_pair_then_torch"] / ms["fused"],
                                "max_rel_err_vs_fp64": err, "max_rel_diff_fused_vs_baseline": agree,
                                "fused_within_1e-5": within, "rounds_ms": rounds,
                                "steps": args.steps, "warmup": args.warmup, "gpu": gpu}
                        print(json.dumps(line), flush=True)
                        assert within, line
                    del pts
                    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
