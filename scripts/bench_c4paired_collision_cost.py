"""Paired collision-cost queries: RobotSDF.paired_collision_cost(points, margin) -- every configuration against its
own cloud, the hinge cost sum_p max(0, m - d)^2 of every segment and its joint gradient -- against the composition
route it is defined by, ComposedSDF._composed_collision_cost(..., paired=True) called directly (query_paired on chunks
of configurations, fp64 terms and one masked sum per link) followed by the same joint_gradient, on the 8-link arm.

    python scripts/bench_c4paired_collision_cost.py [--steps K] [--warmup W] [--rounds R]

Shapes (A configurations x points per configuration): 200 x 10^4, 4096 x 2048, 65 536 x 64 and 1024 x (8 segments x
256), with nearest, trilinear and primitive links, the two clouds of c4bench.clouds (uniform per
configuration, and the tabletop scene shifted per configuration), and margins 0.02 and 0.1 m.  Before timing, both
arms are compared with the fp64 sum of the same fp32 per-pair outputs (query_paired(..., return_which=True)), and
asserted to agree with each other within 1e-5 of the sum of |term| of every cost and joint-gradient entry.  Device
time per call from CUDA events around K calls after W warm-up calls, the two arms alternating for R rounds; pairs/s =
A * (points per configuration) / time.  Prints one JSON line per shape with the card's name and power limit.  Meshes
and table caches go to a temporary directory that is removed at exit."""
import json

import torch

import c4bench  # first: puts the repository root on sys.path
import workloads


def composition(robot, own, m):
    """The composition route over own [A, *B, N, 3], then joint_gradient: (cost [A * n_seg], joint_grad)."""
    A, L = own.shape[0], own.shape[-2]
    n_seg = own.numel() // (3 * A * L)
    cost, twist = robot.sdf._composed_collision_cost(own.reshape(-1, 3), m, 0, A, n_seg, L, paired=True)
    return cost, robot.joint_gradient(twist, robot.joint_twists(), robot.joint_moves_link())


def fp64_reference(robot, own, m, cfg_chunk=256):
    """fp64 cost [A * n_seg], joint gradient [A * n_seg, J] and the sums of |term| of both, from the fp32
    query_paired(..., return_which=True) outputs at every configuration's own points."""
    comp = robot.sdf
    S, A, L = len(comp.sdfs), own.shape[0], own.shape[-2]
    p = own.reshape(A, -1, L, 3)
    n_seg = p.shape[1]
    jt, moves = robot.joint_twists(), robot.joint_moves_link()
    out = [[], [], [], []]
    for c0 in range(0, A, cfg_chunk):
        cc = min(cfg_chunk, A - c0)
        v, g, w = comp.query_paired(p[c0:c0 + cc], c0, cc, return_which=True)
        v, g, w = v.reshape(cc, n_seg, L).double(), g.reshape(cc, n_seg, L, 3).double(), w.reshape(cc, n_seg, L)
        h = (m - v).clamp_min(0.0)
        terms = torch.cat([g, torch.linalg.cross(p[c0:c0 + cc].double(), g, dim=-1)], -1) * (2 * h)[..., None]
        twist = torch.empty(cc, n_seg, S, 6, dtype=torch.float64, device=own.device)
        abs_tw = torch.empty_like(twist)
        for s in range(S):
            mask = (w == s)[..., None]
            twist[:, :, s] = (terms * mask).sum(-2)
            abs_tw[:, :, s] = (terms.abs() * mask).sum(-2)
        j = jt[c0:c0 + cc]
        out[0].append((h * h).sum(-1).reshape(-1))
        out[1].append(robot.joint_gradient(twist, j, moves).reshape(cc * n_seg, -1))
        out[2].append(out[0][-1])
        out[3].append(robot.joint_gradient(abs_tw, j.abs(), moves).reshape(cc * n_seg, -1))
    return [torch.cat(o) for o in out]


def main():
    with c4bench.session(10, 2, 3) as (args, tmp):
        gpu = c4bench.card()
        robots = {k: c4bench.make_robot(k, tmp) for k in ("nearest", "trilinear", "primitive")}
        shapes = [("a200_n1e4", 200, (10_000,)), ("a4096_n2048", 4096, (2048,)), ("a65536_n64", 65_536, (64,)),
                  ("a1024_seg8_n256", 1024, (8, 256))]
        for name, A, seg_shape in shapes:
            for cloud in ("uniform", "scene"):
                own = c4bench.clouds(cloud, A, seg_shape, 300).cuda()
                for kind, robot in robots.items():
                    robot.set_joint_configuration(workloads.arm_configurations(A).cuda())
                    for m in (0.02, 0.1):
                        m = torch.tensor(m, dtype=torch.float32).item()     # the fp32 margin every route uses
                        arms = {"fused": lambda i, r=robot, m=m: r.paired_collision_cost(own, m),
                                "composition": lambda i, r=robot, m=m: composition(r, own, m)}
                        rc, rg, ac, ag = fp64_reference(robot, own, m)
                        outs = {k: f(0) for k, f in arms.items()}
                        err = {k: {"cost": c4bench.rel_err(c, rc, ac), "joint_grad": c4bench.rel_err(g, rg, ag)}
                               for k, (c, g) in outs.items()}
                        (fc, fg), (bc, bg) = outs["fused"], outs["composition"]
                        agree = {"cost": c4bench.rel_err(fc, bc.double().reshape(rc.shape), ac),
                                 "joint_grad": c4bench.rel_err(fg, bg.double().reshape(rg.shape), ag)}
                        contributing = int((rc > 0).sum())
                        del outs, fc, fg, bc, bg, rc, rg, ac, ag
                        torch.cuda.empty_cache()
                        rounds, ms = c4bench.alternate(arms, args, empty_cache=True)
                        pairs = A * own[0].numel() // 3
                        line = {"shape": name, "links": kind, "cloud": cloud, "n_cfg": A, "points": list(seg_shape),
                                "margin": m, "fused_ms": ms["fused"], "fused_pairs_per_s": pairs / (ms["fused"] * 1e-3),
                                "composition_ms": ms["composition"],
                                "composition_pairs_per_s": pairs / (ms["composition"] * 1e-3),
                                "speedup": ms["composition"] / ms["fused"], "max_rel_err_vs_fp64": err,
                                "max_rel_diff_fused_vs_composition": agree, "rows_with_cost": contributing,
                                "rounds_ms": rounds, "steps": args.steps, "warmup": args.warmup, "gpu": gpu}
                        print(json.dumps(line), flush=True)
                        assert agree["cost"] <= 1e-5 and agree["joint_grad"] <= 1e-5, line
                del own
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
