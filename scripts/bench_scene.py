"""Scene queries: every configuration's link points against one static scene SDF (RobotSDF.scene_collision_cost /
scene_clearance, pvb_composed_query_scene_*).

  robots   the cached nearest arm and the primitive arm (workloads.write_arm / write_primitive_arm, 8 links) and the
           hand (workloads.write_hand, 18 links), K link_surface_points per link
  scenes   "boxes": the tabletop c4bench.scene_points samples (the table and its six boxes) as a ComposedSDF of BoxSDF;
           for the hand a small object scene (three boxes and a sphere about the fingers); "cached nearest" /
           "cached trilinear": a CachedSDF of that scene at 0.01 m
  shapes   A x K = 200 x 1024, 4096 x 256 and 65 536 x 64; margins 0.02 and 0.1
  arms     fused scene_collision_cost and scene_clearance; the composition route of both, called directly
           (`_composed_scene_collision_cost` / `_composed_scene_clearance`, "not measured" where one cost call,
           predicted from the previous shape or timed once, exceeds --cap-ms); for context only,
           robot.collision_cost(c4bench.scene_points(10^5, 200), m) -- the point-cloud formulation of the tabletop, a
           different quantity (how far the cloud is from the robot), under the same cap.
Where the fused and composition routes both ran, their outputs are compared: clearance bit for bit, cost within
1e-5 of each row's cost (its sum of terms).  Times are CUDA-event medians over alternating rounds
(c4bench.alternate); the card's name and power limit are read in the same run.  Prints a markdown table and one
JSON line."""
import json
import math
import os
import time

import numpy as np
import torch

import c4bench
import workloads


def _place(t):
    m = torch.eye(4)
    m[:3, 3] = -torch.tensor(t, dtype=torch.float32)
    return m


def _boxes(boxes, spheres=()):
    import pytorch_volumetric_b200 as pv
    sdfs = [pv.BoxSDF(b[3:]) for b in boxes] + [pv.SphereSDF(r) for _, r in spheres]
    mats = [_place([lo + s / 2 for lo, s in zip(b[:3], b[3:])]) for b in boxes] + [_place(c) for c, _ in spheres]
    return pv.ComposedSDF(sdfs, pv.Transform3d(matrix=torch.stack(mats).cuda()))


TABLE = list(workloads.TABLETOP_BOXES)
HAND_OBJECTS = [(-0.05, -0.12, 0.2, 0.1, 0.04, 0.1), (0.06, -0.03, 0.22, 0.04, 0.08, 0.12),
                (-0.08, 0.05, 0.3, 0.16, 0.05, 0.03)]


def _scenes(kind, tmp):
    import pytorch_volumetric_b200 as pv
    if kind == "hand":
        base, rng = _boxes(HAND_OBJECTS, [((0.0, 0.06, 0.2), 0.03)]), [[-0.2, 0.2], [-0.2, 0.2], [0.0, 0.4]]
    else:
        base, rng = _boxes(TABLE), [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]]
    out = {"boxes": base}
    for interp in ("nearest", "trilinear"):
        out[f"cached {interp}"] = pv.CachedSDF(f"{kind}_scene", 0.01, rng, base, device="cuda", clean_cache=True,
                                               cache_path=os.path.join(tmp, f"{kind}_{interp}.pkl"),
                                               interpolation=interp)
    return out


def _robot(kind, tmp):
    import pytorch_volumetric_b200 as pv
    if kind == "hand":
        urdf = workloads.write_hand(os.path.join(tmp, "hand"))
        robot = pv.RobotSDF(pv.build_chain_from_urdf(open(urdf).read()).to(device="cuda"), primitive_visuals=True)
        return robot, lambda A: workloads.tree_configurations(urdf, A, seed=A).cuda()
    return c4bench.make_robot(kind, tmp), lambda A: workloads.arm_configurations(A, seed=A).cuda()


def _once_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    with c4bench.session(steps=3, warmup=1, rounds=3, cap_ms=1000.0) as (args, tmp):
        out = {"card": c4bench.card(), "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
                         "cells": {}}
        cloud = c4bench.scene_points(10 ** 5, 200).cuda()
        agree_all = True
        comp_ms = {}                # (robot, scene, m) -> (ms of one composition-route call, points) at the last shape
        card = out["card"]
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        print("| robot | scene | A x K | m | fused cost ms | fused clearance ms | composition cost ms | "
              "composition clearance ms | point-cloud collision_cost ms (context: a different quantity) | "
              "routes agree |")
        print("|---|---|---|---|---|---|---|---|---|---|", flush=True)
        for kind in ("nearest", "primitive", "hand"):
            robot, configs = _robot(kind, tmp)
            scenes = _scenes(kind, tmp)
            for A, K in ((200, 1024), (4096, 256), (65536, 64)):
                robot.set_joint_configuration(configs(A))
                lp = robot.link_surface_points(num_points=K, seed=1)
                p = lp.float().reshape(-1, 3).contiguous()
                S = len(robot.sdf.sdfs)
                for sname, scene in scenes.items():
                    for m in (0.02, 0.1):
                        key = f"{kind}/{sname}/A{A}xK{K}/m{m}"
                        arms = {"fused cost": lambda i: robot.scene_collision_cost(scene, m, lp),
                                "fused clearance": lambda i: robot.scene_clearance(scene, lp)}
                        comp = lambda: robot.sdf._composed_scene_collision_cost(  # noqa: E731
                            scene, p, K, [True] * S, float(np.float32(m)), 0, A)
                        comp_cl = lambda: robot.sdf._composed_scene_clearance(  # noqa: E731
                            scene, p, K, [True] * S, 0, A, True)
                        context = lambda: robot.collision_cost(cloud, m)     # noqa: E731
                        # the composition route only where one call, predicted from the last shape, stays under the cap
                        last = comp_ms.get((kind, sname, m))
                        ms_comp, ref = math.inf, None
                        if last is None or last[0] * (A * K) / last[1] <= args.cap_ms:
                            ms_comp, ref = _once_ms(comp)
                            comp_ms[(kind, sname, m)] = (ms_comp, A * K)
                        if ms_comp <= args.cap_ms:
                            arms["composition cost"] = lambda i: comp()
                            arms["composition clearance"] = lambda i: comp_cl()
                        if sname == "boxes" and (kind != "hand" or A == 200):     # one cloud per shape
                            ms_ctx, _ = _once_ms(context)
                            if ms_ctx <= args.cap_ms:
                                arms["point-cloud collision_cost (context)"] = lambda i: context()
                        _, med = c4bench.alternate(arms, args)
                        cell = {k: med.get(k) for k in ("fused cost", "fused clearance", "composition cost",
                                                        "composition clearance",
                                                        "point-cloud collision_cost (context)")}
                        if ms_comp <= args.cap_ms:
                            cost, twist = robot.sdf.query_scene_collision_cost(scene, lp, m)
                            cl = robot.sdf.query_scene_clearance(scene, lp, return_which=True)
                            cl_ref = comp_cl()
                            # every cost term h^2 is >= 0, so a row's cost is its sum|term|: the tests' bound
                            diff = (cost.double() - ref[0].double()).abs()
                            rel = float((diff / ref[0].double().clamp_min(1e-30)).max())
                            agree = all(torch.equal(a, b) for a, b in zip(cl, cl_ref)) and rel <= 1e-5
                            cell["agree"], cell["cost_rel_diff"] = agree, rel
                            agree_all &= agree
                        out["cells"][key] = cell
                        fmt = lambda v: "not measured" if v is None else f"{v:.3f}"   # noqa: E731
                        row = (kind, sname, f"{A} x {K}", m, *[fmt(cell[k]) for k in
                               ("fused cost", "fused clearance", "composition cost", "composition clearance",
                                "point-cloud collision_cost (context)")], cell.get("agree", "-"))
                        print("| " + " | ".join(str(x) for x in row) + " |", flush=True)
        out["fused_and_composition_agree"] = agree_all
        print(json.dumps(out))


if __name__ == "__main__":
    main()
