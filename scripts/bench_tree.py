"""RobotSDF on kinematic trees (build_chain_from_urdf): forward kinematics and two query forms.

  fk        set_joint_configuration on the hand (workloads.write_hand: 23 frames, 18 primitive links, 21 joints) at
            A = 200, 4096 and 65 536 configurations: the native tree kernel (pvb_fk_tree) against the eager
            forward_kinematics of the same Chain.
  queries   robot(points) and collision_cost at a C4-like shape (A configurations, N points shared by all of them) on
            the gripper tree (workloads.write_gripper_tree: 8 links, the fused kernels) and on the hand (18 links, the
            composition routes).
Times are CUDA-event medians over alternating rounds (c4bench.alternate); the card's name and power limit are read in
the same run.  Prints a markdown table and one JSON line."""
import json
import os

import torch

import c4bench
import workloads


def _robot(kind, tmp):
    import pytorch_volumetric_b200 as pv
    urdf = workloads.write_hand(os.path.join(tmp, kind)) if kind == "hand" else \
        workloads.write_gripper_tree(os.path.join(tmp, kind))
    robot = pv.RobotSDF(pv.build_chain_from_urdf(open(urdf).read()).to(device="cuda"), primitive_visuals=True)
    return robot, urdf


def main():
    with c4bench.session(steps=20, warmup=3, rounds=5, n_cfg=200, n_pts=20000, margin=0.02) as (args, tmp):
        rows, out = [], {"card": c4bench.card(), "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds}
        hand, hand_urdf = _robot("hand", tmp)
        assert hand._fk_plan is not None
        for A in (200, 4096, 65536):
            q = workloads.tree_configurations(hand_urdf, A, seed=A).cuda()

            def fk(native):
                def step(i):
                    hand.native_fk = native
                    hand.set_joint_configuration(q)
                    return hand.object_to_link_frames
                return step
            _, med = c4bench.alternate({"native": fk(True), "eager": fk(False)}, args)
            hand.native_fk = True
            out[f"fk_hand_A{A}"] = med
            rows.append((f"hand set_joint_configuration, A = {A}", "pvb_fk_tree", med["native"],
                         f"eager {med['eager']:.3f} ms ({med['eager'] / med['native']:.1f}x)"))
        for kind, route in (("gripper", "fused (8 links)"), ("hand", "composition (18 links)")):
            robot, urdf = (hand, hand_urdf) if kind == "hand" else _robot(kind, tmp)
            robot.set_joint_configuration(workloads.tree_configurations(urdf, args.n_cfg, seed=1).cuda())
            lo, hi = ([-0.5, -0.5, -0.1], [0.5, 0.5, 0.6]) if kind == "gripper" else ([-0.2, -0.2, -0.1], [0.2, 0.2, 0.3])
            pts = workloads.uniform_points(args.n_pts, lo, hi, seed=7, device="cuda")
            _, med = c4bench.alternate({"call": lambda i: robot(pts),
                                        "collision_cost": lambda i: robot.collision_cost(pts, args.margin)}, args)
            out[f"{kind}_A{args.n_cfg}_N{args.n_pts}"] = med
            rows.append((f"{kind} robot(points), A = {args.n_cfg}, N = {args.n_pts}", route, med["call"], ""))
            rows.append((f"{kind} collision_cost, A = {args.n_cfg}, N = {args.n_pts}", route, med["collision_cost"],
                         ""))
        card = out["card"]
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        print("| workload | route | ms | |\n|---|---|---|---|")
        for name, route, ms, note in rows:
            print(f"| {name} | {route} | {ms:.3f} | {note} |")
        print(json.dumps(out))


if __name__ == "__main__":
    main()
