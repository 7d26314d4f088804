"""Depth-image scenes: back-projection, free-space carving and OccupancySDF.from_depth on the GPU.

  frames   workloads.tabletop_views: the 7 tabletop boxes rendered in fp64 by 1, 4 and 16 cameras of a ring at
           640 x 480 (f = 800 px, about 2.5 m from the scene)
  grids    the tabletop range [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]] at 0.02 m (91 x 61 x 68) and 0.01 m
           (181 x 121 x 136), and a 256^3 grid from the same corner at 1.8 / 255 m
  arms     "points": depth_to_points; "carve": pvb_depth_carve alone, state buffer and view arrays prepared once;
           "depth_occupancy": the state grid end to end (checks, points, carve, scatter); "from_depth":
           OccupancySDF.from_depth end to end (unknown = occupied), transform and table included
  accuracy (tabletop grids, reported, not asserted) against the exact scene, a ComposedSDF of the 7 BoxSDFs:
           - the share of 100 000 points inside the boxes where the table is negative, for from_depth and for
             from_points of the same frames' valid points;
           - the largest and the 99th-percentile (esdf - exact) over uniform points whose voxel is carved free;
           - the cached arm's scene_clearance at 200 x 1024 against the from_depth scene and the exact scene: the
             largest and the median |difference| over the configurations
Times are CUDA-event medians over alternating rounds (c4bench.alternate); the card's name and power limit are read in
the same run.  Prints markdown tables and one JSON line."""
import ctypes
import json
import math

import numpy as np
import torch

import c4bench
import workloads

TABLE_RANGE = [list(r) for r in workloads.TABLETOP_RANGE]


def _exact_scene():
    import pytorch_volumetric_b200 as pv
    mats = []
    for b in workloads.TABLETOP_BOXES:
        m = torch.eye(4)
        m[:3, 3] = -torch.tensor([lo + s / 2 for lo, s in zip(b[:3], b[3:])])
        mats.append(m)
    return pv.ComposedSDF([pv.BoxSDF(b[3:]) for b in workloads.TABLETOP_BOXES],
                          pv.Transform3d(matrix=torch.stack(mats).cuda()))


def _inside_points(n, seed):
    """[n, 3] uniform inside the boxes, each box taking a share proportional to its volume."""
    g = np.random.default_rng(seed)
    b = np.asarray(workloads.TABLETOP_BOXES)
    k = g.choice(len(b), n, p=b[:, 3:].prod(1) / b[:, 3:].prod(1).sum())
    return torch.from_numpy(b[k, :3] + g.random((n, 3)) * b[k, 3:]).float()


def _carve_arm(depth, K, poses, r, rng):
    """A step running pvb_depth_carve alone, its inputs and output prepared once."""
    from pytorch_volumetric_b200 import _native as nat
    from pytorch_volumetric_b200 import sdf as S
    views = S._depth_views(depth, K, poses, math.inf)
    _, _, margin = S._depth_lattice(r, rng, None)
    grid = S.VoxelGrid(r, rng, dtype=torch.bool, device="cuda")
    state = grid.get_voxel_values().view(torch.uint8)
    V, H, W = depth.shape
    w2c = (ctypes.c_float * (12 * V))(*S.invert_rigid(views.cam_to_world)[:, :3].float().reshape(-1).tolist())
    intr = (ctypes.c_float * (4 * V))(*views.intrinsics.reshape(-1).tolist())
    lo = (ctypes.c_float * 3)(*[float(min(x)) for x in grid.range_per_dim])
    dims = (ctypes.c_int32 * 3)(*state.shape)
    L, stream = nat.lib(), nat.stream_ptr(depth.device)

    def step(i):
        nat.check(L.pvb_depth_carve(nat.ptr(depth), V, H, W, intr, w2c, math.inf, margin, lo, r, dims,
                                    nat.ptr(state), stream), "pvb_depth_carve")
    return step, state.numel()


def _accuracy(depth, K, poses, r, rng, exact, robot, lp, inside):
    import pytorch_volumetric_b200 as pv
    sdf = pv.OccupancySDF.from_depth(depth, K, poses, r, rng, device="cuda")
    pts, valid = pv.depth_to_points(depth, K, poses)
    cloud = pv.OccupancySDF.from_points(pts[valid], r, rng, device="cuda")
    out = {"sign_from_depth": float((sdf(inside)[0] < 0).float().mean()),
           "sign_from_points": float((cloud(inside)[0] < 0).float().mean())}
    q = workloads.uniform_points(200000, [x[0] for x in rng], [x[1] for x in rng], seed=5).cuda()
    state = pv.depth_occupancy(depth, K, poses, r, rng)
    free = pv.VoxelGrid(r, rng, dtype=torch.bool, device="cuda")
    free.get_voxel_values().copy_(state == 0)
    q = q[free[q]]
    err = (sdf(q)[0] - exact(q)[0]).double()
    out["free_points"] = int(q.shape[0])
    out["free_err_max"] = float(err.max())
    out["free_err_p99"] = float(torch.quantile(err, 0.99))
    got = robot.scene_clearance(sdf, lp)[0]
    want = robot.scene_clearance(exact, lp)[0]
    diff = (got - want).abs()
    out["clearance_err_max"], out["clearance_err_median"] = float(diff.max()), float(diff.median())
    return out, sdf


def main():
    import pytorch_volumetric_b200 as pv
    with c4bench.session(steps=10, warmup=2, rounds=3) as (args, tmp):
        card = c4bench.card()
        out = {"card": card, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "times": {},
               "accuracy": {}}
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        grids = [("tabletop 0.02 m", 0.02, TABLE_RANGE), ("tabletop 0.01 m", 0.01, TABLE_RANGE),
                 ("256^3", 1.8 / 255, [[-1.1, 0.7], [-0.6, 1.2], [-0.35, 1.45]])]
        frames = {V: workloads.tabletop_views(V) for V in (1, 4, 16)}
        print("| views | grid | voxels | depth_to_points ms | carve ms | depth_occupancy ms | from_depth ms |")
        print("|---|---|---|---|---|---|---|", flush=True)
        for V, (depth_np, K, poses) in frames.items():
            depth = torch.from_numpy(depth_np).cuda()
            for name, r, rng in grids:
                carve, n_vox = _carve_arm(depth, K, poses, r, rng)
                arms = {"points": lambda i: pv.depth_to_points(depth, K, poses),
                        "carve": carve,
                        "depth_occupancy": lambda i: pv.depth_occupancy(depth, K, poses, r, rng),
                        "from_depth": lambda i: pv.OccupancySDF.from_depth(depth, K, poses, r, rng, device="cuda")}
                _, med = c4bench.alternate(arms, args)
                out["times"][f"V{V} {name}"] = dict(med, voxels=n_vox)
                print(f"| {V} | {name} | {n_vox} | {med['points']:.3f} | {med['carve']:.3f} | "
                      f"{med['depth_occupancy']:.3f} | {med['from_depth']:.3f} |", flush=True)
                del arms, carve
                torch.cuda.empty_cache()

        exact = _exact_scene()
        inside = _inside_points(100000, 1).cuda()
        assert bool((exact(inside)[0] < 0).all())
        robot = c4bench.make_robot("nearest", tmp)
        robot.set_joint_configuration(workloads.arm_configurations(200, seed=200).cuda())
        lp = robot.link_surface_points(num_points=1024, seed=1)
        print("\n| views | grid | sign inside, from_depth | sign inside, from_points | free-space esdf - exact: max | "
              "p99 | scene_clearance vs exact: max | median |")
        print("|---|---|---|---|---|---|---|---|", flush=True)
        for V, (depth_np, K, poses) in frames.items():
            depth = torch.from_numpy(depth_np).cuda()
            for name, r, rng in grids[:2]:
                acc, _ = _accuracy(depth, K, poses, r, rng, exact, robot, lp, inside)
                out["accuracy"][f"V{V} {name}"] = acc
                print(f"| {V} | {name} | {acc['sign_from_depth']:.4f} | {acc['sign_from_points']:.4f} | "
                      f"{acc['free_err_max']:.4f} | {acc['free_err_p99']:.4f} | {acc['clearance_err_max']:.4f} | "
                      f"{acc['clearance_err_median']:.4f} |", flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
