"""OccupancySDF: signed distance tables built on the GPU from an occupancy grid or a point cloud (pvb_occupancy_sdf).

  grids    128^3 and 256^3 at 1 % and 30 % random occupancy, 512^3 at 1 %, 1024 x 64 x 64 at 1 %, and the tabletop:
           c4bench.scene_points(10^5, 200) over bench_scene's range [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]] at
           0.01 m (181 x 121 x 136) and at 0.02 m
  arms     "transform": pvb_occupancy_sdf alone (the three passes and the record writer, workspace and outputs
           allocated once), CUDA events; "from_points" (tabletop only): OccupancySDF.from_points end to end, scatter,
           checks, transform and table installation; "scipy": scipy.ndimage.distance_transform_edt of both states on
           the CPU, timed once and skipped ("not measured") where the grid exceeds --scipy-max-voxels
  scene    the cached arm's scene_collision_cost (m = 0.02) and scene_clearance against the 0.02 m tabletop
           OccupancySDF at 200 x 1024 and 65 536 x 64, beside robot.collision_cost(cloud, 0.02), the point-cloud
           formulation (a different quantity: how far the cloud is from the robot)
Times are CUDA-event medians over alternating rounds (c4bench.alternate); the card's name and power limit are read in
the same run.  Prints markdown tables and one JSON line."""
import ctypes
import json
import time

import numpy as np
import torch

import c4bench

TABLE_RANGE = [[-1.1, 0.7], [-0.6, 0.6], [-0.35, 1.0]]


def _random(shape, p, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    occ = torch.rand(shape, generator=g, device="cuda") < p
    occ.view(-1)[0], occ.view(-1)[-1] = True, False
    return occ


def _scipy_ms(occ):
    from scipy.ndimage import distance_transform_edt
    o = occ.cpu().numpy()
    t = time.perf_counter()
    distance_transform_edt(o)
    distance_transform_edt(~o)
    return (time.perf_counter() - t) * 1e3


def _transform_arm(occ):
    """A step running pvb_occupancy_sdf on occ with preallocated workspace and table."""
    from pytorch_volumetric_b200 import _native as nat
    o = occ.to(torch.uint8).contiguous()
    dims = (ctypes.c_int32 * 3)(*o.shape)
    L = nat.lib()
    ws = torch.empty(int(L.pvb_occupancy_sdf_workspace(dims)), dtype=torch.uint8, device="cuda")
    table = torch.empty(o.numel(), 4, dtype=torch.float32, device="cuda")
    stream = nat.stream_ptr(o.device)

    def step(i):
        nat.check(L.pvb_occupancy_sdf(nat.ptr(o), dims, 0.01, nat.ptr(ws), ws.numel(), None, None, nat.ptr(table),
                                      stream), "pvb_occupancy_sdf")
    return step


def main():
    import pytorch_volumetric_b200 as pv
    with c4bench.session(steps=10, warmup=2, rounds=3, scipy_max_voxels=4_000_000) as (args, tmp):
        card = c4bench.card()
        out = {"card": card, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "grids": {},
               "scene": {}}
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        cloud = c4bench.scene_points(10 ** 5, 200).cuda()
        grids = [("128^3, 1 %", lambda: _random((128,) * 3, 0.01, 1)),
                 ("128^3, 30 %", lambda: _random((128,) * 3, 0.3, 2)),
                 ("256^3, 1 %", lambda: _random((256,) * 3, 0.01, 3)),
                 ("256^3, 30 %", lambda: _random((256,) * 3, 0.3, 4)),
                 ("512^3, 1 %", lambda: _random((512,) * 3, 0.01, 5)),
                 ("1024 x 64 x 64, 1 %", lambda: _random((1024, 64, 64), 0.01, 6))]
        for r in (0.01, 0.02):
            grids.append((f"tabletop at {r} m", lambda r=r: pv.OccupancySDF.from_points(cloud, r, TABLE_RANGE,
                                                                                          device="cuda").occupancy))
        print("| grid | voxels | transform ms | from_points ms | scipy CPU ms (both states) |")
        print("|---|---|---|---|---|", flush=True)
        for name, make in grids:
            occ = make()
            arms = {"transform": _transform_arm(occ)}
            if name.startswith("tabletop"):
                r = float(name.split()[2])
                arms["from_points"] = lambda i, r=r: pv.OccupancySDF.from_points(cloud, r, TABLE_RANGE, device="cuda")
            _, med = c4bench.alternate(arms, args)
            scipy_ms = _scipy_ms(occ) if occ.numel() <= args.scipy_max_voxels else None
            cell = {"shape": list(occ.shape), "voxels": occ.numel(), "transform_ms": med["transform"],
                    "from_points_ms": med.get("from_points"), "scipy_ms": scipy_ms}
            out["grids"][name] = cell
            fmt = lambda v: "not measured" if v is None else f"{v:.3f}"      # noqa: E731
            print(f"| {name} | {occ.numel()} | {fmt(cell['transform_ms'])} | {fmt(cell['from_points_ms'])} | "
                  f"{fmt(scipy_ms)} |", flush=True)
            del occ, arms
            torch.cuda.empty_cache()

        robot = c4bench.make_robot("nearest", tmp)
        scene = pv.OccupancySDF.from_points(cloud, 0.02, TABLE_RANGE, device="cuda")
        print("\n| A x K | scene_collision_cost ms | scene_clearance ms | robot.collision_cost(cloud) ms (context) |")
        print("|---|---|---|---|", flush=True)
        import workloads
        for A, K in ((200, 1024), (65536, 64)):
            robot.set_joint_configuration(workloads.arm_configurations(A, seed=A).cuda())
            lp = robot.link_surface_points(num_points=K, seed=1)
            arms = {"scene_collision_cost": lambda i: robot.scene_collision_cost(scene, 0.02, lp),
                    "scene_clearance": lambda i: robot.scene_clearance(scene, lp),
                    "collision_cost(cloud)": lambda i: robot.collision_cost(cloud, 0.02)}
            _, med = c4bench.alternate(arms, args)
            out["scene"][f"A{A}xK{K}"] = med
            print(f"| {A} x {K} | {med['scene_collision_cost']:.3f} | {med['scene_clearance']:.3f} | "
                  f"{med['collision_cost(cloud)']:.3f} |", flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
