"""Occupancy maps: OccupancyMap.integrate (pvb_depth_integrate) per frame, its map as a scene over a stream of frames,
and how fast a moved object clears.

  frames   workloads.tabletop_views: the 7 tabletop boxes rendered in fp64 by 1, 4 and 16 cameras of a ring at
           640 x 480 (f = 800 px, about 2.5 m from the scene), as in bench_depth_occupancy.py
  grids    the tabletop range at 0.02 m (91 x 61 x 68) and 0.01 m (181 x 121 x 136), and 256^3 at 1.8 / 255 m
  arms     "integrate": OccupancyMap.integrate end to end, depth already on the device (argument checks, points,
           scatter, fused update; no synchronisation);
           "fused": the same device work with every argument prepared once (pvb_depth_points, pvb_voxel_scatter,
           pvb_depth_integrate);
           "kernel": pvb_depth_integrate alone, on the hit grid it leaves all zero, so every voxel runs its view loop
           (an upper bound of the kernel's share of "fused");
           "composition": the unfused route, prepared once (pvb_depth_points, pvb_voxel_scatter, pvb_depth_carve and
           the update in torch, then the hit grid cleared);
           "sdf": OccupancyMap.sdf() (threshold, then the EDT and table of OccupancySDF)
           Both routes' log-odds are asserted equal after three calls on fresh maps.
  stream   256 ring frames (one view each, 640 x 480) integrated one call at a time on the 0.02 m and 0.01 m tabletop
           grids; after 1, 4, 16, 64 and 256 frames, bench_depth_occupancy.py's accuracy columns for map.sdf() against
           the exact 7-box scene (reported, not asserted)
  clearing a box added to the tabletop for 6 frames of a 4-camera rig, then removed: the frames after which every
           voxel it saturated and the rig now carves is free, and how many it saturated that the rig never carves
Times are CUDA-event medians over alternating rounds (c4bench.alternate); the card's name and power limit are read in
the same run.  Prints markdown tables and one JSON line."""
import ctypes
import json
import math

import numpy as np
import torch

import c4bench
import workloads
from bench_depth_occupancy import TABLE_RANGE, _exact_scene, _inside_points

TARGET = (-0.25, 0.0, 0.2)
MOVED_BOX = (-0.1, -0.1, -0.2, 0.2, 0.2, 0.3)


def _prepared(m, depth, K, poses):
    """(fused step, kernel step, composition step, composition's log-odds) over m's lattice and parameters."""
    from pytorch_volumetric_b200 import _native as nat
    from pytorch_volumetric_b200 import sdf as S
    views = S._depth_views(depth, K, poses, math.inf)
    V, H, W = depth.shape
    intr = (ctypes.c_float * (4 * V))(*views.intrinsics.reshape(-1).tolist())
    c2w = (ctypes.c_float * (12 * V))(*views.cam_to_world[:, :3].float().reshape(-1).tolist())
    w2c = (ctypes.c_float * (12 * V))(*S.invert_rigid(views.cam_to_world)[:, :3].float().reshape(-1).tolist())
    L, stream = nat.lib(), nat.stream_ptr(depth.device)
    points = torch.empty(V * H * W, 3, dtype=torch.float32, device="cuda")
    hits = m._hits.get_voxel_values()
    state = torch.empty(m.shape, dtype=torch.uint8, device="cuda")
    comp = torch.full(m.shape, S.LOG_ODDS_UNOBSERVED, dtype=torch.int16, device="cuda")
    hit, miss, lo_c, hi_c, _ = m.params

    def back_project():
        nat.check(L.pvb_depth_points(nat.ptr(depth), V, H, W, intr, c2w, math.inf, nat.ptr(points), stream), "points")
        m._hits[points] = True

    def kernel(i=0):
        nat.check(L.pvb_depth_integrate(nat.ptr(depth), V, H, W, intr, w2c, math.inf, m.free_margin, m._lo,
                                        m.resolution, m._dims, nat.ptr(hits), nat.ptr(m._log_odds), m._update,
                                        stream), "pvb_depth_integrate")

    def fused(i=0):
        back_project()
        kernel()

    def composition(i=0):
        back_project()
        nat.check(L.pvb_depth_carve(nat.ptr(depth), V, H, W, intr, w2c, math.inf, m.free_margin, m._lo, m.resolution,
                                    m._dims, nat.ptr(state), stream), "pvb_depth_carve")
        base = torch.where(comp == S.LOG_ODDS_UNOBSERVED, 0, comp.int())
        new = torch.where(hits, (base + hit).clamp_max(hi_c),
                          torch.where(state == 0, (base + miss).clamp_min(lo_c), comp.int()))
        comp.copy_(new)
        hits.zero_()
    return fused, kernel, composition, comp


def _check_routes(r, rng, depth, K, poses):
    import pytorch_volumetric_b200 as pv
    a, b = pv.OccupancyMap(r, rng, device="cuda"), pv.OccupancyMap(r, rng, device="cuda")
    fused, _, _, _ = _prepared(a, depth, K, poses)
    _, _, composition, comp = _prepared(b, depth, K, poses)
    for _ in range(3):
        fused()
        composition()
    assert torch.equal(a._log_odds, comp), "the fused and composition routes differ"


def _accuracy(sdf, state, r, rng, exact, robot, lp, inside):
    import pytorch_volumetric_b200 as pv
    out = {"sign_inside": float((sdf(inside)[0] < 0).float().mean())}
    q = workloads.uniform_points(200000, [x[0] for x in rng], [x[1] for x in rng], seed=5).cuda()
    free = pv.VoxelGrid(r, rng, dtype=torch.bool, device="cuda")
    free.get_voxel_values().copy_(state == 0)
    q = q[free[q]]
    err = (sdf(q)[0] - exact(q)[0]).double()
    out["free_points"] = int(q.shape[0])
    out["free_err_max"] = float(err.max()) if len(err) else math.nan
    out["free_err_p99"] = float(torch.quantile(err, 0.99)) if len(err) else math.nan
    diff = (robot.scene_clearance(sdf, lp)[0] - robot.scene_clearance(exact, lp)[0]).abs()
    out["clearance_err_max"], out["clearance_err_median"] = float(diff.max()), float(diff.median())
    return out


def _clearing(r):
    """(frames until every saturated voxel the rig carves is free, saturated voxels the rig never carves)."""
    import pytorch_volumetric_b200 as pv
    K, poses = workloads.camera_ring(4, TARGET, 2.2, 1.3, 800.0, seed=7)
    with_box = torch.from_numpy(workloads.render_depth(workloads.TABLETOP_BOXES + (MOVED_BOX,), K, poses)).cuda()
    without = torch.from_numpy(workloads.render_depth(workloads.TABLETOP_BOXES, K, poses)).cuda()
    m = pv.OccupancyMap(r, TABLE_RANGE, device="cuda")
    for _ in range(6):
        m.integrate(with_box, K, poses)
    saturated = m._log_odds == m.params.clamp_hi
    m0 = pv.OccupancyMap(r, TABLE_RANGE, device="cuda")
    m0.integrate(without, K, poses)
    carved = saturated & (m0.state() == 0)
    for k in range(1, 64):
        m.integrate(without, K, poses)
        if not bool((m.state()[carved] == 1).any()):
            return k, int(carved.sum()), int((saturated & ~carved & (m.state() == 1)).sum())
    return None, int(carved.sum()), None


def main():
    import pytorch_volumetric_b200 as pv
    with c4bench.session(steps=20, warmup=3, rounds=3) as (args, tmp):
        card = c4bench.card()
        out = {"card": card, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "times": {},
               "stream": {}, "clearing": {}}
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        grids = [("tabletop 0.02 m", 0.02, TABLE_RANGE), ("tabletop 0.01 m", 0.01, TABLE_RANGE),
                 ("256^3", 1.8 / 255, [[-1.1, 0.7], [-0.6, 1.2], [-0.35, 1.45]])]
        frames = {V: workloads.tabletop_views(V) for V in (1, 4, 16)}
        print("| views | grid | voxels | integrate ms | fused ms | kernel ms | composition ms | sdf() ms |")
        print("|---|---|---|---|---|---|---|---|", flush=True)
        for V, (depth_np, K, poses) in frames.items():
            depth = torch.from_numpy(depth_np).cuda()
            for name, r, rng in grids:
                _check_routes(r, rng, depth, K, poses)
                m = pv.OccupancyMap(r, rng, device="cuda")
                m.integrate(depth, K, poses)
                fused, kernel, composition, _ = _prepared(pv.OccupancyMap(r, rng, device="cuda"), depth, K, poses)
                arms = {"integrate": lambda i: m.integrate(depth, K, poses), "fused": fused, "kernel": kernel,
                        "composition": composition, "sdf": lambda i: m.sdf(device="cuda")}
                _, med = c4bench.alternate(arms, args)
                n_vox = int(np.prod(m.shape))
                out["times"][f"V{V} {name}"] = dict(med, voxels=n_vox)
                print(f"| {V} | {name} | {n_vox} | {med['integrate']:.3f} | {med['fused']:.3f} | {med['kernel']:.3f} "
                      f"| {med['composition']:.3f} | {med['sdf']:.3f} |", flush=True)
                del arms, fused, kernel, composition, m
                torch.cuda.empty_cache()

        exact = _exact_scene()
        inside = _inside_points(100000, 1).cuda()
        robot = c4bench.make_robot("nearest", tmp)
        robot.set_joint_configuration(workloads.arm_configurations(200, seed=200).cuda())
        lp = robot.link_surface_points(num_points=1024, seed=1)
        K, poses = workloads.camera_ring(256, TARGET, 2.2, 1.3, 800.0, seed=11)
        ring = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses)
        print("\n| grid | frames | sign inside | free-space esdf - exact: max | p99 | scene_clearance vs exact: max "
              "| median |")
        print("|---|---|---|---|---|---|---|", flush=True)
        for name, r, rng in grids[:2]:
            m = pv.OccupancyMap(r, rng, device="cuda")
            for k in range(256):
                m.integrate(torch.from_numpy(ring[k:k + 1]).cuda(), K, poses[k:k + 1])
                if k + 1 in (1, 4, 16, 64, 256):
                    acc = _accuracy(m.sdf(device="cuda"), m.state(), r, rng, exact, robot, lp, inside)
                    out["stream"][f"{name} {k + 1}"] = acc
                    print(f"| {name} | {k + 1} | {acc['sign_inside']:.4f} | {acc['free_err_max']:.4f} | "
                          f"{acc['free_err_p99']:.4f} | {acc['clearance_err_max']:.4f} | "
                          f"{acc['clearance_err_median']:.4f} |", flush=True)

        print("\n| grid | frames until free | voxels carved | saturated voxels never carved, still occupied |")
        print("|---|---|---|---|")
        for name, r, _ in grids[:2]:
            k, n_carved, n_kept = _clearing(r)
            out["clearing"][name] = {"frames": k, "carved": n_carved, "kept": n_kept}
            print(f"| {name} | {k} | {n_carved} | {n_kept} |", flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
