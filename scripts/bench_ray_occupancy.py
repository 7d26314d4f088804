"""Ray-cast point clouds: pvb_ray_carve alone, OccupancyMap.integrate_points and ray_occupancy end to end, and the
depth frames fed as rays beside OccupancyMap.integrate of the same frames, with both routes' accuracy over a stream.

  scans    workloads.tabletop_lidar: 64 x 1024 and 128 x 2048 rays per scan from 1 and 4 sensor positions (inside
           and outside the tabletop range, in turn) in the tabletop room
  frames   workloads.tabletop_views: 1, 4 and 16 cameras at 640 x 480, back-projected (depth_to_points, NaN for
           invalid pixels) and fed as rays with the camera centres as origins
  grids    the tabletop range at 0.02 m (91 x 61 x 68) and 0.01 m (181 x 121 x 136), and 256^3 at 1.8 / 255 m
  arms     "carve": pvb_ray_carve alone, its buffers prepared once and the marks zeroed before every launch (outside
           the timed window), as integrate_points leaves them;
           "integrate_points": OccupancyMap.integrate_points end to end, points and origins on the device;
           "ray_occupancy": ray_occupancy end to end (a fresh grid each call);
           "integrate": OccupancyMap.integrate of the same depth frames (frames only)
  visits   the number of voxels the fp64 reference traversal of tests/ray_ref.py gives each ray (path_lengths),
           summed; rays/s and visits/s are over the carve's median time
  stream   256 ring frames (one view each) integrated one call at a time by both routes on the 0.02 m and 0.01 m
           grids; after 1, 16 and 256 frames, bench_occupancy_map.py's accuracy columns for each map's sdf() against
           the exact 7-box scene, and the share of voxels on which the two maps' free sets disagree
The carve's times are CUDA-event medians per launch; the end-to-end arms' are CUDA-event medians over alternating
rounds (c4bench.alternate).  The card's name and power limit are read in the same run.  Prints markdown tables and one
JSON line."""
import ctypes
import json
import math
import os
import statistics
import sys

import numpy as np
import torch

import c4bench
import workloads
from bench_depth_occupancy import TABLE_RANGE, _exact_scene, _inside_points
from bench_occupancy_map import TARGET, _accuracy

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import ray_ref  # noqa: E402  (the fp64 reference's path lengths count the visits)

GRIDS = [("tabletop 0.02 m", 0.02, TABLE_RANGE), ("tabletop 0.01 m", 0.01, TABLE_RANGE),
         ("256^3", 1.8 / 255, [[-1.1, 0.7], [-0.6, 1.2], [-0.35, 1.45]])]


def _depth_rays(depth, K, poses):
    import pytorch_volumetric_b200 as pv
    pts, _ = pv.depth_to_points(depth, K, poses)
    return pts.reshape(len(poses), -1, 3), torch.from_numpy(np.ascontiguousarray(poses[:, :3, 3], np.float32)).cuda()


def _carve_ms(P, O, r, rng, steps, warmup, rounds):
    """(median ms per launch of pvb_ray_carve, visits): the marks zeroed before every launch, outside the events."""
    from pytorch_volumetric_b200 import _native as nat
    lo, dims = ray_ref.lattice(r, rng)
    p, o = P.reshape(-1, 3).contiguous(), O.reshape(-1, 3).contiguous()
    per = p.shape[0] // o.shape[0]
    margin = math.sqrt(3.0) * r / 2
    marks = torch.zeros(dims, dtype=torch.uint8, device="cuda")
    out = torch.empty_like(p)
    lo32, d = (ctypes.c_float * 3)(*lo), (ctypes.c_int32 * 3)(*dims)
    L, stream = nat.lib(), nat.stream_ptr(p.device)

    def launch():
        nat.check(L.pvb_ray_carve(nat.ptr(p), p.shape[0], per, nat.ptr(o), math.inf, margin, lo32, r, d,
                                  nat.ptr(marks), nat.ptr(out), stream), "pvb_ray_carve")
    times = []
    for _ in range(rounds):
        for _ in range(warmup):
            marks.zero_()
            launch()
        ev = []
        for _ in range(steps):
            marks.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            launch()
            b.record()
            ev.append((a, b))
        torch.cuda.synchronize()
        times += [a.elapsed_time(b) for a, b in ev]
    visits = int(ray_ref.path_lengths(p.cpu().numpy(), o.cpu().numpy(), per, math.inf, margin, lo, r, dims).sum())
    return statistics.median(times), visits


def main():
    import pytorch_volumetric_b200 as pv
    with c4bench.session(steps=20, warmup=3, rounds=3) as (args, tmp):
        card = c4bench.card()
        out = {"card": card, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "times": {},
               "stream": {}}
        print(f"{card['name']}, power limit {card.get('power_limit')}")
        inputs = []
        for beams, columns in ((64, 1024), (128, 2048)):
            for n in (1, 4):
                P, O = workloads.tabletop_lidar(n, beams, columns)
                inputs.append((f"lidar {beams}x{columns} x{n}", torch.from_numpy(P).cuda(),
                               torch.from_numpy(O).cuda(), None))
        for V in (1, 4, 16):
            depth_np, K, poses = workloads.tabletop_views(V)
            depth = torch.from_numpy(depth_np).cuda()
            P, O = _depth_rays(depth, K, poses)
            inputs.append((f"depth {V} views", P, O, (depth, K, poses)))
        print("| input | rays | grid | visits | carve ms | rays/s | visits/s | integrate_points ms | ray_occupancy ms "
              "| integrate ms |")
        print("|---|---|---|---|---|---|---|---|---|---|", flush=True)
        for name, P, O, frames in inputs:
            for gname, r, rng in GRIDS:
                ms, visits = _carve_ms(P, O, r, rng, args.steps, args.warmup, args.rounds)
                m = pv.OccupancyMap(r, rng, device="cuda")
                m.integrate_points(P, O)
                arms = {"integrate_points": lambda i: m.integrate_points(P, O),
                        "ray_occupancy": lambda i: pv.ray_occupancy(P, O, r, rng)}
                if frames is not None:
                    md = pv.OccupancyMap(r, rng, device="cuda")
                    md.integrate(*frames)
                    arms["integrate"] = lambda i: md.integrate(*frames)
                _, med = c4bench.alternate(arms, args)
                n_rays = int(P.numel() // 3)
                row = dict(med, rays=n_rays, visits=visits, carve=ms, rays_per_s=n_rays / ms * 1e3,
                           visits_per_s=visits / ms * 1e3)
                out["times"][f"{name} {gname}"] = row
                dep = f"{med['integrate']:.3f}" if "integrate" in med else "—"
                print(f"| {name} | {n_rays} | {gname} | {visits} | {ms:.4f} | {row['rays_per_s']:.3g} | "
                      f"{row['visits_per_s']:.3g} | {med['integrate_points']:.3f} | {med['ray_occupancy']:.3f} | "
                      f"{dep} |", flush=True)
                del arms, m
                torch.cuda.empty_cache()

        exact = _exact_scene()
        inside = _inside_points(100000, 1).cuda()
        robot = c4bench.make_robot("nearest", tmp)
        robot.set_joint_configuration(workloads.arm_configurations(200, seed=200).cuda())
        lp = robot.link_surface_points(num_points=1024, seed=1)
        K, poses = workloads.camera_ring(256, TARGET, 2.2, 1.3, 800.0, seed=11)
        ring = workloads.render_depth(workloads.TABLETOP_BOXES, K, poses)
        print("\n| grid | frames | route | sign inside | free-space esdf - exact: max | p99 | scene_clearance vs "
              "exact: max | median | free sets disagree |")
        print("|---|---|---|---|---|---|---|---|---|", flush=True)
        for gname, r, rng in GRIDS[:2]:
            a, b = pv.OccupancyMap(r, rng, device="cuda"), pv.OccupancyMap(r, rng, device="cuda")
            for k in range(256):
                d = torch.from_numpy(ring[k:k + 1]).cuda()
                a.integrate(d, K, poses[k:k + 1])
                b.integrate_points(*_depth_rays(d, K, poses[k:k + 1]))
                if k + 1 in (1, 16, 256):
                    sa, sb = a.state(), b.state()
                    disagree = float(((sa == 0) != (sb == 0)).float().mean())
                    for route, mp, st in (("integrate", a, sa), ("integrate_points", b, sb)):
                        acc = _accuracy(mp.sdf(device="cuda"), st, r, rng, exact, robot, lp, inside)
                        acc["free_disagree"] = disagree
                        out["stream"][f"{gname} {k + 1} {route}"] = acc
                        print(f"| {gname} | {k + 1} | {route} | {acc['sign_inside']:.4f} | {acc['free_err_max']:.4f} "
                              f"| {acc['free_err_p99']:.4f} | {acc['clearance_err_max']:.4f} | "
                              f"{acc['clearance_err_median']:.4f} | {disagree:.4%} |", flush=True)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
