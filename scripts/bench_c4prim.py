"""C4 with analytic primitive links: RobotSDF(..., primitive_visuals=True) of workloads.write_primitive_arm (the 7-DOF
arm with every link a URDF box / cylinder / sphere) x 200 joint configurations x 100 000 points, value + gradient, on
the fused kernels -- against today's workaround for such robots: the same geometry tessellated to OBJ meshes and
cached through cache_link_sdf_factory(0.02, 1.0), also on the fused kernels.  The two arms are timed in alternating
rounds.

    python scripts/bench_c4prim.py [--steps K] [--warmup W] [--rounds R] [--n-cfg 200] [--n-pts 100000]

One GPU.  Device time per step from CUDA events around K steps of the public call (3 rotating point buffers, as
bench.py's C4).  Both arms are also compared with an fp64 composition of the exact primitives (every link restated
in fp64 under the fp32 link transforms) over all configurations and the first 10 000 points: the primitive arm must
be within 1e-5; the tessellated arm's error is reported.  Prints one JSON line with ms per step, pairs per second,
the per-round times, the errors and the card's name and power limit.  Meshes and table caches go to a temporary
directory that is removed at exit.  The reference project has no primitive links, so there is no reference arm."""
import json
import os

import numpy as np
import torch

import c4bench  # first: puts the repository root on sys.path
import pytorch_volumetric_b200 as pv
import workloads


def tessellate(geom):
    """(vertices, faces) of a URDF primitive element string of workloads.PRIMITIVE_ARM_LINKS: box 12 triangles,
    cylinder a 64-sided prism, sphere a 64 x 32 UV sphere (vertices on the surface)."""
    import xml.etree.ElementTree as ET
    e = ET.fromstring(geom)
    if e.tag == "box":
        h = np.array([float(s) for s in e.get("size").split()]) / 2
        v = np.array([[x, y, z] for x in (-h[0], h[0]) for y in (-h[1], h[1]) for z in (-h[2], h[2])])
        f = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
             [0, 6, 4], [1, 5, 7], [1, 7, 3]]
        return v, np.array(f)
    if e.tag == "cylinder":
        r, h, n = float(e.get("radius")), float(e.get("length")) / 2, 64
        a = 2 * np.pi * np.arange(n) / n
        ring = np.stack([r * np.cos(a), r * np.sin(a)], 1)
        v = np.concatenate([np.c_[ring, np.full(n, -h)], np.c_[ring, np.full(n, h)], [[0, 0, -h], [0, 0, h]]])
        f = []
        for i in range(n):
            j = (i + 1) % n
            f += [[i, j, n + j], [i, n + j, n + i], [2 * n, j, i], [2 * n + 1, n + i, n + j]]
        return v, np.array(f)
    r, nl, nt = float(e.get("radius")), 64, 32
    v = [[0, 0, r]]
    for i in range(1, nt):
        ph = np.pi * i / nt
        for j in range(nl):
            th = 2 * np.pi * j / nl
            v.append([r * np.sin(ph) * np.cos(th), r * np.sin(ph) * np.sin(th), r * np.cos(ph)])
    v.append([0, 0, -r])
    vid = lambda i, j: 1 + (i - 1) * nl + j % nl                          # noqa: E731
    f = [[0, vid(1, j), vid(1, j + 1)] for j in range(nl)]
    for i in range(1, nt - 1):
        for j in range(nl):
            f += [[vid(i, j), vid(i + 1, j), vid(i + 1, j + 1)], [vid(i, j), vid(i + 1, j + 1), vid(i, j + 1)]]
    f += [[len(v) - 1, vid(nt - 1, j + 1), vid(nt - 1, j)] for j in range(nl)]
    return np.array(v), np.array(f)


def write_tessellated_arm(dirname):
    """The URDF of write_primitive_arm with every primitive replaced by its tessellation (same <origin>)."""
    from pytorch_volumetric_b200.meshio import write_obj
    os.makedirs(dirname, exist_ok=True)
    parts = ['<robot name="arm7_tessellated">']
    for i, (geom, xyz, rpy) in enumerate(workloads.PRIMITIVE_ARM_LINKS):
        v, f = tessellate(geom)
        write_obj(os.path.join(dirname, f"link{i}.obj"), v, f)
        parts.append(f'<link name="link_{i}"><visual><origin xyz="{xyz}" rpy="{rpy}"/><geometry>'
                     f'<mesh filename="link{i}.obj"/></geometry></visual></link>')
    for i, (xyz, axis) in enumerate(workloads.ARM_JOINTS):
        parts.append(f'<joint name="joint_{i + 1}" type="revolute"><parent link="link_{i}"/>'
                     f'<child link="link_{i + 1}"/><origin xyz="{xyz[0]} {xyz[1]} {xyz[2]}" rpy="0 0 0"/>'
                     f'<axis xyz="{axis[0]} {axis[1]} {axis[2]}"/></joint>')
    parts.append("</robot>")
    path = os.path.join(dirname, "arm.urdf")
    with open(path, "w") as fh:
        fh.write("\n".join(parts))
    return path, "link_7"


def fp64_composition(prim_robot, pts):
    """min over links of the exact primitives in fp64, under prim_robot's fp32 link transforms: [A, P]."""
    from pytorch_volumetric_b200.transforms import matrix_of
    S = len(prim_robot.sdf.sdfs)
    M = matrix_of(prim_robot.sdf.obj_frame_to_link_frame).detach().double().reshape(S, -1, 4, 4)
    best = None
    for s, link in enumerate(prim_robot.sdf.sdfs):
        q = torch.einsum("ajk,pk->apj", M[s, :, :3, :3], pts.double()) + M[s, :, None, :3, 3]
        d = link.native_desc(pts.device)
        if isinstance(link, pv.BoxSDF):
            e = q.abs() - torch.tensor([float(x) for x in d.bb_max], dtype=torch.float64, device=pts.device)
            n = e.clamp(min=0).norm(dim=-1)
            val = torch.where(n > 0, n, e.max(-1).values)
        elif isinstance(link, pv.CylinderSDF):
            dr = torch.hypot(q[..., 0], q[..., 1]) - float(d.radius)
            dz = q[..., 2].abs() - float(d.bb_max[2])
            n = torch.hypot(dr.clamp(min=0), dz.clamp(min=0))
            val = torch.where(n > 0, n, torch.maximum(dr, dz))
        else:
            val = q.norm(dim=-1) - float(np.float32(link.radius))
        best = val if best is None else torch.minimum(best, val)
    return best


def main():
    with c4bench.session(50, 5, 3, n_cfg=200, n_pts=100_000) as (args, tmp):
        th = workloads.arm_configurations(args.n_cfg).cuda()
        prim = c4bench.make_robot("primitive", tmp)
        urdf, end = write_tessellated_arm(os.path.join(tmp, "tess"))
        tess = pv.RobotSDF(pv.build_serial_chain_from_urdf(open(urdf).read(), end).to(device="cuda"),
                           path_prefix=os.path.join(tmp, "tess"),
                           link_sdf_cls=pv.cache_link_sdf_factory(0.02, 1.0, device="cuda",
                                                                  cache_path=os.path.join(tmp, "tess", "cache.pkl")))
        for r in (prim, tess):
            r.set_joint_configuration(th)
        bufs = [c4bench.uniform(args.n_pts, seed=100 + i).cuda() for i in range(3)]

        # accuracy against the fp64 composition of the exact primitives
        sub = bufs[0][:10_000]
        ref = fp64_composition(prim, sub)
        err = {}
        for name, robot in (("primitive", prim), ("tessellated", tess)):
            v, _ = robot(sub)
            e = (v.double() - ref).abs()
            err[name] = {"max_abs": float(e.max()), "mean_abs": float(e.mean()),
                         "frac_over_1e-3": float((e > 1e-3).float().mean())}
        assert err["primitive"]["max_abs"] < 1e-5, err

        pairs = args.n_cfg * args.n_pts
        rounds, ms = c4bench.alternate({"primitive": lambda i: prim(bufs[i % 3]),
                                        "tessellated": lambda i: tess(bufs[i % 3])}, args)
        line = {"metric": "c4prim_pairs_per_s", "value": pairs / (ms["primitive"] * 1e-3), "unit": "pairs/s",
                "ms_per_step": ms["primitive"], "tessellated_ms_per_step": ms["tessellated"],
                "tessellated_pairs_per_s": pairs / (ms["tessellated"] * 1e-3),
                "speedup_vs_tessellated": ms["tessellated"] / ms["primitive"], "rounds_ms": rounds,
                "error_vs_fp64": err, "n_cfg": args.n_cfg, "n_pts": args.n_pts, "steps": args.steps,
                "warmup": args.warmup, "gpu": c4bench.card()}
        print(json.dumps(line))


if __name__ == "__main__":
    main()
