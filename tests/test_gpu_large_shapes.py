"""GPU: the RobotSDF-family queries at the sizes their launch limits exist for -- past 65535 configuration tiles and
past 2^31 (configuration, point) pairs -- against configuration slabs of the same call and against the fp64 robot
(tests/robot_ref.py).

Size limits of the kernels and launchers (pvb_kernels.cu), and the index expression per limit exercised here:
  composed_dispatch (point query)   robot_serial_kernel needs rs_tile_count(cfg_count) <= 65535 grid rows and
                                    rs_int_pts_ok(n_pts); robot_query_kernel and composed_cfgmajor_kernel one row per
                                    32 configurations.  A slab of more tiles runs as balanced slabs of whole tiles,
                                    each on the route the whole would take: robot_serial_kernel launched twice at
                                    65535 x 32 + 1 configurations.  Exercised: the output row (c0 + cl) * n_pts + pt of
                                    the last tiles, and the slab offsets b * n_pts.
  robot_serial_kernel / robot_query_kernel   int n_pts: the step ends reach n_pts + 2047 (rs_int_pts_ok, exact; the
                                    CPU tier pins it in tests/test_hostsim.py).  2^31 points (24 GB of input) are not
                                    run on the GPU.
  composed_paired_kernel            1-D over cfg_count * n_pts pairs in 64 bits (paired_index); no tile limit.
  robot_swept_kernel                1-D over points (n_pts < 2^31, exact: its point index is 64-bit), the tiles walked
                                    inside the block (n_tiles = rs_tile_count): no grid-row limit.  Exercised: the
                                    fold over tiles past 65535 and over 40 000 x 60 000 pairs.
  robot_clearance_kernel            one grid row per rs_tile tile: fused while rs_tile_count(cfg_count) <= 65535,
                                    else composed_clearance_kernel (1-D, 64-bit pair index).  Work index w over
                                    n_seg * chunks_per_seg in 64 bits; chunks at most 2^30 points (kRsMaxChunk: the
                                    point loop steps in int).  Exercised: keys (c0 + cl) * n_seg + b at 2.4e9 pairs.
  clearance_finish_kernel           1-D over cfg_count * n_seg, 64-bit.
  robot_paired_clearance_kernel     1-D over units of (configuration, segment, chunk), w / pairs in 64 bits: no tile
                                    limit.  Exercised past 65535 tiles; C * K >= 2^31 needs 24 GB of points and is not
                                    run.
  robot_self_clearance_kernel (+ finish)   1-D over (configuration, source, chunk) units, K < 2^24: no tile limit.
  robot_collision_cost_kernel (+ finish)   1-D over (tile, segment, chunk) units: u / n_tiles and sc / chunks_per_seg
                                    in 64 bits, the partial index ((c * n_seg + b) * cps + kc) * E in size_t.
                                    Exercised past 65535 tiles and at 2.4e9 pairs with 1 and 3 segments.

Every test reads the free device memory first and skips, naming its need, when there is less; peaks stay below about
12 GB, and nothing here launches a kernel outside its limits: every size above a limit is a legal call the library
routes elsewhere."""
import collections
import gc
import re

import numpy as np
import pytest
import torch

from helpers import arm_robot
from robot_ref import analyse, build_robot, check, joint_values, sample_points
pytestmark = pytest.mark.gpu

LIMIT = 65535 * 32              # configurations of 65535 full tiles
SIDES = (LIMIT, LIMIT + 1, LIMIT + 33)


def _need(gb):
    free = torch.cuda.mem_get_info()[0]
    if free < gb * 2 ** 30:
        pytest.skip(f"needs {gb} GB of free device memory, {free / 2 ** 30:.1f} GB free")


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# the project's kernels on the RobotSDF-family routes
KERNELS = ("robot_serial_kernel", "robot_query_kernel", "composed_cfgmajor_kernel", "composed_query_kernel",
           "composed_paired_kernel", "robot_swept_kernel", "composed_swept_kernel", "robot_clearance_kernel",
           "composed_clearance_kernel", "clearance_finish_kernel", "robot_paired_clearance_kernel",
           "composed_paired_clearance_kernel", "paired_clearance_finish_kernel", "robot_self_clearance_kernel",
           "self_clearance_finish_kernel", "robot_collision_cost_kernel", "collision_cost_finish_kernel")


def _graph_kernels(fn):
    """Counter of the project's kernels fn launches, read from the kernel nodes of a CUDA graph that captures fn (never
    replayed: its outputs are left unwritten and dropped).  Capture records every launch the calls enqueue, whatever
    else the process has run, where torch.profiler's activity records came back incomplete in long test processes.
    fn must not synchronise, and every cache it fills must be warm (a warm-up call of the same forms does that)."""
    import os
    import tempfile
    import warnings
    g = torch.cuda.CUDAGraph(keep_graph=True)         # the captured graph itself stays readable after capture
    g.enable_debug_mode()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        out = fn()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "graph.dot")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", UserWarning)        # torch announces every dump
            g.debug_dump(path)
        text = open(path).read()
    del out, g
    _free()
    # one record per node ("graph_0_node_3"[... label="{KERNEL ...}"], its label over several lines); a kernel node
    # names its function, mangled (19robot_serial_kernel...) or demangled, and the longest match wins
    # (paired_clearance_finish_kernel over clearance_finish_kernel)
    nodes = [n for n in re.split(r'\n(?="graph_\d+_node_\d+"\[)', text) if "{KERNEL" in n]
    names = collections.Counter()
    for n in nodes:
        hit = [k for k in KERNELS if re.search(rf"(?<![0-9]){len(k)}{k}|(?<![\w]){k}(?![\w])", n)]
        if hit:
            names[max(hit, key=len)] += 1
    if not names:
        print("no project kernel among the graph's kernel nodes:", [n[:400] for n in nodes[:3]])
    return names


def _route(what, names, want):
    """The project's kernels launched are exactly `want` {name: launches}."""
    got = dict(names)
    print(f"{what}: {dict(sorted(got.items()))}")
    assert got == want, (what, got, want)


def _same(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, k, int((x != y).reshape(len(x), -1).any(-1).sum()))


def _rows(t, per, lo, hi):
    return t.reshape(-1, per, *t.shape[1:])[lo:hi].reshape(-1, *t.shape[1:])


def _fold(a, b):
    """The swept result of two consecutive slabs from theirs: the later slab wins only with a strictly smaller value."""
    take = b[0] < a[0]
    return (torch.where(take, b[0], a[0]), torch.where(take[:, None], b[1], a[1]), torch.where(take, b[2], a[2]),
            torch.where(take, b[3], a[3]))


def _sample(C, n, seed):
    """About n configuration indices of [0, C): the first tile, the last full tile, the ragged tail and uniform ones."""
    last_full = (C // 32) * 32
    idx = np.concatenate([np.arange(32), np.arange(last_full - 32, C),
                          np.random.default_rng(seed).integers(0, C, n - 64 - (C - last_full))])
    return np.unique(idx)


def _robot(kind, tmp_path, C, seed):
    """(RobotSDF with C configurations installed, fp64 RefRobot or None, fp32 joint values)."""
    if kind == "nearest_arm":
        import workloads
        robot = arm_robot(tmp_path, "nearest")
        q = workloads.arm_configurations(C, seed=seed)
        robot.set_joint_configuration(q.cuda())
        return robot, None, q.numpy()
    robot, ref, text = build_robot("mixed", tmp_path)
    q = joint_values(ref, text, C, seed)
    robot.set_joint_configuration(torch.from_numpy(q).cuda())
    return robot, ref, q


# ------------------------------------------------------------------------------------ 65535 configuration tiles
@pytest.mark.parametrize("kind", ["nearest_arm", "mixed"])
def test_every_form_across_the_tile_limit(tmp_path, kind):
    """Point, paired, swept, clearance, paired-clearance, self-clearance and collision-cost queries on configuration
    slabs [0, C) of C = 65535 x 32, C + 1 and C + 33: (a) the kernels each launches, (b) the rows of the first tile, the
    last full tile and the ragged tail bit for bit against the same configurations queried as small slabs, and, on the
    mixed primitive robot, (c) those rows against the fp64 robot."""
    _need(8)
    A = SIDES[-1]
    robot, ref, q = _robot(kind, tmp_path, A, seed=5)
    comp = robot.sdf
    g = torch.Generator().manual_seed(3)
    if ref is not None:
        pts64 = sample_points(ref, ref.object_to_link(q[:64]), 12, seed=9)[:32]
    else:
        import workloads
        lo = [r[0] for r in workloads.ARM_QUERY_RANGE]; hi = [r[1] for r in workloads.ARM_QUERY_RANGE]
        pts64 = workloads.uniform_points(32, lo, hi, seed=9).double().numpy()
    pts = torch.from_numpy(pts64).float().cuda()                       # 32 shared points
    P = len(pts)
    cloud = (pts[torch.randint(0, P, (256,), generator=g)] + 0.05 * torch.randn(256, 3, generator=g).cuda())
    own = (pts[torch.randint(0, P, (A, 8), generator=g)] + 0.05 * torch.randn(A, 8, 3, generator=g).cuda())
    lp = robot.link_surface_points(num_points=32, seed=1)
    allowed = robot.self_collision_pairs()
    allowed = allowed.cpu() if torch.is_tensor(allowed) else allowed      # read on the host: no copy under capture
    m = 0.05
    for C in SIDES:
        tail = _sample(C, 2000, seed=C)
        slabs = [(0, 32), ((C // 32) * 32 - 32, C - ((C // 32) * 32 - 32))]

        # (a) the seven calls captured into one CUDA graph: no kernel serves two forms, so the launch counts name
        # the route of each.  The point query launches robot_serial_kernel once per slab of at most 65531 tiles;
        # clearance is fused while its tiles fit the grid rows, the composition kernel beyond.
        def every_form(n=C):
            return dict(query=comp.query(pts, cfg_count=n, return_which=True),
                        paired=comp.query_paired(own[:n], cfg_count=n),
                        swept=comp.query_swept(pts, cfg_count=n, return_which=True),
                        clearance=comp.query_clearance(cloud, cfg_count=n, return_which=True),
                        paired_clearance=comp.query_paired_clearance(own[:n].reshape(n, 2, 4, 3), cfg_count=n,
                                                                     return_which=True),
                        self_clearance=comp.query_self_clearance(lp, allowed, cfg_count=n, return_which=True),
                        collision_cost=comp.query_collision_cost(cloud, m, cfg_count=n))
        if C == SIDES[0]:
            every_form(64)                   # warm every cache the calls fill before the first capture
        names = _graph_kernels(every_form)
        _route(f"{kind} C={C}", names,
               {"robot_serial_kernel": 1 if C <= LIMIT else 2, "composed_paired_kernel": 1, "robot_swept_kernel": 1,
                "robot_clearance_kernel" if C <= LIMIT else "composed_clearance_kernel": 1,
                "clearance_finish_kernel": 1, "robot_paired_clearance_kernel": 1, "paired_clearance_finish_kernel": 1,
                "robot_self_clearance_kernel": 1, "self_clearance_finish_kernel": 1, "robot_collision_cost_kernel": 1,
                "collision_cost_finish_kernel": 1})
        out = every_form()

        # (b) and (c), form by form
        v, gr, w = out.pop("query")
        for b, n in slabs:
            _same((_rows(v, P, b, b + n), _rows(gr, P, b, b + n), _rows(w, P, b, b + n)),
                  comp.query(pts, cfg_begin=b, cfg_count=n, return_which=True), (kind, "query", C, b))
        if ref is not None:
            idx = torch.from_numpy(tail).cuda()
            check(f"{kind} query C={C} sample={len(tail)}", analyse(ref, q[tail], pts64),
                  v.reshape(C, P)[idx].cpu().numpy(), gr.reshape(C, P, 3)[idx].cpu().numpy(),
                  w.reshape(C, P)[idx].cpu().numpy())
        del v, gr, w

        # paired: 8 own points per configuration
        pv_, pg = out.pop("paired")
        for b, n in slabs:
            _same((_rows(pv_, 8, b, b + n), _rows(pg, 8, b, b + n)),
                  comp.query_paired(own[b:b + n], cfg_begin=b, cfg_count=n), (kind, "paired", C, b))
        if ref is not None:
            idx = torch.from_numpy(tail).cuda()
            own64 = own[idx].double().cpu().numpy()
            check(f"{kind} paired C={C} sample={len(tail)}", analyse(ref, q[tail], own64),
                  pv_.reshape(C, 8)[idx].cpu().numpy(), pg.reshape(C, 8, 3)[idx].cpu().numpy())
        del pv_, pg

        # swept: the fold over every tile equals the fold of two slab calls
        sw = out.pop("swept")
        h = (C // 64) * 32
        _same(sw, _fold(comp.query_swept(pts, cfg_begin=0, cfg_count=h, return_which=True),
                        comp.query_swept(pts, cfg_begin=h, cfg_count=C - h, return_which=True)),
              (kind, "swept", C))
        del sw

        # clearance over the 256-point cloud
        cl = out.pop("clearance")
        for b, n in slabs:
            _same([t[b:b + n] for t in cl], comp.query_clearance(cloud, cfg_begin=b, cfg_count=n, return_which=True),
                  (kind, "clearance", C, b))
        if ref is not None:
            _check_clearance(f"{kind} clearance C={C}", ref, q[tail], cloud, [t[torch.from_numpy(tail).cuda()]
                                                                            for t in cl])
        del cl

        # paired clearance: 8 own points per configuration, 2 segments of 4
        pc = out.pop("paired_clearance")
        for b, n in slabs:
            _same([t[2 * b:2 * (b + n)] for t in pc],
                  comp.query_paired_clearance(own[b:b + n].reshape(n, 2, 4, 3), cfg_begin=b, cfg_count=n,
                                              return_which=True), (kind, "paired clearance", C, b))
        del pc

        # self-clearance
        sc = out.pop("self_clearance")
        for b, n in slabs:
            _same([t[b:b + n] for t in sc], comp.query_self_clearance(lp, allowed, cfg_begin=b, cfg_count=n,
                                                                      return_which=True), (kind, "self", C, b))
        del sc

        # collision cost over the 256-point cloud
        cc = out.pop("collision_cost")
        for b, n in slabs:
            _same([t[b:b + n] for t in cc], comp.query_collision_cost(cloud, m, cfg_begin=b, cfg_count=n),
                  (kind, "collision cost", C, b))
        assert ref is None or float(cc[0].sum()) > 0
        del cc
        _free()
    del robot, comp, own
    _free()


def _check_clearance(label, ref, q, cloud, got, min_decided=0.8):
    """Clearance rows (value, gradient, point, link) of configurations q against the fp64 minimum over the cloud:
    the value within the largest tolerance of the row, point, link and gradient where fp64 decides the minimum."""
    pts = cloud.double().cpu().numpy()
    truth = analyse(ref, q, pts)
    rv, tol = truth["value"], truth["tol"]
    A = len(q)
    cv, cg, ci, cw = (t.cpu().numpy() for t in got)
    p_best = rv.argmin(1)
    rows = np.arange(A)
    srt = np.sort(rv, axis=1)
    tmax = tol.max(1)
    ok = (srt[:, 1] - srt[:, 0] > 2 * tmax) & truth["decided"][rows, p_best]
    err = np.abs(cv - srt[:, 0])
    print(f"{label}: max |value error| {err.max():.3g}, error / bound max {(err / tmax).max():.3f}, "
          f"skipped {int((~ok).sum())} of {A}")
    assert (err <= tmax).all() and ok.mean() >= min_decided
    assert (ci[ok] == p_best[ok]).all() and (cw[ok] == truth["which"][rows, p_best][ok]).all()
    assert (np.abs(cg - truth["grad"][rows, p_best]).max(1) <= truth["gtol"][rows, p_best])[ok].all()


# ------------------------------------------------------------------------------------ 2^31 pairs and beyond
C_BIG, N_BIG = 40_000, 60_000                     # 2.4e9 pairs


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    """The mixed primitive robot at 40 000 configurations and 60 000 points (in 3 segments of 20 000: not a multiple
    of the collision cost's 512-point chunk)."""
    _need(4)
    robot, ref, q = _robot("mixed", tmp_path_factory.mktemp("big"), C_BIG, seed=21)
    pts64 = sample_points(ref, ref.object_to_link(q[:256]), 20_000, seed=22)
    rng = np.random.default_rng(23)
    pts64 = pts64[rng.integers(0, len(pts64), N_BIG)] + rng.normal(0, 0.01, (N_BIG, 3))
    pts64 = pts64.astype(np.float32).astype(np.float64)
    yield robot, ref, q, pts64, torch.from_numpy(pts64).float().cuda()
    del robot
    _free()


def _big_sample():
    """Configurations of the sampled fp64 checks: some of the first slab, and every 250th above 2^31 / N (the first
    whose pair index c * N passes 2^31 is 35 792)."""
    first = (2 ** 31) // N_BIG + 1
    return np.unique(np.concatenate([np.arange(0, 16), np.arange(first, C_BIG, 250), [first, C_BIG - 1]]))


SLAB = 10_000                                     # 6e8 pairs per slab


def test_routes_past_2_31_pairs(big):
    """The kernels the 2.4e9-pair calls below take, from one CUDA graph capturing the same calls on 64-configuration
    slabs (for these forms the route depends on the link set and the point count, not on cfg_count)."""
    robot, ref, q, pts64, pts = big
    comp = robot.sdf
    b = C_BIG - 64

    def calls():
        return [comp.query_clearance(pts, cfg_begin=b, cfg_count=64),
                comp.query_swept(pts, cfg_begin=b, cfg_count=64)] + \
            [comp.query_collision_cost(pts.reshape(n_seg, -1, 3), 0.05, cfg_begin=b, cfg_count=64) for n_seg in (1, 3)]
    calls()                                  # warm every cache the calls fill before the capture
    _route("clearance, swept, collision cost (1 and 3 segments) at 40000 x 60000", _graph_kernels(calls),
           {"robot_clearance_kernel": 1, "clearance_finish_kernel": 1, "robot_swept_kernel": 1,
            "robot_collision_cost_kernel": 2, "collision_cost_finish_kernel": 2})


def test_clearance_past_2_31_pairs(big):
    """Clearance over 40 000 x 60 000 pairs: bit for bit the rows of four 10 000-configuration slabs, and the sampled
    configurations above 2^31 / N against the fp64 robot."""
    robot, ref, q, pts64, pts = big
    comp = robot.sdf
    full = comp.query_clearance(pts, return_which=True)
    for b in range(0, C_BIG, SLAB):
        _same([t[b:b + SLAB] for t in full], comp.query_clearance(pts, cfg_begin=b, cfg_count=SLAB, return_which=True),
              ("clearance slab", b))
    s = _big_sample()
    _check_clearance(f"clearance 40000 x 60000 sample={len(s)}", ref, q[s], pts,
                     [t[torch.from_numpy(s).cuda()] for t in full], min_decided=0.1)
    del full
    _free()


def test_swept_past_2_31_pairs(big):
    """Swept over 40 000 x 60 000 pairs: bit for bit the fold of two 20 000-configuration slabs, and the minimum over
    configurations against the fp64 robot at sampled points, with the winning configuration's fp64 value."""
    robot, ref, q, pts64, pts = big
    comp = robot.sdf
    full = comp.query_swept(pts, return_which=True)
    h = C_BIG // 2
    _same(full, _fold(comp.query_swept(pts, cfg_begin=0, cfg_count=h, return_which=True),
                      comp.query_swept(pts, cfg_begin=h, cfg_count=h, return_which=True)), "swept slabs")
    # at sampled points: the swept value is at most every sampled configuration's fp64 value (+ its tolerance), and
    # it is the fp64 value of the configuration it names (the winner's own point query)
    j = np.random.default_rng(24).integers(0, N_BIG, 200)
    s = _big_sample()
    sv, scfg = full[0].cpu().numpy()[j], full[2].cpu().numpy()[j]
    truth = analyse(ref, q[s], pts64[j])
    bound = (truth["value"] + truth["tol"]).min(0)
    win = analyse(ref, q[scfg], pts64[j][:, None, :])
    err = np.abs(sv - win["value"][:, 0])
    print(f"swept 40000 x 60000: {len(j)} points, max |value error| at the named configuration {err.max():.3g}, "
          f"error / bound max {(err / win['tol'][:, 0]).max():.3f}, configurations above 2^31 / N named "
          f"{int((scfg > 2 ** 31 // N_BIG).sum())}")
    assert (sv <= bound).all()
    assert (err <= win["tol"][:, 0]).all()
    del full
    _free()


@pytest.mark.parametrize("n_seg", [1, 3])
def test_collision_cost_past_2_31_pairs(big, n_seg):
    """Collision cost over 40 000 x 60 000 pairs, as one segment and as 3 segments of 20 000 points (not a multiple of
    the 512-point chunk): bit for bit the rows of four 10 000-configuration slabs, and the sampled configurations
    above 2^31 / N against the fp64 robot's hinge cost."""
    robot, ref, q, pts64, pts = big
    comp = robot.sdf
    m = 0.05
    cloud = pts.reshape(n_seg, N_BIG // n_seg, 3)
    full = comp.query_collision_cost(cloud, m)
    for b in range(0, C_BIG, SLAB):
        _same([t[b * n_seg:(b + SLAB) * n_seg] for t in full],
              comp.query_collision_cost(cloud, m, cfg_begin=b, cfg_count=SLAB), ("collision cost slab", n_seg, b))
    s = _big_sample()
    truth = analyse(ref, q[s], pts64)
    d = truth["value"]                                                       # [len(s), N]
    m32 = float(np.float32(m))
    hinge = np.maximum(0.0, m32 - d) ** 2
    cost = hinge.reshape(len(s), n_seg, -1).sum(-1)
    # the cost's error: each pair's hinge moves by at most 2 (m - d) tol + tol^2, and the fp32 sum rounds
    dv = (2 * np.maximum(0.0, m32 - d + truth["tol"]) * truth["tol"] + truth["tol"] ** 2)
    bound = dv.reshape(len(s), n_seg, -1).sum(-1) + 1e-5 * cost + 1e-12
    got = full[0].reshape(C_BIG, n_seg).cpu().numpy()[s]
    err = np.abs(got - cost)
    print(f"collision cost 40000 x 60000, {n_seg} segment(s), sample={len(s)}: max |cost error| {err.max():.3g}, "
          f"error / bound max {(err / bound).max():.3f}, rows with contact {int((cost > 0).sum())} of {cost.size}")
    assert (err <= bound).all()
    assert (cost > 0).any()
    del full
    _free()
