// Host build of the device building blocks (pvb_device.cuh) behind a small C interface for tests/test_hostsim.py.
// Every loop body below is the per-thread work of the corresponding kernel: one call of grid_eval / mesh_eval /
// sphere_eval / bvh_winding per query, with host pointers in the descriptor.  Test infrastructure only.
#include "cuda_runtime.h"

// traversal statistics (SURVEY 8d-iii): per-thread counters behind the header's PVB_STAT hook
struct SimStats { long long closest_nodes, closest_tris, parity_nodes, parity_tris; };
static thread_local SimStats t_stats = {0, 0, 0, 0};
#define PVB_STAT(counter) ++t_stats.counter;
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline f3 point(const float *pts, long long i) { return mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]); }

extern "C" void sim_grid_lookup(const pvb_sdf_desc *g, const float *pts, long long n, float *val, float *grad,
                                long long *key) {
    NodeStage st; st.smem = nullptr; st.n = 0;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        long long k = -1;
        // <kMesh = true>: the instantiation that can fall back to the mesh for PVB_GRID_OOB_GT, like grid_lookup_*<true>
        const SdfOut o = grid_eval<true, false>(*g, st, point(pts, i), PVB_MESH_DEFAULT, (uint64_t)i, &k);
        val[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
        if (key) key[i] = k;
    }
}

// the branchy variant the composed kernels use (<kBranchOOB = true>) must agree with the select-based one
extern "C" void sim_grid_lookup_branchy(const pvb_sdf_desc *g, const float *pts, long long n, float *val, float *grad) {
    NodeStage st; st.smem = nullptr; st.n = 0;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        const SdfOut o = grid_eval<false, true>(*g, st, point(pts, i), 0u, (uint64_t)i, nullptr);
        val[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
    }
}

// stats_out (optional): totals over the n queries {closest nodes, closest triangles, parity nodes, parity triangles}
extern "C" void sim_mesh_query(const pvb_sdf_desc *m, const float *pts, long long n, uint32_t mode, float *dist,
                               float *grad, float *closest, int *face, long long *stats_out) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    long long a = 0, b = 0, c2 = 0, d2 = 0;
#pragma omp parallel reduction(+ : a, b, c2, d2)
    {
        t_stats = SimStats{0, 0, 0, 0};
#pragma omp for schedule(dynamic, 256)
        for (long long i = 0; i < n; ++i) {
            f3 c; int f = -1;
            const SdfOut o = mesh_eval(*m, st, point(pts, i), mode, (uint64_t)i, &c, &f);
            dist[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
            if (closest) { closest[3 * i] = c.x; closest[3 * i + 1] = c.y; closest[3 * i + 2] = c.z; }
            if (face) face[i] = f;
        }
        a += t_stats.closest_nodes; b += t_stats.closest_tris; c2 += t_stats.parity_nodes; d2 += t_stats.parity_tris;
    }
    if (stats_out) { stats_out[0] = a; stats_out[1] = b; stats_out[2] = c2; stats_out[3] = d2; }
}

// crossing parity alone: the exact axis-aligned walk (closed meshes) and the watertight diagonal ray
extern "C" void sim_parity(const pvb_sdf_desc *m, const float *pts, long long n, const float *dirs, int *parity_x,
                           int *parity_ray) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const float4 *nodes = reinterpret_cast<const float4 *>(m->nodes), *tris = reinterpret_cast<const float4 *>(m->tris);
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < n; ++i) {
        if (parity_x) parity_x[i] = bvh_parity_x(nodes, st, tris, point(pts, i));
        if (parity_ray) parity_ray[i] = bvh_parity(nodes, st, tris, point(pts, i), point(dirs, i));
    }
}

extern "C" void sim_winding(const pvb_sdf_desc *m, const float *pts, long long n, float *w) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const float4 *nodes = reinterpret_cast<const float4 *>(m->nodes), *tris = reinterpret_cast<const float4 *>(m->tris);
    const float4 *wn = reinterpret_cast<const float4 *>(m->wn_nodes);
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < n; ++i) w[i] = bvh_winding(nodes, wn, st, tris, point(pts, i));
}

// ComposedSDF / RobotSDF for every (configuration, point) pair: the loop of the composed kernels (visit the
// sub-SDFs in `order`, composed_xform -> composed_consider, rotate the winning gradient back) around the header's
// primitives, through the composed_consider<kMesh, kExt> instantiation that `mesh` and `ext` pick.
// xforms: [n_sdf * n_cfg][16] row-major, sub-SDF-major like pvb_composed_query; idx as in the kernels.
template <bool kMesh, bool kExt>
static void composed_loop(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                          int n_cfg, const float *pts, long long n_pts, uint32_t mesh_mode, float *out_val,
                          float *out_grad, int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
#pragma omp parallel for schedule(dynamic, 64) collapse(2)
    for (int c = 0; c < n_cfg; ++c) {
        for (long long i = 0; i < n_pts; ++i) {
            const f3 p = point(pts, i);
            float best = PVB_INF; f3 bg = mk3(0.f, 0.f, 0.f); int bs = -1;
            for (int si = 0; si < n_sdf; ++si) {
                const int s = order ? order[si] : si;
                const float4 *row = xf_rows(xforms, n_cfg, s, c);
                const uint64_t idx = ((uint64_t)c * (uint64_t)n_pts + (uint64_t)i) * (uint64_t)n_sdf + (uint64_t)s;
                composed_consider<kMesh, kExt>(descs[s], st, s, composed_xform(row[0], row[1], row[2], p), mesh_mode,
                                               idx, best, bg, bs);
            }
            const float4 *row = xf_rows(xforms, n_cfg, max(bs, 0), c);
            const f3 go = composed_rotate_back(row[0], row[1], row[2], bg);
            const long long o = (long long)c * n_pts + i;
            out_val[o] = best; out_grad[3 * o] = go.x; out_grad[3 * o + 1] = go.y; out_grad[3 * o + 2] = go.z;
            if (out_which) out_which[o] = bs;
        }
    }
}

extern "C" void sim_composed(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                             int n_cfg, const float *pts, long long n_pts, uint32_t mesh_mode, int mesh, int ext,
                             float *out_val, float *out_grad, int *out_which) {
    using Loop = decltype(&composed_loop<true, true>);
    static const Loop loops[2][2] = {{composed_loop<false, false>, composed_loop<false, true>},
                                     {composed_loop<true, false>, composed_loop<true, true>}};
    loops[mesh != 0][ext != 0](descs, n_sdf, order, xforms, n_cfg, pts, n_pts, mesh_mode, out_val, out_grad, out_which);
}

extern "C" void sim_sphere(float radius, const float *pts, long long n, float *val, float *grad) {
    for (long long i = 0; i < n; ++i) {
        const SdfOut o = sphere_eval(radius, point(pts, i));
        val[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
    }
}

extern "C" float sim_hash_normal(uint32_t seed, unsigned long long idx, uint32_t comp) { return hash_normal(seed, idx, comp); }

// index arithmetic of robot_serial_kernel
extern "C" void sim_rs_tile(int cfg_count, int t, int *c0, int *lc_log2) { rs_tile(cfg_count, t, *c0, *lc_log2); }
extern "C" int sim_rs_tile_count(int cfg_count) { return rs_tile_count(cfg_count); }
extern "C" int sim_rs_int_pts_ok(long long n_pts) { return rs_int_pts_ok(n_pts) ? 1 : 0; }
extern "C" void sim_rs_flush_piece(int c, int chunk_log2, int sub_log2, int w_log2, int *is_val, int *row, int *part) {
    bool v;
    rs_flush_piece(c, chunk_log2, sub_log2, w_log2, v, *row, *part);
    *is_val = v ? 1 : 0;
}

// nearest-sphere selection of robot_serial_kernel: bounds -> keys -> smallest key -> link index (n rows of 8 bounds)
extern "C" void sim_rs_nearest(const float *lb, long long n, int n_sdf, int *pred) {
    for (long long i = 0; i < n; ++i) {
        float key[8];
        for (int si = 0; si < 8; ++si) key[si] = rs_bound_key(lb[8 * i + si], ~7, si);
        pred[i] = rs_nearest(key, n_sdf);
    }
}

// closest-point walk with a per-query initial search radius (squared): how many node visits / triangle tests are
// irreducible once the answer is known (scripts/traversal_stats.py, the lower bound any seeding scheme could reach)
extern "C" void sim_closest_seeded(const pvb_sdf_desc *m, const float *pts, long long n, const float *init_d2,
                                   long long *stats_out) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    long long a = 0, b = 0;
#pragma omp parallel reduction(+ : a, b)
    {
        t_stats = SimStats{0, 0, 0, 0};
#pragma omp for schedule(dynamic, 256)
        for (long long i = 0; i < n; ++i)
            (void)bvh_closest(reinterpret_cast<const float4 *>(m->nodes), st, reinterpret_cast<const float4 *>(m->tris),
                              point(pts, i), init_d2 ? init_d2[i] : PVB_INF);
        a += t_stats.closest_nodes; b += t_stats.closest_tris;
    }
    stats_out[0] = a; stats_out[1] = b;
}
