// Host build of the swept composed query of pvb_device.cuh (ComposedSDF.swept / pvb_composed_query_swept) behind a
// small C interface for tests/test_swept_cpu.py.  simswept_fused follows robot_swept_kernel point by point: the
// configuration tiles of rs_tile in ascending order, rs_swept_pair for every lane of a tile with the point's best from
// earlier tiles, the lexicographic winner of the tile (swept_before) and swept_fold, the rotation back at the end.
// simswept_generic is the per-thread work of composed_swept_kernel.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline void load_rows(const float *xforms, int n_cfg, int s, int cfg, float4 &r0, float4 &r1, float4 &r2) {
    const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
    r0 = row[0]; r1 = row[1]; r2 = row[2];
}

// robot_swept_kernel's evaluation of a link: primitive, trilinear or nearest-voxel lookup (the same arithmetic as
// robot_primitive / robot_lookup_trilinear / robot_lookup)
static inline float4 eval_link(const pvb_sdf_desc &d, f3 q) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    SdfOut o;
    if (d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
    else if (d.flags & PVB_GRID_TRILINEAR) o = grid_trilinear_eval(d, q);
    else o = grid_eval<false, true>(d, st, q, 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

// first >= 0: every point group visits link `first` first instead of its nearest sphere (any link is a valid first
// visit); lanes_reversed: the tile's lanes are folded from the last to the first (the winner does not depend on it).
extern "C" void simswept_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                               int cfg_count, const float *pts, long long n_pts, int first, int lanes_reversed,
                               float *out_val, float *out_grad, int *out_cfg, int *out_which, long long *n_evals) {
    float sph_rad[8], visit_margin[8];
    for (int s = 0; s < 8; ++s) {
        if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
        else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
    }
    const int low3_off = ~7;
    const int n_tiles = (cfg_count >> 5) + __builtin_popcount((unsigned)(cfg_count & 31));
    long long evals = 0;
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : evals)
    for (long long i = 0; i < n_pts; ++i) {
        const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        long long ev = 0;           // (a lambda must not capture the reduction variable itself)
        SweptBest b;
        b.val = PVB_INF; b.grad = mk3(0.f, 0.f, 0.f); b.cfg = -1; b.which = -1;
        for (int t = 0; t < n_tiles; ++t) {
            int c0, lc_log2;
            rs_tile(cfg_count, t, c0, lc_log2);
            const int LC = 1 << lc_log2;
            const float bp = b.val;
            int pred = -1;
            float wv = PVB_INF, wbest = PVB_INF;
            f3 wbg = mk3(0.f, 0.f, 0.f);
            int wl = -1, wbs = -1;
            for (int k = 0; k < LC; ++k) {
                const int cl = lanes_reversed ? LC - 1 - k : k;
                const int cfg = cfg_begin + c0 + cl;
                float lb[8], key[8];
                for (int s = 0; s < 8; ++s) {
                    f3 cen = mk3(0.f, 0.f, 0.f);
                    if (s < n_sdf) {
                        float4 r0, r1, r2;
                        load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
                        cen = rs_sphere_centre(descs[s], r0, r1, r2);
                    }
                    lb[s] = rs_sphere_lb(p, cen.x, cen.y, cen.z, sph_rad[s]);
                    key[s] = rs_bound_key(lb[s], low3_off, s);
                }
                if (pred < 0) {         // the point group's first lane (configuration c0) names the first visit
                    float key0[8];
                    for (int s = 0; s < 8; ++s) {
                        f3 cen = mk3(0.f, 0.f, 0.f);
                        if (s < n_sdf) {
                            float4 r0, r1, r2;
                            load_rows(xforms, n_cfg, s, cfg_begin + c0, r0, r1, r2);
                            cen = rs_sphere_centre(descs[s], r0, r1, r2);
                        }
                        key0[s] = rs_bound_key(rs_sphere_lb(p, cen.x, cen.y, cen.z, sph_rad[s]), low3_off, s);
                    }
                    pred = first >= 0 ? first : rs_nearest(key0, n_sdf);
                }
                auto link = [&](const int si, const float thr, float4 &o) -> bool {
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                    const f3 q = composed_xform(r0, r1, r2, p);
                    const float tm = thr + visit_margin[si];
                    if (tm < 0.f || composed_aabb_lb2(descs[si], q) > tm * tm) return false;
                    o = eval_link(descs[si], q);
                    ++ev;
                    return true;
                };
                float best;
                f3 bg;
                int bs;
                rs_swept_pair(lb, pred, bp, link, best, bg, bs);
                if (wl < 0 || swept_before(best, cl, wv, wl)) { wv = best; wl = cl; wbest = best; wbg = bg; wbs = bs; }
            }
            swept_fold(b, wbest, wbg, c0 + wl, wbs);
        }
        const int cfg = cfg_begin + b.cfg;
        float4 r0, r1, r2;
        load_rows(xforms, n_cfg, b.which < 0 ? 0 : b.which, cfg, r0, r1, r2);
        const f3 go = composed_rotate_back(r0, r1, r2, b.grad);
        out_val[i] = b.val;
        out_grad[3 * i] = go.x; out_grad[3 * i + 1] = go.y; out_grad[3 * i + 2] = go.z;
        out_cfg[i] = cfg;
        out_which[i] = b.which;
        evals += ev;
    }
    *n_evals = evals;
}

// composed_swept_kernel<kMesh = true, kExt = true>: composed_point for every configuration, folded by swept_fold
extern "C" void simswept_generic(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                                 int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_pts,
                                 float margin_max, float *out_val, float *out_grad, int *out_cfg, int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long i = 0; i < n_pts; ++i) {
        const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        SweptBest b;
        b.val = PVB_INF; b.grad = mk3(0.f, 0.f, 0.f); b.cfg = -1; b.which = -1;
        for (int c = 0; c < cfg_count; ++c) {
            const int cfg = cfg_begin + c;
            auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
            const ComposedOut o = composed_point<true, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                             (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i, 1,
                                                             margin_max);
            swept_fold(b, o.val, o.grad, cfg, o.which);
        }
        out_val[i] = b.val;
        out_grad[3 * i] = b.grad.x; out_grad[3 * i + 1] = b.grad.y; out_grad[3 * i + 2] = b.grad.z;
        out_cfg[i] = b.cfg;
        out_which[i] = b.which;
    }
}
