// Host build of the self-clearance query of pvb_device.cuh (ComposedSDF.self_clearance /
// pvb_composed_query_self_clearance) behind a small C interface for tests/test_self_clearance_cpu.py.
//   simscl_fused follows robot_self_clearance_kernel unit by unit: work units (configuration, source sub-SDF, chunk of
//   its points) numbered chunk-major and run in a chosen order; each unit reads its configuration's one key as the
//   seed, its lanes pose the chunk's link points with W_i step by step and run rs_swept_pair against min(running
//   value, seed) with the masked links given a +inf bound and refused inside the visit, optionally with the per-step
//   warp minimum of the running values, and the unit's key minimum is folded into the key.
//   simscl_finish is self_clearance_finish_kernel's per-configuration work.
//   simscl_key packs (value, i, k) the way both do.
// Test infrastructure only.
#include <algorithm>
#include <random>
#include <vector>

#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline void load_rows(const float *xforms, int n_cfg, int s, int cfg, float4 &r0, float4 &r1, float4 &r2) {
    const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
    r0 = row[0]; r1 = row[1]; r2 = row[2];
}

// the kernels' evaluation of a link: primitive, trilinear or nearest-voxel lookup (the same arithmetic as
// robot_primitive / robot_lookup_trilinear / robot_lookup)
static inline float4 eval_link(const pvb_sdf_desc &d, f3 q) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    SdfOut o;
    if (d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
    else if (d.flags & PVB_GRID_TRILINEAR) o = grid_trilinear_eval(d, q);
    else o = grid_eval<false, true>(d, st, q, 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

extern "C" uint64_t simscl_key(float v, int i, int k) { return self_clearance_key(v, i, k); }

// transform_points_paired_kernel's per-point work with every configuration's W on the same K points: out[c][k] =
// composed_xform(W_c, pts[k])
extern "C" void simscl_pose(const float *w, int n_cfg, const float *pts, int K, float *out) {
    for (int c = 0; c < n_cfg; ++c) {
        const float4 *row = reinterpret_cast<const float4 *>(w + (size_t)c * 16);
        for (int k = 0; k < K; ++k) {
            const f3 q = composed_xform(row[0], row[1], row[2], mk3(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]));
            float *o = out + 3 * ((size_t)c * K + k);
            o[0] = q.x; o[1] = q.y; o[2] = q.z;
        }
    }
}

// masks[i]: bit j allows (i, j), the diagonal already cleared.  chunk: points per unit; lanes: threads per unit (32: a
// warp); share: the running value is the warp minimum after every step; unit_order 0 ascending, 1 descending, 2
// shuffled by shuffle_seed; seeded = 0: units do not read the key when they start; first >= 0: every lane visits link
// `first` first (else its own nearest sphere).  visits[i * 8 + j] counts the evaluations of link j for points of i.
extern "C" void simscl_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, const float *inv_xforms,
                             int n_cfg, int cfg_begin, int cfg_count, const float *link_pts, int K,
                             const unsigned char *masks, int chunk, int lanes, int share, int unit_order,
                             int shuffle_seed, int seeded, int first, uint64_t *keys, long long *visits) {
    float sph_rad[8], visit_margin[8];
    for (int s = 0; s < 8; ++s) {
        if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
        else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
    }
    for (int c = 0; c < cfg_count; ++c) keys[c] = ~0ull;
    for (int q = 0; q < 64; ++q) visits[q] = 0;
    std::vector<int> src;
    for (int i = 0; i < n_sdf; ++i)
        if (masks[i]) src.push_back(i);
    const long long n_src = (long long)src.size(), pairs = (long long)cfg_count * n_src;
    const int per_src = (K + chunk - 1) / chunk;
    std::vector<long long> units;
    for (long long w = 0; w < pairs * per_src; ++w) units.push_back(w);
    if (unit_order == 1) std::reverse(units.begin(), units.end());
    if (unit_order == 2) std::shuffle(units.begin(), units.end(), std::mt19937(shuffle_seed));
    for (const long long w : units) {
        const long long kc = w / pairs, r = w - kc * pairs;
        const int c = (int)(r / n_src), i = src[r - (long long)c * n_src];
        const int cfg = cfg_begin + c;
        const unsigned mask = masks[i];
        const int k0 = (int)kc * chunk;
        const int len = std::min(chunk, K - k0);
        f3 cen[8];
        for (int s = 0; s < 8; ++s) {
            cen[s] = mk3(0.f, 0.f, 0.f);
            if (s < n_sdf) {
                float4 r0, r1, r2;
                load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
                cen[s] = rs_sphere_centre(descs[s], r0, r1, r2);
            }
        }
        float4 w0, w1, w2;
        load_rows(inv_xforms, n_cfg, i, cfg, w0, w1, w2);
        const uint64_t seed_key = seeded ? keys[c] : ~0ull;
        const float seed = clearance_key_value(seed_key);
        std::vector<uint64_t> run(lanes, ~0ull);
        std::vector<float> rv(lanes, PVB_INF);
        for (int j0 = 0; j0 < len; j0 += lanes) {
            for (int l = 0; l < lanes && j0 + l < len; ++l) {
                const int k = k0 + j0 + l;
                const float *lp = link_pts + 3 * ((size_t)i * K + k);
                const f3 p = composed_xform(w0, w1, w2, mk3(lp[0], lp[1], lp[2]));
                float lb[8], key[8];
                for (int s = 0; s < 8; ++s) {
                    lb[s] = ((mask >> s) & 1u) ? rs_sphere_lb(p, cen[s].x, cen[s].y, cen[s].z, sph_rad[s]) : PVB_INF;
                    key[s] = rs_bound_key(lb[s], ~7, s);
                }
                auto link = [&](const int si, const float thr, float4 &o) -> bool {
                    if (!((mask >> si) & 1u)) return false;
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                    const f3 q = composed_xform(r0, r1, r2, p);
                    const float tm = thr + visit_margin[si];
                    if (tm < 0.f || composed_aabb_lb2(descs[si], q) > tm * tm) return false;
                    o = eval_link(descs[si], q);
                    ++visits[i * 8 + si];
                    return true;
                };
                float best;
                f3 bg;
                int bs;
                rs_swept_pair(lb, first >= 0 ? first : rs_nearest(key, n_sdf), fminf(rv[l], seed), link, best, bg, bs);
                if (bs >= 0) {
                    const uint64_t kk = self_clearance_key(best, i, k);
                    if (kk < run[l]) { run[l] = kk; rv[l] = best; }
                }
            }
            if (share)
                for (int g0 = 0; g0 < lanes; g0 += 32) {
                    float m = PVB_INF;
                    for (int l = g0; l < std::min(g0 + 32, lanes); ++l) m = fminf(m, rv[l]);
                    for (int l = g0; l < std::min(g0 + 32, lanes); ++l) rv[l] = m;
                }
        }
        uint64_t m = ~0ull;
        for (int l = 0; l < lanes; ++l) m = std::min(m, run[l]);
        keys[c] = std::min(keys[c], m);
    }
}

// self_clearance_finish_kernel: the point named by each configuration's key, posed again and evaluated against the
// allowed links of its source in index order
extern "C" void simscl_finish(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, const float *inv_xforms,
                              int n_cfg, int cfg_begin, int cfg_count, const float *link_pts, int K,
                              const unsigned char *masks, const uint64_t *keys, float *out_val, float *out_grad,
                              int *out_src, int *out_point, int *out_which) {
    for (int c = 0; c < cfg_count; ++c) {
        const int cfg = cfg_begin + c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
        auto load_inv = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
            load_rows(inv_xforms, n_cfg, s, cfg, r0, r1, r2);
        };
        auto load_pt = [&](int i, int k) {
            const float *lp = link_pts + 3 * ((size_t)i * K + k);
            return mk3(lp[0], lp[1], lp[2]);
        };
        const SelfClearanceOut o = self_clearance_finish_one(keys[c], masks, n_sdf, load_xf, load_inv, load_pt,
                                                             [&](int s, f3 q) { return eval_link(descs[s], q); });
        out_val[c] = o.val;
        out_grad[3 * c] = o.grad.x; out_grad[3 * c + 1] = o.grad.y; out_grad[3 * c + 2] = o.grad.z;
        out_src[c] = o.src; out_point[c] = o.point; out_which[c] = o.which;
    }
}
