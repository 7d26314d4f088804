// Host build of the clearance query of pvb_device.cuh (ComposedSDF.clearance / pvb_composed_query_clearance) behind a
// small C interface for tests/test_clearance_cpu.py.
//   simclear_fused follows robot_clearance_kernel block by block: work units (configuration tile, chunk of one
//   segment) in a chosen order, each lane of a unit seeded from the keys left by earlier units, rs_swept_pair per
//   (point, lane) against min(running value, seed), the per-configuration minimum over the unit's point groups folded
//   into the keys.  simclear_generic is composed_clearance_kernel's per-pair work, simclear_finish the per-(configuration,
//   segment) work of clearance_finish_kernel, simclear_serial_pairs robot_serial_kernel's visit sequence per pair.
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

// robot_clearance_kernel's evaluation of a link: primitive, trilinear or nearest-voxel lookup (the same arithmetic as
// robot_primitive / robot_lookup_trilinear / robot_lookup)
static inline float4 eval_link(const pvb_sdf_desc &d, f3 q) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    SdfOut o;
    if (d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
    else if (d.flags & PVB_GRID_TRILINEAR) o = grid_trilinear_eval(d, q);
    else o = grid_eval<false, true>(d, st, q, 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

struct Consts {
    float sph_rad[8], visit_margin[8];
    Consts(const pvb_sdf_desc *descs, int n_sdf) {
        for (int s = 0; s < 8; ++s) {
            if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
            else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
        }
    }
};

static void bounds(const pvb_sdf_desc *descs, int n_sdf, const Consts &k, const float *xforms, int n_cfg, int cfg, f3 p,
                   float (&lb)[8], float (&key)[8]) {
    for (int s = 0; s < 8; ++s) {
        f3 cen = mk3(0.f, 0.f, 0.f);
        if (s < n_sdf) {
            float4 r0, r1, r2;
            load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
            cen = rs_sphere_centre(descs[s], r0, r1, r2);
        }
        lb[s] = rs_sphere_lb(p, cen.x, cen.y, cen.z, k.sph_rad[s]);
        key[s] = rs_bound_key(lb[s], ~7, s);
    }
}

// chunk: points per chunk (>= seg_len: whole segments); unit_order 0 ascending, 1 descending, 2 shuffled by
// shuffle_seed; seeded = 0: lanes do not read the keys at the start of a unit; first >= 0: every point group visits
// link `first` first; lanes_reversed: every lane walks its points from the last to the first.
extern "C" void simclear_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                               int cfg_count, const float *pts, long long n_seg, int seg_len, int chunk,
                               int unit_order, int shuffle_seed, int seeded, int first, int lanes_reversed,
                               uint64_t *keys, long long *n_evals) {
    const Consts k(descs, n_sdf);
    for (long long t = 0; t < (long long)cfg_count * n_seg; ++t) keys[t] = ~0ull;
    const int n_tiles = (cfg_count >> 5) + __builtin_popcount((unsigned)(cfg_count & 31));
    const int per_seg = (seg_len + chunk - 1) / chunk;
    std::vector<std::pair<int, long long>> units;            // (tile, chunk index over all segments)
    for (int t = 0; t < n_tiles; ++t)
        for (long long w = 0; w < n_seg * per_seg; ++w) units.emplace_back(t, w);
    if (unit_order == 1) std::reverse(units.begin(), units.end());
    if (unit_order == 2) std::shuffle(units.begin(), units.end(), std::mt19937(shuffle_seed));
    long long evals = 0;
    for (const auto &u : units) {
        int c0, lc_log2;
        rs_tile(cfg_count, u.first, c0, lc_log2);
        const int LC = 1 << lc_log2, G = 8 << (5 - lc_log2);
        const long long b = u.second / per_seg;
        const int i0 = (int)(u.second - b * per_seg) * chunk;
        const int len = std::min(chunk, seg_len - i0);
        std::vector<uint64_t> seed_key(LC), blk(LC, ~0ull);
        for (int cl = 0; cl < LC; ++cl) seed_key[cl] = seeded ? keys[(size_t)(c0 + cl) * n_seg + b] : ~0ull;
        for (int g = 0; g < G; ++g) {
            std::vector<int> mine;
            for (int j = g; j < len; j += G) mine.push_back(j);
            if (lanes_reversed) std::reverse(mine.begin(), mine.end());
            std::vector<uint64_t> run(LC, ~0ull);
            std::vector<float> rv(LC, PVB_INF);
            for (int j : mine) {
                const long long i = b * seg_len + i0 + j;
                const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
                float lb0[8], key0[8];
                bounds(descs, n_sdf, k, xforms, n_cfg, cfg_begin + c0, p, lb0, key0);
                const int pred = first >= 0 ? first : rs_nearest(key0, n_sdf);   // the point group's first lane
                for (int cl = 0; cl < LC; ++cl) {
                    const int cfg = cfg_begin + c0 + cl;
                    float lb[8], key[8];
                    bounds(descs, n_sdf, k, xforms, n_cfg, cfg, p, lb, key);
                    auto link = [&](const int si, const float thr, float4 &o) -> bool {
                        float4 r0, r1, r2;
                        load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                        const f3 q = composed_xform(r0, r1, r2, p);
                        const float tm = thr + k.visit_margin[si];
                        if (tm < 0.f || composed_aabb_lb2(descs[si], q) > tm * tm) return false;
                        o = eval_link(descs[si], q);
                        ++evals;
                        return true;
                    };
                    float best;
                    f3 bg;
                    int bs;
                    rs_swept_pair(lb, pred, fminf(rv[cl], clearance_key_value(seed_key[cl])), link, best, bg, bs);
                    if (bs >= 0) {
                        const uint64_t key_ = clearance_key(best, (uint32_t)(i0 + j));
                        if (key_ < run[cl]) { run[cl] = key_; rv[cl] = best; }
                    }
                }
            }
            for (int cl = 0; cl < LC; ++cl) blk[cl] = std::min(blk[cl], run[cl]);
        }
        for (int cl = 0; cl < LC; ++cl) {
            uint64_t &dst = keys[(size_t)(c0 + cl) * n_seg + b];
            dst = std::min(dst, blk[cl]);
        }
    }
    *n_evals = evals;
}

// composed_clearance_kernel<kMesh = true, kExt = true>: composed_point for every (configuration, point) pair, its key
// folded into the pair's (configuration, segment) key
extern "C" void simclear_generic(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                                 int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_seg,
                                 int seg_len, float margin_max, uint64_t *keys) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pts = n_seg * seg_len;
#pragma omp parallel for schedule(dynamic, 1)
    for (int c = 0; c < cfg_count; ++c) {
        const int cfg = cfg_begin + c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
        for (long long b = 0; b < n_seg; ++b) {
            uint64_t m = ~0ull;
            for (int ip = 0; ip < seg_len; ++ip) {
                const long long i = b * seg_len + ip;
                const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
                const ComposedOut o = composed_point<true, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                                 (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i, 1,
                                                                 margin_max);
                m = std::min(m, clearance_key(o.val, (uint32_t)ip));
            }
            keys[(size_t)c * n_seg + b] = m;
        }
    }
}

// clearance_finish_kernel<kMesh, kExt = true>: the pair named by each key, evaluated with composed_point
extern "C" void simclear_finish(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                                int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_seg, int seg_len,
                                int mesh, float margin_max, const uint64_t *keys, float *out_val, float *out_grad,
                                int *out_point, int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pts = n_seg * seg_len;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long t = 0; t < (long long)cfg_count * n_seg; ++t) {
        const long long c = t / n_seg, b = t - c * n_seg;
        const int ip = (int)(uint32_t)keys[t];
        const long long i = b * seg_len + ip;
        const int cfg = cfg_begin + (int)c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
        const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        const uint64_t pair = (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i;
        const ComposedOut o = mesh ? composed_point<true, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                                pair, 1, margin_max)
                                   : composed_point<false, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                                 pair, 1, margin_max);
        out_val[t] = o.val;
        out_grad[3 * t] = o.grad.x; out_grad[3 * t + 1] = o.grad.y; out_grad[3 * t + 2] = o.grad.z;
        out_point[t] = ip;
        out_which[t] = o.which;
    }
}

// robot_serial_kernel's per-pair sequence for every (configuration, point): the first visit (link `first`, or the
// configuration's nearest sphere when first < 0) always evaluated, then every other link unless its sphere bound or
// exact AABB bound is strictly above the running minimum; the winner's gradient rotated back.
extern "C" void simclear_serial_pairs(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg,
                                      const float *pts, long long n_pts, int first, float *out_val, float *out_grad,
                                      int *out_which) {
    const Consts k(descs, n_sdf);
#pragma omp parallel for schedule(dynamic, 64)
    for (long long t = 0; t < (long long)n_cfg * n_pts; ++t) {
        const int cfg = (int)(t / n_pts);
        const long long i = t - (long long)cfg * n_pts;
        const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        float lb[8], key[8];
        bounds(descs, n_sdf, k, xforms, n_cfg, cfg, p, lb, key);
        const int pred = first >= 0 ? first : rs_nearest(key, n_sdf);
        float best = PVB_INF;
        f3 bg = mk3(0.f, 0.f, 0.f);
        int bs = -1;
        auto visit = [&](const int si, const bool is_first) {
            float4 r0, r1, r2;
            load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
            const f3 q = composed_xform(r0, r1, r2, p);
            if (!is_first) {
                const float thr = best + k.visit_margin[si];
                if (thr < 0.f || composed_aabb_lb2(descs[si], q) > thr * thr) return;
            }
            const float4 o = eval_link(descs[si], q);
            if (is_first || o.x < best || (o.x == best && si < bs)) { best = o.x; bg = mk3(o.y, o.z, o.w); bs = si; }
        };
        visit(pred, true);
        for (int si = 0; si < 8; ++si)
            if (si != pred && !(lb[si] > best)) visit(si, false);
        float4 r0, r1, r2;
        load_rows(xforms, n_cfg, bs < 0 ? 0 : bs, cfg, r0, r1, r2);
        const f3 go = composed_rotate_back(r0, r1, r2, bg);
        out_val[t] = best;
        out_grad[3 * t] = go.x; out_grad[3 * t + 1] = go.y; out_grad[3 * t + 2] = go.z;
        out_which[t] = bs;
    }
}

// ---- the key encoding
extern "C" void simclear_keys(const float *v, const uint32_t *idx, long long n, uint64_t *out, float *decoded) {
    for (long long t = 0; t < n; ++t) {
        out[t] = clearance_key(v[t], idx[t]);
        decoded[t] = clearance_key_value(out[t]);
    }
}

static inline float as_float(uint32_t u) { return __int_as_float((int)u); }
static inline uint32_t high(float f) { return (uint32_t)(clearance_key(f, 0u) >> 32); }

// Exhaustive checks over every 32-bit pattern; returns the number of violations of
//   [0] order: consecutive floats in value order get strictly increasing high words (-0 and +0 the same one);
//   [1] NaN: every NaN pattern (both signs, every payload) maps to 0xffffffff, and every number below it;
//   [2] decoding: clearance_key_value gives back every number (+0 for -0), and every high word that is not a NaN's
//       decodes to a number whose key has that high word (except the one word of -0).
extern "C" void simclear_check_all_patterns(long long *bad) {
    long long b0 = 0, b1 = 0, b2 = 0;
#pragma omp parallel for reduction(+ : b0, b1, b2) schedule(static)
    for (long long s = 0; s < (1ll << 32); ++s) {
        const uint32_t u = (uint32_t)s;
        const float f = as_float(u);
        const uint32_t h = high(f);
        if (f != f) {
            if (h != 0xffffffffu) ++b1;
        } else {
            if (h == 0xffffffffu) ++b1;
            const float d = clearance_key_value((uint64_t)h << 32);
            if (!(d == f) || __float_as_int(d) == (int)0x80000000u) ++b2;
            // successor in value order: the next pattern up (positive half) or down (negative half)
            if (u < 0x7f800000u && high(as_float(u + 1)) <= h) ++b0;
            if (u > 0x80000000u && u <= 0xff800000u && high(as_float(u - 1)) <= h) ++b0;
            if (u == 0x80000000u && high(as_float(0u)) != h) ++b0;
        }
        // u as a high word
        const float dv = clearance_key_value((uint64_t)u << 32);
        if (dv == dv && u != 0x7fffffffu && high(dv) != u) ++b2;
    }
    bad[0] = b0; bad[1] = b1; bad[2] = b2;
}
