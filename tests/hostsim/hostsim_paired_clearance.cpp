// Host build of the paired clearance query of pvb_device.cuh (ComposedSDF.paired_clearance /
// pvb_composed_query_paired_clearance) behind a small C interface for tests/test_paired_clearance_cpu.py.
//   simpcl_fused follows robot_paired_clearance_kernel unit by unit: work units (configuration, segment, chunk)
//   numbered chunk-major and run in a chosen order; each unit reads its seed from the keys left by earlier units, its
//   lanes take the chunk's points step by step and run rs_swept_pair against min(running value, seed), optionally with
//   the per-step warp minimum of the running values, and the unit's key minimum is folded into the keys.
//   simpcl_generic is composed_paired_clearance_kernel's per-pair work, simpcl_finish the per-(configuration,
//   segment) work of paired_clearance_finish_kernel.
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

// the kernel's evaluation of a link: primitive, trilinear or nearest-voxel lookup (the same arithmetic as
// robot_primitive / robot_lookup_trilinear / robot_lookup)
static inline float4 eval_link(const pvb_sdf_desc &d, f3 q) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    SdfOut o;
    if (d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
    else if (d.flags & PVB_GRID_TRILINEAR) o = grid_trilinear_eval(d, q);
    else o = grid_eval<false, true>(d, st, q, 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

// chunk: points per unit (>= seg_len: whole segments); lanes: threads per unit (32: a warp, 256: a block); share: the
// running value is the minimum over each warp of the unit after every step; unit_order 0 ascending, 1 descending, 2
// shuffled by shuffle_seed; seeded = 0: units do not read the keys when they start; first >= 0: every lane visits link
// `first` first (else its own nearest sphere); steps_reversed: a unit walks its steps from the last to the first.
extern "C" void simpcl_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                             int cfg_count, const float *pts, long long n_seg, int seg_len, int chunk, int lanes,
                             int share, int unit_order, int shuffle_seed, int seeded, int first, int steps_reversed,
                             uint64_t *keys, long long *n_evals) {
    float sph_rad[8], visit_margin[8];
    for (int s = 0; s < 8; ++s) {
        if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
        else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
    }
    const long long pairs = (long long)cfg_count * n_seg;
    for (long long t = 0; t < pairs; ++t) keys[t] = ~0ull;
    const int per_seg = (seg_len + chunk - 1) / chunk;
    std::vector<long long> units;
    for (long long w = 0; w < pairs * per_seg; ++w) units.push_back(w);
    if (unit_order == 1) std::reverse(units.begin(), units.end());
    if (unit_order == 2) std::shuffle(units.begin(), units.end(), std::mt19937(shuffle_seed));
    long long evals = 0;
    for (const long long w : units) {
        const long long k = w / pairs, cb = w - k * pairs;
        const int cfg = cfg_begin + (int)(cb / n_seg);
        const int i0 = (int)k * chunk;
        const int len = std::min(chunk, seg_len - i0);
        const long long pt0 = cb * seg_len + i0;
        // the unit's staging: sphere centres of its one configuration
        f3 cen[8];
        for (int s = 0; s < 8; ++s) {
            cen[s] = mk3(0.f, 0.f, 0.f);
            if (s < n_sdf) {
                float4 r0, r1, r2;
                load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
                cen[s] = rs_sphere_centre(descs[s], r0, r1, r2);
            }
        }
        const uint64_t seed_key = seeded ? keys[cb] : ~0ull;
        const float seed = clearance_key_value(seed_key);
        std::vector<uint64_t> run(lanes, ~0ull);
        std::vector<float> rv(lanes, PVB_INF);
        std::vector<int> steps;
        for (int j0 = 0; j0 < len; j0 += lanes) steps.push_back(j0);
        if (steps_reversed) std::reverse(steps.begin(), steps.end());
        for (const int j0 : steps) {
            for (int l = 0; l < lanes && j0 + l < len; ++l) {
                const int j = j0 + l;
                const long long i = pt0 + j;
                const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
                float lb[8], key[8];
                for (int s = 0; s < 8; ++s) {
                    lb[s] = rs_sphere_lb(p, cen[s].x, cen[s].y, cen[s].z, sph_rad[s]);
                    key[s] = rs_bound_key(lb[s], ~7, s);
                }
                auto link = [&](const int si, const float thr, float4 &o) -> bool {
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                    const f3 q = composed_xform(r0, r1, r2, p);
                    const float tm = thr + visit_margin[si];
                    if (tm < 0.f || composed_aabb_lb2(descs[si], q) > tm * tm) return false;
                    o = eval_link(descs[si], q);
                    ++evals;
                    return true;
                };
                float best;
                f3 bg;
                int bs;
                rs_swept_pair(lb, first >= 0 ? first : rs_nearest(key, n_sdf), fminf(rv[l], seed), link, best, bg, bs);
                if (bs >= 0) {
                    const uint64_t kk = clearance_key(best, (uint32_t)(i0 + j));
                    if (kk < run[l]) { run[l] = kk; rv[l] = best; }
                }
            }
            if (share)
                for (int w0 = 0; w0 < lanes; w0 += 32) {
                    float m = PVB_INF;
                    for (int l = w0; l < w0 + 32; ++l) m = fminf(m, rv[l]);
                    for (int l = w0; l < w0 + 32; ++l) rv[l] = m;
                }
        }
        uint64_t m = ~0ull;
        for (int l = 0; l < lanes; ++l) m = std::min(m, run[l]);
        keys[cb] = std::min(keys[cb], m);
    }
    *n_evals = evals;
}

// composed_paired_clearance_kernel<kMesh = true, kExt = true>: composed_point for every (configuration,
// own point) pair with the jitter index of the per-configuration query, its key folded into the (configuration,
// segment) key
extern "C" void simpcl_generic(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                               int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_seg, int seg_len,
                               float margin_max, uint64_t *keys) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pts = n_seg * seg_len;
#pragma omp parallel for schedule(dynamic, 1)
    for (int c = 0; c < cfg_count; ++c) {
        const int cfg = cfg_begin + c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
        for (long long b = 0; b < n_seg; ++b) {
            uint64_t m = ~0ull;
            for (int ip = 0; ip < seg_len; ++ip) {
                const long long i = b * seg_len + ip, t = (long long)c * n_pts + i;
                const f3 p = mk3(pts[3 * t], pts[3 * t + 1], pts[3 * t + 2]);
                const ComposedOut o = composed_point<true, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                                 (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i, 1,
                                                                 margin_max);
                m = std::min(m, clearance_key(o.val, (uint32_t)ip));
            }
            keys[(size_t)c * n_seg + b] = m;
        }
    }
}

// paired_clearance_finish_kernel<kMesh, kExt = true>: the pair named by each key, evaluated with
// composed_point at configuration c's own point
extern "C" void simpcl_finish(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                              int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_seg, int seg_len,
                              int mesh, float margin_max, const uint64_t *keys, float *out_val, float *out_grad,
                              int *out_point, int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pts = n_seg * seg_len;
#pragma omp parallel for schedule(dynamic, 16)
    for (long long t = 0; t < (long long)cfg_count * n_seg; ++t) {
        const long long c = t / n_seg, b = t - c * n_seg;
        const int ip = (int)(uint32_t)keys[t];
        const long long i = b * seg_len + ip, pi = c * n_pts + i;
        const int cfg = cfg_begin + (int)c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { load_rows(xforms, n_cfg, s, cfg, r0, r1, r2); };
        const f3 p = mk3(pts[3 * pi], pts[3 * pi + 1], pts[3 * pi + 2]);
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
