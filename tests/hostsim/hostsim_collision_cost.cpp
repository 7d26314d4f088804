// Host build of the collision-cost query of pvb_device.cuh (ComposedSDF.collision_cost /
// pvb_composed_query_collision_cost) behind a small C interface for tests/test_collision_cost_cpu.py.
//   simcc_fused follows robot_collision_cost_kernel unit by unit: work units (configuration tile, segment, chunk) in a
//   chosen order; in a unit, accumulator w takes the chunk's points w, w + n_acc, ... in order; a point is skipped when
//   no lane of the tile has a sphere bound below the margin, otherwise every lane runs rs_swept_pair with bp = margin
//   and a contributing pair adds collision_cost_term to its accumulator; the accumulators of a unit are added in order
//   in fp64 into an fp32 partial, and the partials of a segment in order in fp64 (collision_cost_finish_kernel).
//   Every pair the sequence evaluates is reported with its (value, gradient, sub-SDF), so that the tests can compare
//   them with the per-pair query and check that no pair below the margin is skipped.
// Test infrastructure only.
#include <algorithm>
#include <array>
#include <random>
#include <vector>

#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline void load_rows(const float *xforms, int n_cfg, int s, int cfg, float4 &r0, float4 &r1, float4 &r2) {
    const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
    r0 = row[0]; r1 = row[1]; r2 = row[2];
}

// robot_collision_cost_kernel's evaluation of a link: primitive, trilinear or nearest-voxel lookup (the arithmetic of
// robot_primitive / robot_lookup_trilinear / robot_lookup)
static inline float4 eval_link(const pvb_sdf_desc &d, f3 q) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    SdfOut o;
    if (d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
    else if (d.flags & PVB_GRID_TRILINEAR) o = grid_trilinear_eval(d, q);
    else o = grid_eval<false, true>(d, st, q, 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

// chunk: points per chunk (0: collision_cost_chunk(seg_len), the kernel's rule); n_acc: accumulators per unit (8 in the
// kernel); lanes: configurations per tile (32 in the kernel); unit_order 0 ascending, 1 descending, 2 shuffled by
// shuffle_seed; first >= 0: every lane visits link `first` first.
// Outputs: cost [cfg_count * n_seg], twist [cfg_count * n_seg * n_sdf * 6]; per pair (c * n_seg * seg_len + point):
// visited (rs_swept_pair ran), pair_val / pair_grad / pair_which (bs >= 0; which = -1 otherwise); *n_evals: lookups.
extern "C" void simcc_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                            int cfg_count, const float *pts, long long n_seg, int seg_len, float margin, int chunk,
                            int n_acc, int lanes, int unit_order, int shuffle_seed, int first, float *out_cost,
                            float *out_twist, unsigned char *visited, float *pair_val, float *pair_grad,
                            int *pair_which, long long *n_evals) {
    float sph_rad[8], visit_margin[8];
    for (int s = 0; s < 8; ++s) {
        if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
        else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
    }
    const int E = 1 + 6 * n_sdf;
    if (chunk <= 0) chunk = (int)collision_cost_chunk(seg_len);
    const int cps = seg_len > 0 ? (seg_len + chunk - 1) / chunk : 0;
    const long long n_pts = n_seg * seg_len;
    std::vector<float> partial((size_t)cfg_count * n_seg * cps * E, 0.f);
    const int n_tiles = (cfg_count + lanes - 1) / lanes;
    std::vector<long long> units;
    for (long long u = 0; u < (long long)n_tiles * n_seg * cps; ++u) units.push_back(u);
    if (unit_order == 1) std::reverse(units.begin(), units.end());
    if (unit_order == 2) std::shuffle(units.begin(), units.end(), std::mt19937(shuffle_seed));
    for (long long t = 0; t < (long long)cfg_count * n_pts; ++t) { visited[t] = 0; pair_which[t] = -1; }
    long long evals = 0;
    const float m = margin;
    for (const long long u : units) {
        const long long sc = u / n_tiles;
        const int c0 = (int)(u - sc * n_tiles) * lanes;
        const long long b = sc / cps;
        const int kc = (int)(sc - b * cps);
        const int i0 = kc * chunk, len = std::min(chunk, seg_len - i0);
        const int active = std::min(lanes, cfg_count - c0);
        // acc[w][e][lane]
        std::vector<float> acc((size_t)n_acc * E * lanes, 0.f);
        for (int w = 0; w < n_acc; ++w) {
            for (int j = w; j < len; j += n_acc) {
                const long long i = b * seg_len + i0 + j;
                const f3 p = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
                std::vector<std::array<float, 8>> lbs(lanes), keys(lanes);
                bool any = false;
                for (int cl = 0; cl < lanes; ++cl) {
                    const int cfg = cfg_begin + std::min(c0 + cl, cfg_count - 1);
                    float lb[8], key[8];
                    for (int s = 0; s < 8; ++s) {
                        f3 cen = mk3(0.f, 0.f, 0.f);
                        if (s < n_sdf) {
                            float4 r0, r1, r2;
                            load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
                            cen = rs_sphere_centre(descs[s], r0, r1, r2);
                        }
                        lb[s] = rs_sphere_lb(p, cen.x, cen.y, cen.z, sph_rad[s]);
                        key[s] = rs_bound_key(lb[s], ~7, s);
                        lbs[cl][s] = lb[s]; keys[cl][s] = key[s];
                    }
                    any |= collision_cost_near(lb, m);
                }
                if (!any) continue;                             // the whole warp skips the point
                int pred;
                {
                    float key0[8];
                    for (int s = 0; s < 8; ++s) key0[s] = keys[0][s];
                    pred = first >= 0 ? first : rs_nearest(key0, n_sdf);       // the tile's first lane
                }
                for (int cl = 0; cl < lanes; ++cl) {
                    const int cfg = cfg_begin + std::min(c0 + cl, cfg_count - 1);
                    float lb[8];
                    for (int s = 0; s < 8; ++s) lb[s] = lbs[cl][s];
                    auto link = [&](const int si, const float thr, float4 &o) -> bool {
                        float4 r0, r1, r2;
                        load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                        const f3 q = composed_xform(r0, r1, r2, p);
                        const float tm = thr + visit_margin[si];
                        if (tm < 0.f || composed_aabb_lb2(descs[si], q) > tm * tm) return false;
                        o = eval_link(descs[si], q);
                        evals += cl < active;           // lanes past the slab are not counted

                        return true;
                    };
                    float best;
                    f3 bg;
                    int bs;
                    rs_swept_pair(lb, pred, m, link, best, bg, bs);
                    if (cl >= active) continue;
                    const long long pr = (long long)(c0 + cl) * n_pts + i;
                    visited[pr] = 1;
                    if (bs < 0) continue;
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, bs, cfg, r0, r1, r2);
                    const f3 g = composed_rotate_back(r0, r1, r2, bg);
                    pair_val[pr] = best;
                    pair_grad[3 * pr] = g.x; pair_grad[3 * pr + 1] = g.y; pair_grad[3 * pr + 2] = g.z;
                    pair_which[pr] = bs;
                    if (!(best < m)) continue;
                    const CollisionTerm t = collision_cost_term(m, best, g, p);
                    float *a = &acc[((size_t)w * E) * lanes + cl];
                    a[0] += t.cost;
                    for (int k = 0; k < 6; ++k) a[(size_t)(1 + 6 * bs + k) * lanes] += t.tw[k];
                }
            }
        }
        for (int cl = 0; cl < active; ++cl)
            for (int e = 0; e < E; ++e) {
                double s = 0.0;
                for (int w = 0; w < n_acc; ++w) s += (double)acc[((size_t)w * E + e) * lanes + cl];
                partial[(((size_t)(c0 + cl) * n_seg + b) * cps + kc) * E + e] = (float)s;
            }
    }
    for (long long r = 0; r < (long long)cfg_count * n_seg; ++r)
        for (int e = 0; e < E; ++e) {
            double s = 0.0;
            for (int kc = 0; kc < cps; ++kc) s += (double)partial[((size_t)r * cps + kc) * E + e];
            if (e == 0) out_cost[r] = (float)s;
            else out_twist[(size_t)r * (E - 1) + e - 1] = (float)s;
        }
    *n_evals = evals;
}

extern "C" long long simcc_chunk(long long seg_len) { return collision_cost_chunk(seg_len); }
extern "C" long long simcc_chunks(long long seg_len) { return collision_cost_chunks(seg_len); }
