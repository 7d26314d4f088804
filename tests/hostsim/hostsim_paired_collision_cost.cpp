// Host build of the paired collision-cost query of pvb_device.cuh (ComposedSDF.paired_collision_cost /
// pvb_composed_query_paired_collision_cost) behind a small C interface for tests/test_paired_collision_cost_cpu.py.
//   simpcc_fused follows robot_paired_collision_cost_kernel unit by unit: warp units (configuration, segment, chunk)
//   numbered chunk-major and run in a chosen order; a unit's 32 lanes take the chunk's points step by step, a step is
//   skipped when no lane has a sphere bound below the margin, otherwise every lane runs rs_swept_pair on its own point
//   with bp = margin; the contributing lanes then add collision_cost_term into accumulator lane & 7 in four ordered
//   sub-steps (lanes 8r .. 8r + 7 in sub-step r); the 8 accumulators of a unit are added in order in fp64 into an fp32
//   partial, and the partials of a segment in order in fp64 (collision_cost_finish_kernel).
//   Every pair the sequence evaluates is reported with its (value, gradient, sub-SDF), as simcc_fused does.
// Test infrastructure only.
#include <algorithm>
#include <random>
#include <vector>

// The link visits (lookups included) and sphere bounds are the kernels' own: rs_link_visit, rs_link_eval and
// rs_point_bounds of pvb_device.cuh.
#include "hostsim_robot.h"

// pts [cfg_count][n_seg][seg_len][3]: configuration cfg_begin + c's own points are pts[c].  chunk: points per chunk
// (0: collision_cost_chunk(seg_len), the kernel's rule); unit_order 0 ascending, 1 descending, 2 shuffled by
// shuffle_seed; first >= 0: every lane visits link `first` first (else its own nearest sphere).
// Outputs: cost [cfg_count * n_seg], twist [cfg_count * n_seg * n_sdf * 6]; per pair (c * n_seg * seg_len + point):
// visited (rs_swept_pair ran), pair_val / pair_grad / pair_which (bs >= 0; which = -1 otherwise); *n_evals: lookups.
extern "C" void simpcc_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                             int cfg_count, const float *pts, long long n_seg, int seg_len, float margin, int chunk,
                             int unit_order, int shuffle_seed, int first, float *out_cost, float *out_twist,
                             unsigned char *visited, float *pair_val, float *pair_grad, int *pair_which,
                             long long *n_evals) {
    const RsConsts links(descs, n_sdf);
    const int E = 1 + 6 * n_sdf;
    constexpr int kLanes = 32, kAcc = 8;
    if (chunk <= 0) chunk = (int)collision_cost_chunk(seg_len);
    const int cps = seg_len > 0 ? (seg_len + chunk - 1) / chunk : 0;
    const long long pairs = (long long)cfg_count * n_seg;
    std::vector<float> partial((size_t)pairs * cps * E, 0.f);
    std::vector<long long> units;
    for (long long w = 0; w < pairs * cps; ++w) units.push_back(w);
    if (unit_order == 1) std::reverse(units.begin(), units.end());
    if (unit_order == 2) std::shuffle(units.begin(), units.end(), std::mt19937(shuffle_seed));
    for (long long t = 0; t < pairs * seg_len; ++t) { visited[t] = 0; pair_which[t] = -1; }
    long long evals = 0;
    const float m = margin;
    for (const long long w : units) {
        const long long kc = w / pairs, cb = w - kc * pairs;
        const int cfg = cfg_begin + (int)(cb / n_seg);
        const int i0 = (int)kc * chunk, len = std::min(chunk, seg_len - i0);
        const long long pt0 = cb * seg_len + i0;
        // the unit's staging: sphere centres of its one configuration
        float4 sph[6];
        rs_centres(descs, n_sdf, xforms, n_cfg, cfg, sph);
        std::vector<float> acc((size_t)E * kAcc, 0.f);              // acc[e][lane & 7]
        for (int j0 = 0; j0 < len; j0 += kLanes) {
            f3 p[kLanes];
            float lb[kLanes][8], key[kLanes][8];
            bool any = false;
            for (int l = 0; l < kLanes; ++l) {
                const bool on = j0 + l < len;
                const long long i = pt0 + j0 + l;
                p[l] = on ? mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]) : mk3(0.f, 0.f, 0.f);
                rs_point_bounds(sph, links.sph_rad, p[l], ~7, 0xffu, lb[l], key[l]);
                any |= on && collision_cost_near(lb[l], m);
            }
            if (!any) continue;                                     // the whole warp skips the step
            float best[kLanes];
            f3 bg[kLanes];
            int bs[kLanes];
            for (int l = 0; l < kLanes; ++l) {
                const bool on = j0 + l < len;
                auto link = [&](const int si, const float thr, float4 &o) -> bool {
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                    if (!rs_link_visit<true>(descs[si], links.visit_margin[si], r0, r1, r2, p[l], thr, o)) return false;
                    evals += on;
                    return true;
                };
                rs_swept_pair(lb[l], first >= 0 ? first : rs_nearest(key[l], n_sdf), on ? m : -PVB_INF, link, best[l],
                              bg[l], bs[l]);
                if (!on) { bs[l] = -1; continue; }
                const long long pr = pt0 + j0 + l;
                visited[pr] = 1;
                if (bs[l] < 0) continue;
                float4 r0, r1, r2;
                load_rows(xforms, n_cfg, bs[l], cfg, r0, r1, r2);
                const f3 g = composed_rotate_back(r0, r1, r2, bg[l]);
                pair_val[pr] = best[l];
                pair_grad[3 * pr] = g.x; pair_grad[3 * pr + 1] = g.y; pair_grad[3 * pr + 2] = g.z;
                pair_which[pr] = bs[l];
            }
            // four ordered sub-steps: accumulator w takes lanes w, w + 8, w + 16, w + 24 in turn
            for (int r = 0; r < kLanes / kAcc; ++r)
                for (int l = kAcc * r; l < kAcc * (r + 1); ++l) {
                    if (bs[l] < 0 || !(best[l] < m)) continue;
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, bs[l], cfg, r0, r1, r2);
                    const CollisionTerm t = collision_cost_term(m, best[l], composed_rotate_back(r0, r1, r2, bg[l]),
                                                                p[l]);
                    float *a = &acc[l & (kAcc - 1)];
                    a[0] += t.cost;
                    for (int k = 0; k < 6; ++k) a[(size_t)(1 + 6 * bs[l] + k) * kAcc] += t.tw[k];
                }
        }
        for (int e = 0; e < E; ++e) {
            double s = 0.0;
            for (int v = 0; v < kAcc; ++v) s += (double)acc[(size_t)e * kAcc + v];
            partial[((size_t)cb * cps + kc) * E + e] = (float)s;
        }
    }
    for (long long r = 0; r < pairs; ++r)
        for (int e = 0; e < E; ++e) {
            double s = 0.0;
            for (int kc = 0; kc < cps; ++kc) s += (double)partial[((size_t)r * cps + kc) * E + e];
            if (e == 0) out_cost[r] = (float)s;
            else out_twist[(size_t)r * (E - 1) + e - 1] = (float)s;
        }
    *n_evals = evals;
}
