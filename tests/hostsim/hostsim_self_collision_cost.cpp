// Host build of the self-collision-cost query of pvb_device.cuh (ComposedSDF.self_collision_cost /
// pvb_composed_query_self_collision_cost) behind a small C interface for tests/test_self_collision_cost_cpu.py.
//   simscc_fused follows robot_self_collision_cost_kernel configuration by configuration, in a chosen order: its
//   sources with a non-empty row in ascending order, their link points posed with W_i in steps of `lanes` points; a
//   step is skipped when no lane has an allowed link whose sphere bound is below the margin, otherwise every lane runs
//   rs_swept_pair with bp = margin (masked links +inf and refused inside the visit), and a contributing pair adds
//   collision_cost_term to its target's slots and subtracts it from its source's, in the lane's fp32 accumulators;
//   the lanes' accumulators are then added in lane order in fp64 and rounded to fp32.
//   Every pair the sequence evaluates is reported with its (value, gradient, sub-SDF) and the posed point, so that
//   the tests can compare them with the per-point query of the allowed sub-composition and check that no pair below
//   the margin is skipped.
// Test infrastructure only.
#include <algorithm>
#include <array>
#include <random>
#include <vector>

// The link visits (lookups included) and sphere bounds are the kernels' own: rs_link_visit, rs_link_eval and
// rs_point_bounds of pvb_device.cuh.
#include "hostsim_robot.h"

// masks[i]: bit j allows (i, j), the diagonal already cleared.  lanes: points per step and accumulators (32 in the
// kernel); cfg_order 0 ascending, 1 descending, 2 shuffled by shuffle_seed; first >= 0: every lane visits link
// `first` first (else its own nearest sphere).
// Outputs: cost [cfg_count], twist [cfg_count * n_sdf * 6]; per (configuration, source, point) pair
// ((c * n_sdf + i) * K + k): visited (rs_swept_pair ran), pair_val / pair_grad / pair_which (bs >= 0; -1 otherwise),
// pair_x (the posed point); *n_evals: lookups.
extern "C" void simscc_fused(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, const float *inv_xforms,
                             int n_cfg, int cfg_begin, int cfg_count, const float *link_pts, int K,
                             const unsigned char *masks, float margin, int lanes, int cfg_order, int shuffle_seed,
                             int first, float *out_cost, float *out_twist, unsigned char *visited, float *pair_val,
                             float *pair_grad, int *pair_which, float *pair_x, long long *n_evals) {
    const RsConsts links(descs, n_sdf);
    const int E = 1 + 6 * n_sdf;
    const float m = margin;
    std::vector<int> order;
    for (int c = 0; c < cfg_count; ++c) order.push_back(c);
    if (cfg_order == 1) std::reverse(order.begin(), order.end());
    if (cfg_order == 2) std::shuffle(order.begin(), order.end(), std::mt19937(shuffle_seed));
    for (long long t = 0; t < (long long)cfg_count * n_sdf * K; ++t) { visited[t] = 0; pair_which[t] = -1; }
    long long evals = 0;
    for (const int c : order) {
        const int cfg = cfg_begin + c;
        float4 sph[6];
        rs_centres(descs, n_sdf, xforms, n_cfg, cfg, sph);
        std::vector<float> acc((size_t)E * lanes, 0.f);              // acc[e][lane]
        for (int i = 0; i < n_sdf; ++i) {
            const unsigned mask = masks[i];
            if (!mask) continue;
            float4 w0, w1, w2;
            load_rows(inv_xforms, n_cfg, i, cfg, w0, w1, w2);
            for (int j0 = 0; j0 < K; j0 += lanes) {
                const int len = std::min(lanes, K - j0);
                std::vector<f3> ps(len);
                std::vector<std::array<float, 8>> lbs(len), keys(len);
                bool any = false;
                for (int l = 0; l < len; ++l) {
                    const float *lp = link_pts + 3 * ((size_t)i * K + j0 + l);
                    ps[l] = composed_xform(w0, w1, w2, mk3(lp[0], lp[1], lp[2]));
                    float lb[8], key[8];
                    rs_point_bounds(sph, links.sph_rad, ps[l], ~7, mask, lb, key);
                    for (int s = 0; s < 8; ++s) { lbs[l][s] = lb[s]; keys[l][s] = key[s]; }
                    any |= collision_cost_near(lb, m);
                }
                if (!any) continue;                                  // the whole warp skips the step
                for (int l = 0; l < len; ++l) {
                    const int k = j0 + l;
                    const f3 p = ps[l];
                    float lb[8], key[8];
                    for (int s = 0; s < 8; ++s) { lb[s] = lbs[l][s]; key[s] = keys[l][s]; }
                    auto link = [&](const int si, const float thr, float4 &o) -> bool {
                        if (!((mask >> si) & 1u)) return false;
                        float4 r0, r1, r2;
                        load_rows(xforms, n_cfg, si, cfg, r0, r1, r2);
                        if (!rs_link_visit<true>(descs[si], links.visit_margin[si], r0, r1, r2, p, thr, o)) return false;
                        ++evals;
                        return true;
                    };
                    float best;
                    f3 bg;
                    int bs;
                    rs_swept_pair(lb, first >= 0 ? first : rs_nearest(key, n_sdf), m, link, best, bg, bs);
                    const long long pr = ((long long)c * n_sdf + i) * K + k;
                    visited[pr] = 1;
                    pair_x[3 * pr] = p.x; pair_x[3 * pr + 1] = p.y; pair_x[3 * pr + 2] = p.z;
                    if (bs < 0) continue;
                    float4 r0, r1, r2;
                    load_rows(xforms, n_cfg, bs, cfg, r0, r1, r2);
                    const f3 g = composed_rotate_back(r0, r1, r2, bg);
                    pair_val[pr] = best;
                    pair_grad[3 * pr] = g.x; pair_grad[3 * pr + 1] = g.y; pair_grad[3 * pr + 2] = g.z;
                    pair_which[pr] = bs;
                    if (!(best < m)) continue;
                    const CollisionTerm t = collision_cost_term(m, best, g, p);
                    acc[l] += t.cost;
                    for (int q = 0; q < 6; ++q) {
                        acc[(size_t)(1 + 6 * bs + q) * lanes + l] += t.tw[q];
                        acc[(size_t)(1 + 6 * i + q) * lanes + l] -= t.tw[q];
                    }
                }
            }
        }
        for (int e = 0; e < E; ++e) {
            double s = 0.0;
            for (int l = 0; l < lanes; ++l) s += (double)acc[(size_t)e * lanes + l];
            if (e == 0) out_cost[c] = (float)s;
            else out_twist[(size_t)c * (E - 1) + e - 1] = (float)s;
        }
    }
    *n_evals = evals;
}

// transform_points_paired_kernel's per-point work with every configuration's W on the same K points: out[c][k] =
// composed_xform(W_c, pts[k])
extern "C" void simscc_pose(const float *w, int n_cfg, const float *pts, int K, float *out) {
    for (int c = 0; c < n_cfg; ++c) {
        const float4 *row = reinterpret_cast<const float4 *>(w + (size_t)c * 16);
        for (int k = 0; k < K; ++k) {
            const f3 q = composed_xform(row[0], row[1], row[2], mk3(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]));
            float *o = out + 3 * ((size_t)c * K + k);
            o[0] = q.x; o[1] = q.y; o[2] = q.z;
        }
    }
}

// collision_cost_term of one pair, for the hand-computed sign test
extern "C" void simscc_term(float m, float d, const float *g, const float *p, float *out) {
    const CollisionTerm t = collision_cost_term(m, d, mk3(g[0], g[1], g[2]), mk3(p[0], p[1], p[2]));
    out[0] = t.cost;
    for (int q = 0; q < 6; ++q) out[1 + q] = t.tw[q];
}
