// Host build of the scene queries of pvb_device.cuh (ComposedSDF.scene_clearance / scene_collision_cost,
// pvb_composed_query_scene_clearance / _collision_cost) behind a small C interface for tests/test_scene_cpu.py.
//   simscene_fused follows scene_clearance_kernel and scene_collision_cost_kernel configuration by configuration:
//   every tested source's link points posed with W_i in steps of 32 lanes, lane l taking the points l, l + 32, ...;
//   the scene evaluated with composed_point<false, true> over its descriptors in `order`.  Clearance: the smallest
//   self_clearance_key, then the winning point posed and evaluated again.  Cost: a step skipped when scene_near clears
//   every lane's point, collision_cost_add into the lane's fp32 accumulators, the lanes' sums in lane order in fp64
//   (the twist row rounded once and negated), the sources' costs in source order in fp64.
// Test infrastructure only.
#include <vector>

#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

// scene: n_scene descriptors, their visiting order and scene_xforms [n_scene][16] (one configuration); inv_xforms
// [n_sdf * n_cfg][16]; link_pts [n_sdf][K][3]; links [n_sdf].  Outputs for configurations cfg_begin ..: val, grad
// [3], link, point, cost, twist [n_sdf * 6]; *n_skipped: 32-point steps the cost loop skipped.
extern "C" void simscene_fused(const pvb_sdf_desc *scene, int n_scene, const unsigned char *order,
                               const float *scene_xforms, const float *inv_xforms, int n_sdf, int n_cfg, int cfg_begin,
                               int cfg_count, const float *link_pts, int K, const unsigned char *links, float margin,
                               float *out_val, float *out_grad, int *out_link, int *out_point, float *out_cost,
                               float *out_twist, long long *n_skipped) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
        const float4 *row = xf_rows(scene_xforms, 1, s, 0);
        r0 = row[0]; r1 = row[1]; r2 = row[2];
    };
    auto pose = [&](int i, int cfg, int k) {
        const float4 *w = xf_rows(inv_xforms, n_cfg, i, cfg);
        const float *lp = link_pts + 3 * ((size_t)i * K + k);
        return composed_xform(w[0], w[1], w[2], mk3(lp[0], lp[1], lp[2]));
    };
    auto eval = [&](f3 x) { return composed_point<false, true>(scene, order, n_scene, load_xf, st, x, 0u, 0ull, 0, 0.f); };
    const float m = margin;
    long long skipped = 0;
    for (int c = 0; c < cfg_count; ++c) {
        const int cfg = cfg_begin + c;
        uint64_t best = ~0ull;
        std::vector<double> cost_part(n_sdf, 0.0);
        for (int i = 0; i < n_sdf; ++i) {
            float *row = out_twist + ((size_t)c * n_sdf + i) * 6;
            for (int q = 0; q < 6; ++q) row[q] = 0.f;
            if (!links[i]) continue;
            float acc[kSceneLanes][7] = {};
            for (int j0 = 0; j0 < K; j0 += kSceneLanes) {
                const int len = K - j0 < kSceneLanes ? K - j0 : kSceneLanes;
                bool any = false;
                for (int l = 0; l < len; ++l) any |= scene_near(scene, n_scene, load_xf, pose(i, cfg, j0 + l), m);
                for (int l = 0; l < len; ++l) {
                    const f3 x = pose(i, cfg, j0 + l);
                    const ComposedOut o = eval(x);
                    const uint64_t kk = self_clearance_key(o.val, i, j0 + l);
                    best = kk < best ? kk : best;
                    if (any && o.val < m) collision_cost_add(m, o.val, o.grad, x, &acc[l][0], &acc[l][1], 1);
                }
                skipped += any ? 0 : 1;
            }
            for (int e = 0; e < 7; ++e) {
                double s = 0.0;
                for (int l = 0; l < kSceneLanes; ++l) s += (double)acc[l][e];
                if (e == 0) cost_part[i] = s;
                else row[e - 1] = (float)(0.0 - s);
            }
        }
        double s = 0.0;
        for (int i = 0; i < n_sdf; ++i) s += cost_part[i];
        out_cost[c] = (float)s;
        float val = PVB_INF;
        f3 g = mk3(0.f, 0.f, 0.f);
        int li = -1, pk = -1;
        if (best != ~0ull) {
            li = (int)((uint32_t)best >> 24); pk = (int)((uint32_t)best & 0xffffffu);
            const ComposedOut o = eval(pose(li, cfg, pk));
            val = o.val; g = o.grad;
        }
        out_val[c] = val;
        out_grad[3 * c] = g.x; out_grad[3 * c + 1] = g.y; out_grad[3 * c + 2] = g.z;
        out_link[c] = li; out_point[c] = pk;
    }
    *n_skipped = skipped;
}
