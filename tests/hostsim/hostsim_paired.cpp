// Host build of the paired composed query of pvb_device.cuh (ComposedSDF.paired / pvb_composed_query_paired) behind
// a small C interface for tests/test_paired_cpu.py.  The loop body is the per-thread work of composed_paired_kernel,
// with host pointers in the descriptors.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

// composed_point<kMesh = true, kTri = true> for every pair t in [0, cfg_count * n_pts): configuration cfg_begin + c at
// its own point pts[t].  xforms: [n_sdf * n_cfg][16] row-major, sub-SDF-major like pvb_composed_query.
extern "C" void simpair_composed(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                                 int n_cfg, int cfg_begin, int cfg_count, const float *pts, long long n_pts,
                                 int nearest_first, float margin_max, float *out_val, float *out_grad,
                                 int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pairs = (long long)cfg_count * n_pts;
#pragma omp parallel for schedule(dynamic, 64)
    for (long long t = 0; t < n_pairs; ++t) {
        long long c, i;
        paired_index(t, n_pts, c, i);
        const int cfg = cfg_begin + (int)c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
            const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
            r0 = row[0]; r1 = row[1]; r2 = row[2];
        };
        const f3 p = mk3(pts[3 * t], pts[3 * t + 1], pts[3 * t + 2]);
        const ComposedOut o = composed_point<true, true>(descs, order, n_sdf, load_xf, st, p, PVB_MESH_DEFAULT,
                                                         (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i, nearest_first,
                                                         margin_max);
        out_val[t] = o.val;
        out_grad[3 * t] = o.grad.x; out_grad[3 * t + 1] = o.grad.y; out_grad[3 * t + 2] = o.grad.z;
        out_which[t] = o.which;
    }
}

// pair index -> (configuration, point) and the mesh jitter index of sub-SDF s of that pair, as the kernel forms them
extern "C" void simpair_index(const long long *t, long long n, long long n_pts, int cfg_begin, int n_sdf, int s,
                              long long *c_out, long long *i_out, unsigned long long *jitter_out) {
    for (long long k = 0; k < n; ++k) {
        long long c, i;
        paired_index(t[k], n_pts, c, i);
        c_out[k] = c; i_out[k] = i;
        const int cfg = cfg_begin + (int)c;
        jitter_out[k] = ((uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i) * (uint64_t)n_sdf + (uint64_t)s;
    }
}
