// Host build of the trilinear building blocks of pvb_device.cuh (CachedSDF(interpolation="trilinear") in the fused
// composed kernels) behind a small C interface for tests/test_trilinear_composed_cpu.py.  Every loop body is the
// per-thread work of the corresponding kernel, with host pointers in the descriptors.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline f3 point(const float *pts, long long i) { return mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]); }

// grid_trilinear_eval per query: the per-thread work of grid_trilinear_kernel
extern "C" void simtri_grid_trilinear(const pvb_sdf_desc *g, const float *pts, long long n, float *val, float *grad) {
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        const SdfOut o = grid_trilinear_eval(*g, point(pts, i));
        val[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
    }
}

// ComposedSDF for every (configuration, point) pair through composed_consider<kMesh = true, kTri = true>: the loop of
// the composed kernels' trilinear instantiations (visit the sub-SDFs in `order`, composed_xform -> composed_consider,
// rotate the winning gradient back).  xforms: [n_sdf * n_cfg][16] row-major, sub-SDF-major like pvb_composed_query.
extern "C" void simtri_composed(const pvb_sdf_desc *descs, int n_sdf, const unsigned char *order, const float *xforms,
                                int n_cfg, const float *pts, long long n_pts, float *out_val, float *out_grad,
                                int *out_which) {
    NodeStage st; st.smem = nullptr; st.n = 0;
#pragma omp parallel for schedule(dynamic, 64) collapse(2)
    for (int c = 0; c < n_cfg; ++c) {
        for (long long i = 0; i < n_pts; ++i) {
            const f3 p = point(pts, i);
            float best = PVB_INF; f3 bg = mk3(0.f, 0.f, 0.f); int bs = -1;
            for (int si = 0; si < n_sdf; ++si) {
                const int s = order ? order[si] : si;
                const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + c) * 16);
                const uint64_t idx = ((uint64_t)c * (uint64_t)n_pts + (uint64_t)i) * (uint64_t)n_sdf + (uint64_t)s;
                composed_consider<true, true>(descs[s], st, s, composed_xform(row[0], row[1], row[2], p),
                                              PVB_MESH_DEFAULT, idx, best, bg, bs);
            }
            const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)max(bs, 0) * n_cfg + c) * 16);
            const f3 go = composed_rotate_back(row[0], row[1], row[2], bg);
            const long long o = (long long)c * n_pts + i;
            out_val[o] = best; out_grad[3 * o] = go.x; out_grad[3 * o + 1] = go.y; out_grad[3 * o + 2] = go.z;
            if (out_which) out_which[o] = bs;
        }
    }
}
