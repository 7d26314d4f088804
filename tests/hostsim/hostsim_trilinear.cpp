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
