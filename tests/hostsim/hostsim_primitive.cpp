// Host build of the analytic primitives of pvb_device.cuh (BoxSDF / CylinderSDF / SphereSDF links in the fused composed
// kernels) behind a small C interface for tests/test_primitive_cpu.py.  Every loop body is the per-thread work of the
// corresponding kernel, with host pointers in the descriptors.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline f3 point(const float *pts, long long i) { return mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]); }

// fn: 0 = box_eval, 1 = cylinder_eval, 2 = primitive_eval
extern "C" void simprim_eval(const pvb_sdf_desc *d, int fn, const float *pts, long long n, float *val, float *grad) {
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) {
        const f3 q = point(pts, i);
        const SdfOut o = fn == 0 ? box_eval(*d, q) : (fn == 1 ? cylinder_eval(*d, q) : primitive_eval(*d, q));
        val[i] = o.val; grad[3 * i] = o.grad.x; grad[3 * i + 1] = o.grad.y; grad[3 * i + 2] = o.grad.z;
    }
}

// The squared distance to the descriptor's box as the composed kernels compute it (composed_aabb_lb2)
extern "C" void simprim_aabb_lb2(const pvb_sdf_desc *d, const float *pts, long long n, float *lb2) {
    for (long long i = 0; i < n; ++i) lb2[i] = composed_aabb_lb2(*d, point(pts, i));
}

// robot_serial_kernel's bounding-sphere bound of one link (rs_link_consts, rs_sphere_centre, rs_sphere_lb) under one
// object->link transform (16 floats, row-major) at every point: lb[i] <= value of the link at point i.
extern "C" void simprim_sphere_lb(const pvb_sdf_desc *d, const float *xform, const float *pts, long long n, float *lb,
                                  float *visit_margin) {
    float rad, margin;
    rs_link_consts(*d, rad, margin);
    *visit_margin = margin;
    const float4 *row = reinterpret_cast<const float4 *>(xform);
    const f3 c = rs_sphere_centre(*d, row[0], row[1], row[2]);
    for (long long i = 0; i < n; ++i) lb[i] = rs_sphere_lb(point(pts, i), c.x, c.y, c.z, rad);
}
