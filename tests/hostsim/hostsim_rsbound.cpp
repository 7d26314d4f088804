// Host build of the bounding-sphere bound of robot_serial_kernel (rs_link_consts, rs_sphere_centre and rs_sphere_lb of
// pvb_device.cuh) behind a small C interface for tests/test_rs_bound_cpu.py.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

// lb[((c * n_pts) + i) * 8 + s]: the bound of link slot s for configuration c at point i, with the link constants and
// the empty slots (s >= n_sdf: centre 0, radius -inf) as launch_robot_serial and the kernel's staging set them up.
// xforms: [n_sdf * n_cfg][16] row-major, sub-SDF-major like pvb_composed_query.
extern "C" void simrs_sphere_lb(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, const float *pts,
                                long long n_pts, float *lb) {
    for (int c = 0; c < n_cfg; ++c) {
        for (int s = 0; s < 8; ++s) {
            float rad = -PVB_INF, margin = 0.f;
            f3 cen = mk3(0.f, 0.f, 0.f);
            if (s < n_sdf) {
                rs_link_consts(descs[s], rad, margin);
                const float4 *row = xf_rows(xforms, n_cfg, s, c);
                cen = rs_sphere_centre(descs[s], row[0], row[1], row[2]);
            }
            for (long long i = 0; i < n_pts; ++i)
                lb[((size_t)c * n_pts + i) * 8 + s] =
                    rs_sphere_lb(mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]), cen.x, cen.y, cen.z, rad);
        }
    }
}

// the visit's margin per link (rs_link_consts)
extern "C" float simrs_visit_margin(const pvb_sdf_desc *d) {
    float rad, margin;
    rs_link_consts(*d, rad, margin);
    return margin;
}
