// What the host builds of the robot-family kernels (hostsim_swept / _clearance / _paired_clearance / _self_clearance /
// _collision_cost) share: the transform rows of one (sub-SDF, configuration), the link constants of the kernels' pack
// and a configuration's staged row of sphere centres.  The link visit and the bound pass themselves are the device
// header's rs_link_visit / rs_link_eval / rs_point_bounds.  Test infrastructure only.
#pragma once
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline void load_rows(const float *xforms, int n_cfg, int s, int cfg, float4 &r0, float4 &r1, float4 &r2) {
    const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
    r0 = row[0]; r1 = row[1]; r2 = row[2];
}

// RobotPack::sph_rad / visit_margin as rs_pack fills them: slots beyond n_sdf get radius -inf (a bound of +inf)
struct RsConsts {
    float sph_rad[8], visit_margin[8];
    RsConsts(const pvb_sdf_desc *descs, int n_sdf) {
        for (int s = 0; s < 8; ++s) {
            if (s < n_sdf) rs_link_consts(descs[s], sph_rad[s], visit_margin[s]);
            else { sph_rad[s] = -PVB_INF; visit_margin[s] = 0.f; }
        }
    }
};

// configuration cfg's row of sphere centres as the kernels stage it ({x, y, z} of the 8 links back to back; slots
// beyond n_sdf: centre 0)
static inline void rs_centres(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg,
                              float4 (&sph)[6]) {
    float *c = reinterpret_cast<float *>(sph);
    for (int s = 0; s < 8; ++s) {
        f3 co = mk3(0.f, 0.f, 0.f);
        if (s < n_sdf) {
            float4 r0, r1, r2;
            load_rows(xforms, n_cfg, s, cfg, r0, r1, r2);
            co = rs_sphere_centre(descs[s], r0, r1, r2);
        }
        c[3 * s] = co.x; c[3 * s + 1] = co.y; c[3 * s + 2] = co.z;
    }
}
