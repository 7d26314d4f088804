// What the host builds of the robot-family kernels (hostsim_swept / _clearance / _paired_clearance / _self_clearance /
// _collision_cost / _paired_collision_cost / _self_collision_cost) share: the transform rows of one (sub-SDF,
// configuration) through the device header's xf_rows, the link constants of the kernels' pack, and a configuration's
// staged row of sphere centres through rs_centre_slot -- the helper robot_paired_clearance_kernel and
// robot_self_collision_cost_kernel stage with; the other robot kernels restate the same rule inline.  The link visit
// and the bound pass are the device header's rs_link_visit / rs_link_eval / rs_point_bounds.  Test infrastructure only.
#pragma once
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static inline void load_rows(const float *xforms, int n_cfg, int s, int cfg, float4 &r0, float4 &r1, float4 &r2) {
    const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
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

// configuration cfg's row of sphere centres as the kernels stage it: its rows, then rs_centre_slot for the 8 slots
static inline void rs_centres(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg,
                              float4 (&sph)[6]) {
    float4 xf[3 * 8];
    for (int s = 0; s < n_sdf; ++s) load_rows(xforms, n_cfg, s, cfg, xf[3 * s], xf[3 * s + 1], xf[3 * s + 2]);
    for (int s = 0; s < 8; ++s) rs_centre_slot(descs, s, n_sdf, xf, sph);
}
