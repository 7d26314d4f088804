// Host build of the ray routines of pvb_device.cuh (pvb_ray_carve, pvb_occupancy_apply) behind a small C interface
// for tests/test_ray_occupancy_cpu.py.
//   simray_carve runs ray_carve_kernel's per-ray body: ray_valid, out_points, then ray_walk writing 2 into marks;
//   simray_walks records every ray's walk in visiting order: idx [n_rays][nx + ny + nz][3], count [n_rays] (0 for an
//   invalid ray), valid [n_rays];
//   simray_apply runs occupancy_apply_kernel's per-voxel body.
// Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static void ray_at(const float *points, const float *origins, long long t, long long per_origin, f3 &o, f3 &p) {
    const float *q = origins + 3 * (t / per_origin), *s = points + 3 * t;
    o = mk3(q[0], q[1], q[2]);
    p = mk3(s[0], s[1], s[2]);
}

extern "C" void simray_carve(const float *points, long long n_rays, long long per_origin, const float *origins,
                             float max_range, float margin, const float *lo, float r, const int *dims, uint8_t *marks,
                             float *out) {
    const float nan = __int_as_float(0x7fc00000);
    const int ny = dims[1], nz = dims[2];
    for (long long t = 0; t < n_rays; ++t) {
        f3 o, p, d;
        float len;
        ray_at(points, origins, t, per_origin, o, p);
        const bool valid = ray_valid(o, p, max_range, d, len);
        out[3 * t] = valid ? p.x : nan; out[3 * t + 1] = valid ? p.y : nan; out[3 * t + 2] = valid ? p.z : nan;
        if (valid)
            ray_walk(o, d, len, margin, lo, r, dims, [&](int ix, int iy, int iz) {
                marks[((long long)ix * ny + iy) * nz + iz] = 2;
            });
    }
}

extern "C" void simray_walks(const float *points, long long n_rays, long long per_origin, const float *origins,
                             float max_range, float margin, const float *lo, float r, const int *dims, int *idx,
                             int *count, uint8_t *valid) {
    const long long cap = (long long)dims[0] + dims[1] + dims[2];
#pragma omp parallel for
    for (long long t = 0; t < n_rays; ++t) {
        f3 o, p, d;
        float len;
        ray_at(points, origins, t, per_origin, o, p);
        valid[t] = ray_valid(o, p, max_range, d, len);
        int *row = idx + 3 * cap * t;
        int k = 0;
        if (valid[t])
            ray_walk(o, d, len, margin, lo, r, dims, [&](int ix, int iy, int iz) {
                row[3 * k] = ix; row[3 * k + 1] = iy; row[3 * k + 2] = iz;
                ++k;
            });
        count[t] = k;
    }
}

extern "C" void simray_apply(uint8_t *marks, int16_t *log_odds, long long n_vox, const int *params) {
    const OccupancyParams p = OccupancyParams{params[0], params[1], params[2], params[3]};
    for (long long c = 0; c < n_vox; ++c) {
        const uint8_t m = marks[c];
        if (m == 0) continue;
        log_odds[c] = (int16_t)occupancy_update(log_odds[c], m == 1, m == 2, p);
        marks[c] = 0;
    }
}
