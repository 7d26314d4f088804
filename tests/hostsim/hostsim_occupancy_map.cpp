// Host build of the occupancy-map routines of pvb_device.cuh (pvb_depth_integrate) behind a small C interface for
// tests/test_occupancy_map_cpu.py.
//   simocc_update runs occupancy_update on n (L, observation) pairs, the observation in depth_occupancy's encoding
//   (1 hit, 0 free, 2 nothing);
//   simocc_integrate runs depth_integrate_kernel's per-voxel body: the hit byte, else depth_voxel_centre and
//   depth_says_free up to the first free view, then occupancy_update, and clears the hit byte.
// params is the entry point's HOST {hit, miss, clamp_lo, clamp_hi}.  Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static OccupancyParams params_of(const int *p) { return OccupancyParams{p[0], p[1], p[2], p[3]}; }

extern "C" void simocc_update(const int16_t *L, const uint8_t *obs, long long n, const int *params, int16_t *out) {
    const OccupancyParams p = params_of(params);
    for (long long i = 0; i < n; ++i) out[i] = (int16_t)occupancy_update(L[i], obs[i] == 1, obs[i] == 0, p);
}

extern "C" void simocc_integrate(const float *depth, int V, int H, int W, const float *intrinsics,
                                 const float *world_to_cam, float max_depth, float margin, const float *lo, float r,
                                 const int *dims, uint8_t *hits, int16_t *log_odds, const int *params) {
    const OccupancyParams p = params_of(params);
    const int nx = dims[0], ny = dims[1], nz = dims[2];
    const long long hw = (long long)H * W;
#pragma omp parallel for
    for (int ix = 0; ix < nx; ++ix)
        for (int iy = 0; iy < ny; ++iy)
            for (int iz = 0; iz < nz; ++iz) {
                const long long c = ((long long)ix * ny + iy) * nz + iz;
                const bool hit = hits[c] != 0;
                bool free = false;
                if (!hit) {
                    const f3 x = depth_voxel_centre(lo, r, ix, iy, iz);
                    for (int v = 0; v < V && !free; ++v) {
                        const float *k = intrinsics + 4 * v, *m = world_to_cam + 12 * v;
                        free = depth_says_free(depth + v * hw, H, W, make_float4(k[0], k[1], k[2], k[3]),
                                               make_float4(m[0], m[1], m[2], m[3]), make_float4(m[4], m[5], m[6], m[7]),
                                               make_float4(m[8], m[9], m[10], m[11]), x, max_depth, margin);
                    }
                }
                if (hit || free) log_odds[c] = (int16_t)occupancy_update(log_odds[c], hit, free, p);
                if (hit) hits[c] = 0;
            }
}
