// Host build of the depth-image routines of pvb_device.cuh (pvb_depth_points, pvb_depth_carve) behind a small C
// interface for tests/test_depth_occupancy_cpu.py.
//   simdepth_points runs depth_valid and depth_point for every pixel, as depth_points_kernel does;
//   simdepth_carve runs depth_voxel_centre and depth_says_free for every voxel and view, as depth_carve_kernel does
//   (0 at the first view that says free, 2 when none does).
// The view parameters are the entry points' HOST arrays: intrinsics [V][4], transform rows [V][12].
// Test infrastructure only.
#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

static void rows_of(const float *m, float4 &r0, float4 &r1, float4 &r2) {
    r0 = make_float4(m[0], m[1], m[2], m[3]);
    r1 = make_float4(m[4], m[5], m[6], m[7]);
    r2 = make_float4(m[8], m[9], m[10], m[11]);
}

extern "C" void simdepth_points(const float *depth, int V, int H, int W, const float *intrinsics,
                                const float *cam_to_world, float max_depth, float *out) {
    const float nan = __int_as_float(0x7fc00000);
    for (int v = 0; v < V; ++v) {
        const float *k = intrinsics + 4 * v;
        const float4 cam = make_float4(k[0], k[1], k[2], k[3]);
        float4 r0, r1, r2;
        rows_of(cam_to_world + 12 * v, r0, r1, r2);
#pragma omp parallel for
        for (int i = 0; i < H; ++i)
            for (int j = 0; j < W; ++j) {
                const long long t = ((long long)v * H + i) * W + j;
                f3 p = mk3(nan, nan, nan);
                if (depth_valid(depth[t], max_depth)) p = depth_point(i, j, depth[t], cam, r0, r1, r2);
                out[3 * t] = p.x; out[3 * t + 1] = p.y; out[3 * t + 2] = p.z;
            }
    }
}

extern "C" void simdepth_carve(const float *depth, int V, int H, int W, const float *intrinsics,
                               const float *world_to_cam, float max_depth, float margin, const float *lo, float r,
                               const int *dims, unsigned char *out) {
    const int nx = dims[0], ny = dims[1], nz = dims[2];
    const long long hw = (long long)H * W;
#pragma omp parallel for
    for (int ix = 0; ix < nx; ++ix)
        for (int iy = 0; iy < ny; ++iy)
            for (int iz = 0; iz < nz; ++iz) {
                const f3 c = depth_voxel_centre(lo, r, ix, iy, iz);
                unsigned char state = 2;
                for (int v = 0; v < V; ++v) {
                    const float *k = intrinsics + 4 * v;
                    float4 r0, r1, r2;
                    rows_of(world_to_cam + 12 * v, r0, r1, r2);
                    if (depth_says_free(depth + v * hw, H, W, make_float4(k[0], k[1], k[2], k[3]), r0, r1, r2, c,
                                        max_depth, margin)) {
                        state = 0;
                        break;
                    }
                }
                out[((long long)ix * ny + iy) * nz + iz] = state;
            }
}
