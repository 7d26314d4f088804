// Peer-store micro-benchmark: how NVLink write throughput depends on the size of the contiguous segment a warp
// instruction writes.  One process, two GPUs (device 0 stores into device 1's memory through peer access), the access
// pattern of the RobotSDF row flush: 32 result rows far apart, each written front to back in segments of S bytes, 16 B
// per lane.   nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/ubench_peer_store.cu -o /tmp/ubench_peer_store
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>

__global__ void store_kernel(float4 *dst, size_t row_f4, int rows, int seg_f4, size_t segs_per_row, int mode) {
    const size_t n_seg = segs_per_row * rows;
    const int lanes_per_seg = seg_f4;                       // 16 B per lane
    const int segs_per_warp = 32 / lanes_per_seg > 0 ? 32 / lanes_per_seg : 1;
    const size_t warp_id = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const size_t n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    const float4 v = make_float4(1.f, 2.f, 3.f, (float)lane);
    if (lanes_per_seg <= 32) {
        for (size_t s0 = warp_id * segs_per_warp; s0 < n_seg; s0 += n_warps * segs_per_warp) {
            const size_t seg = s0 + lane / lanes_per_seg;
            if (seg >= n_seg) continue;
            const size_t row = seg % rows, k = seg / rows;
            float4 *p = dst + row * row_f4 + k * seg_f4 + lane % lanes_per_seg;
            if (mode == 0) __stcs(p, v); else *p = v;
        }
    } else {                                                // segments longer than one warp instruction: 512 B pieces
        const int pieces = lanes_per_seg / 32;
        for (size_t seg = warp_id; seg < n_seg; seg += n_warps) {
            const size_t row = seg % rows, k = seg / rows;
            for (int j = 0; j < pieces; ++j) {
                float4 *p = dst + row * row_f4 + k * seg_f4 + j * 32 + lane;
                if (mode == 0) __stcs(p, v); else *p = v;
            }
        }
    }
}

int main() {
    int n = 0;
    cudaGetDeviceCount(&n);
    const size_t bytes = 256ull << 20;
    const int rows = 32;
    for (int peer = 0; peer <= (n > 1 ? 1 : 0); ++peer) {
        float4 *dst = nullptr;
        cudaSetDevice(peer);
        cudaMalloc(&dst, bytes);
        cudaSetDevice(0);
        if (peer) cudaDeviceEnablePeerAccess(1, 0);
        cudaEvent_t a, b;
        cudaEventCreate(&a); cudaEventCreate(&b);
        for (int seg_bytes : {16, 32, 64, 96, 128, 256, 512, 2048}) {
            if (seg_bytes == 96) continue;                  // 6 lanes do not divide 32: covered by 64 / 128
            const int seg_f4 = seg_bytes / 16;
            const size_t row_f4 = bytes / 16 / rows;
            const size_t segs_per_row = row_f4 / seg_f4;
            float best = 1e9f;
            for (int it = 0; it < 5; ++it) {
                cudaEventRecord(a);
                store_kernel<<<132 * 8, 256>>>(dst, row_f4, rows, seg_f4, segs_per_row, 0);
                cudaEventRecord(b);
                cudaEventSynchronize(b);
                float ms; cudaEventElapsedTime(&ms, a, b);
                if (it > 0 && ms < best) best = ms;
            }
            printf("{\"dst\": \"%s\", \"segment_bytes\": %d, \"ms\": %.4f, \"GBps\": %.1f}\n", peer ? "peer" : "local", seg_bytes,
                   best, bytes / best / 1e6);
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) printf("{\"error\": \"%s\"}\n", cudaGetErrorString(e));
    }
    return 0;
}
