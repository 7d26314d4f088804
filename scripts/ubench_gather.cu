// Micro-benchmark: random 16-byte gathers from an L2-resident table (the CachedSDF / RobotSDF access pattern).
// Compares LDG.128, cp.async (LDGSTS) -> smem, and texture fetches.  Tuning aid only.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__global__ void k_ldg(const float4* __restrict__ tab, const int* __restrict__ idx, long long n, float4* __restrict__ out) {
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        out[i] = __ldg(tab + idx[i]);
    }
}

__global__ void k_ldg4(const float4* __restrict__ tab, const int4* __restrict__ idx4, long long n4, float4* __restrict__ out) {
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        int4 k = idx4[i];
        float4 a = __ldg(tab + k.x), b = __ldg(tab + k.y), c = __ldg(tab + k.z), d = __ldg(tab + k.w);
        out[4 * i] = a; out[4 * i + 1] = b; out[4 * i + 2] = c; out[4 * i + 3] = d;
    }
}

__global__ void k_ldgsts(const float4* __restrict__ tab, const int* __restrict__ idx, long long n, float4* __restrict__ out) {
    __shared__ float4 buf[256];
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        unsigned s = (unsigned)__cvta_generic_to_shared(&buf[threadIdx.x]);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(tab + idx[i]));
        asm volatile("cp.async.commit_group;");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        out[i] = buf[threadIdx.x];
    }
}

__global__ void k_ldgsts4(const float4* __restrict__ tab, const int4* __restrict__ idx4, long long n4, float4* __restrict__ out) {
    __shared__ float4 buf[4][256];
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        int4 k = idx4[i];
        const int kk[4] = {k.x, k.y, k.z, k.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            unsigned s = (unsigned)__cvta_generic_to_shared(&buf[u][threadIdx.x]);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(tab + kk[u]));
        }
        asm volatile("cp.async.commit_group;");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int u = 0; u < 4; ++u) out[4 * i + u] = buf[u][threadIdx.x];
    }
}

__global__ void k_tex(cudaTextureObject_t tex, const int* __restrict__ idx, long long n, float4* __restrict__ out) {
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        out[i] = tex1Dfetch<float4>(tex, idx[i]);
    }
}

__global__ void k_tex4(cudaTextureObject_t tex, const int4* __restrict__ idx4, long long n4, float4* __restrict__ out) {
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        int4 k = idx4[i];
        float4 a = tex1Dfetch<float4>(tex, k.x), b = tex1Dfetch<float4>(tex, k.y), c = tex1Dfetch<float4>(tex, k.z), d = tex1Dfetch<float4>(tex, k.w);
        out[4 * i] = a; out[4 * i + 1] = b; out[4 * i + 2] = c; out[4 * i + 3] = d;
    }
}

// write-only and read-only streaming baselines
__global__ void k_write(long long n, float4* __restrict__ out) {
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = make_float4(1, 2, 3, 4);
}

template <typename F> float timeit(F f, int iters = 20) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    for (int i = 0; i < 3; ++i) f();
    cudaEventRecord(a);
    for (int i = 0; i < iters; ++i) f();
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    CK(cudaGetLastError());
    return ms / iters;
}

int main(int argc, char** argv) {
    const long long n = 10000000;
    const int nvox = argc > 1 ? atoi(argv[1]) : 380952;
    std::vector<int> h(n);
    srand(1);
    for (long long i = 0; i < n; ++i) h[i] = (int)(((long long)rand() * 32768 + rand()) % nvox);
    float4* tab; int* idx; float4* out;
    CK(cudaMalloc(&tab, sizeof(float4) * (size_t)nvox)); CK(cudaMemset(tab, 0, sizeof(float4) * (size_t)nvox));
    CK(cudaMalloc(&idx, sizeof(int) * n)); CK(cudaMemcpy(idx, h.data(), sizeof(int) * n, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&out, sizeof(float4) * n));
    cudaResourceDesc rd = {}; rd.resType = cudaResourceTypeLinear; rd.res.linear.devPtr = tab;
    rd.res.linear.desc = cudaCreateChannelDesc<float4>(); rd.res.linear.sizeInBytes = sizeof(float4) * (size_t)nvox;
    cudaTextureDesc td = {}; td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex; CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));
    const int blocks = 132 * 8, thr = 256;   // 8 blocks per SM of an H100 SXM
    printf("table %d voxels (%.1f MB), %lld gathers, out 160 MB\n", nvox, nvox * 16 / 1e6, n);
    printf("write-only 160MB        : %.1f us\n", 1e3 * timeit([&] { k_write<<<blocks, thr>>>(n, out); }));
    printf("LDG.128 1/thread        : %.1f us\n", 1e3 * timeit([&] { k_ldg<<<blocks, thr>>>(tab, idx, n, out); }));
    printf("LDG.128 4/thread        : %.1f us\n", 1e3 * timeit([&] { k_ldg4<<<blocks, thr>>>(tab, (const int4*)idx, n / 4, out); }));
    printf("LDGSTS.128 1/thread     : %.1f us\n", 1e3 * timeit([&] { k_ldgsts<<<blocks, thr>>>(tab, idx, n, out); }));
    printf("LDGSTS.128 4/thread     : %.1f us\n", 1e3 * timeit([&] { k_ldgsts4<<<blocks, thr>>>(tab, (const int4*)idx, n / 4, out); }));
    printf("tex1Dfetch float4 1/thr : %.1f us\n", 1e3 * timeit([&] { k_tex<<<blocks, thr>>>(tex, idx, n, out); }));
    printf("tex1Dfetch float4 4/thr : %.1f us\n", 1e3 * timeit([&] { k_tex4<<<blocks, thr>>>(tex, (const int4*)idx, n / 4, out); }));
    return 0;
}
