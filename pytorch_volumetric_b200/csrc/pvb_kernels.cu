// pvb_kernels.cu -- sm_90a (H100) kernels and the C ABI of libpvb.so (see include/pvb.h).
//
// No tensor-core work anywhere on this path (there is no dense contraction).  The kernels are
//   grid_lookup_tma / vec4 / scalar   HBM-streaming nearest-voxel lookup (CachedSDF)
//   composed_query / composed_cfgmajor  transform + lookup / tree walk + min over sub-SDFs (ComposedSDF, RobotSDF)
//   sort_hist / sort_scan / sort_scatter  Morton binning of large query batches
//   mesh_query, chamfer_partial / finish  BVH4 tree walks (MeshSDF, chamfer)
//   mesh_sample, sphere, transform_points  small helpers
// Tuning knobs that are build macros or PVB_* environment variables can be swept without editing the source.
#include "pvb_device.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <type_traits>

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";

void pvb_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *pvb_last_error(void) { return g_err; }
extern "C" int pvb_version(void) { return PVB_VERSION; }
extern "C" int pvb_sizeof_sdf_desc(void) { return (int)sizeof(pvb_sdf_desc); }
extern "C" int pvb_sizeof_bvh4_node(void) { return (int)sizeof(pvb_bvh4_node); }

static_assert(sizeof(pvb_bvh4_node) == 128, "BVH4 node must be 128 bytes");
static_assert(sizeof(pvb_sdf_desc) % 8 == 0, "descriptor arrays must keep 8-byte alignment");

#define PVB_CHECK_LAUNCH(name)                                                        \
    do {                                                                              \
        cudaError_t e_ = cudaGetLastError();                                          \
        if (e_ != cudaSuccess) {                                                      \
            pvb_set_error("%s: launch failed: %s", name, cudaGetErrorString(e_));     \
            return PVB_ERR_CUDA;                                                      \
        }                                                                             \
    } while (0)

namespace pvb {

// ------------------------------------------------------------ device info
// Function attributes and device properties are per device: one process may drive several GPUs (CachedSDF /
// ComposedSDF accept any device=), so everything cached here is indexed by the current device.
constexpr int kMaxDevices = 64;
static int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}

static int sm_count() {
    static int n[kMaxDevices] = {0};
    const int dev = current_device();
    if (n[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;   // H100 SXM
        n[dev] = v;
    }
    return n[dev];
}

// Opt-in to > 48 KB of dynamic shared memory for `kernel`, once per (kernel, device).  `slot` is a small per-kernel
// id; returns false when the runtime refuses.
enum { kSlotMesh = 0, kSlotGridTma, kSlotCfgMajor, kSlotCfgMajorMulti, kSlotChamfer, kSlotRobot, kSlotRobotMulti,
       kSlotRobotMc, kSlotRobotWide, kSlotRobotWideMulti, kSlotRobotWideMc, kSlotSerial, kSlotSerialMulti, kSlotSerialMc,
       kSlotSerialExt, kSlotSerialExtMulti, kSlotSerialExtMc, kSlotCfgMajorExt, kSlotCfgMajorExtMulti,
       kSlotCollisionCost, kSlotCollisionCostExt, kSlotCount };
template <typename K>
static bool ensure_smem(K kernel, int slot, int bytes) {
    static unsigned char done[kSlotCount][kMaxDevices] = {{0}};
    const int dev = current_device();
    if (done[slot][dev] == 1) return true;
    const bool ok = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess;
    if (ok) done[slot][dev] = 1;
    return ok;
}

// ------------------------------------------------------------ kernel timing hook (bench.py roofline)
// When enabled (pvb_timing_enable), every query entry point brackets its DOMINANT kernel launch with a pair of CUDA
// events on the caller's stream; pvb_timing_last_ms waits for the stop event and returns the elapsed device time of
// that one launch.  Off by default: two extra event records per call otherwise.
static int g_timing = 0;
static cudaEvent_t g_ev[kMaxDevices][2];
static unsigned char g_ev_ok[kMaxDevices] = {0};
static unsigned char g_ev_set[kMaxDevices] = {0};
static void timing_mark(int which, cudaStream_t stream) {
    if (!g_timing) return;
    const int dev = current_device();
    if (!g_ev_ok[dev]) {
        if (cudaEventCreate(&g_ev[dev][0]) != cudaSuccess || cudaEventCreate(&g_ev[dev][1]) != cudaSuccess) return;
        g_ev_ok[dev] = 1;
    }
    cudaEventRecord(g_ev[dev][which], stream);
    if (which == 1) g_ev_set[dev] = 1;
}

// ------------------------------------------- TMA bulk copy (global -> smem)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

__device__ __forceinline__ void bulk_s2g(void *gdst, const void *ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Stage the first n_stage BVH nodes (BFS prefix = top of the tree) into shared
// memory with one bulk asynchronous copy; every thread then waits on the mbarrier.
__device__ __forceinline__ NodeStage stage_nodes(const void *gnodes, int n_nodes, int n_stage_max,
                                                 unsigned char *smem_raw, uint64_t *bar) {
    NodeStage st;
    const int n = min(n_nodes, n_stage_max);
    st.smem = reinterpret_cast<const float4 *>(smem_raw);
    st.n = n;
    if (n > 0) {
        if (threadIdx.x == 0) mbar_init(bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t bytes = (uint32_t)n * 128u;
            mbar_expect_tx(bar, bytes);
            bulk_g2s(smem_raw, gnodes, bytes, bar);
        }
        mbar_wait(bar, 0);
    }
    return st;
}

__device__ __forceinline__ f3 load_point(const float *__restrict__ pts, long long i) {
    return mk3(__ldg(pts + 3 * i), __ldg(pts + 3 * i + 1), __ldg(pts + 3 * i + 2));
}

// ===================================================== spatial binning of queries
// A random query batch makes every lane of a warp walk a different part of the BVH: the first version of the mesh
// kernel kept few lanes of a warp busy.  Large
// batches are therefore binned into 64^3 Morton-ordered cells over the padded mesh AABB with a counting sort
// (histogram by atomics, single-block scan, scatter) and the tree walk processes them in that order through an
// index permutation; results are written to the original slots, so callers see no reordering.
constexpr int kSortBits = 6;                               // per axis: 64^3 cells (default)
constexpr int kSortBitsMax = 8;                            // 256^3 cells = 64 MB of counters

// Cells per axis for a batch of n queries.  Lanes of a warp are 32 consecutive queries of the binned order: they walk
// the same part of the tree only if a cell is not much larger than the triangles around it, and a cell holds n / cells
// queries in arbitrary order.  PVB_SORT_BITS overrides.
static int sort_bits_for(long long n) {
    static const int forced = [] { const char *e = getenv("PVB_SORT_BITS"); return e ? atoi(e) : 0; }();
    if (forced >= 4 && forced <= kSortBitsMax) return forced;
    // finer cells than 64^3 cost a larger histogram (zeroing + single-block scan) for little gain in coherence
    (void)n;
    return kSortBits;
}
constexpr long long kSortMinPoints = 1 << 15;

__device__ __forceinline__ uint32_t part1by2(uint32_t x) {  // spread the low 10 bits, two zeros between bits
    x &= 0x3ffu;
    x = (x | (x << 16)) & 0x030000ffu;
    x = (x | (x << 8)) & 0x0300f00fu;
    x = (x | (x << 4)) & 0x030c30c3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

struct SortFrame {           // cell = morton(quantise(((M p) - lo) * scale)); M optional (chamfer: first transform)
    float lo[3], scale[3];
    float xf[12];
    int use_xf;
    int bits;                // cells per axis = 1 << bits
};

__device__ __forceinline__ uint32_t sort_cell(const SortFrame &f, f3 p) {
    if (f.use_xf)
        p = mk3(fmaf(f.xf[0], p.x, fmaf(f.xf[1], p.y, fmaf(f.xf[2], p.z, f.xf[3]))),
                fmaf(f.xf[4], p.x, fmaf(f.xf[5], p.y, fmaf(f.xf[6], p.z, f.xf[7]))),
                fmaf(f.xf[8], p.x, fmaf(f.xf[9], p.y, fmaf(f.xf[10], p.z, f.xf[11]))));
    const float m = (float)((1 << f.bits) - 1);
    const uint32_t cx = (uint32_t)fminf(fmaxf((p.x - f.lo[0]) * f.scale[0], 0.f), m);   // NaN -> 0
    const uint32_t cy = (uint32_t)fminf(fmaxf((p.y - f.lo[1]) * f.scale[1], 0.f), m);
    const uint32_t cz = (uint32_t)fminf(fmaxf((p.z - f.lo[2]) * f.scale[2], 0.f), m);
    return part1by2(cx) | (part1by2(cy) << 1) | (part1by2(cz) << 2);
}

__global__ void sort_hist_kernel(const SortFrame f, const float *__restrict__ pts, long long n, const float *xf_dev,
                                 uint32_t *__restrict__ cell, uint32_t *__restrict__ hist) {
    SortFrame fr = f;
    if (xf_dev) {
#pragma unroll
        for (int e = 0; e < 12; ++e) fr.xf[e] = __ldg(xf_dev + e);
    }
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t c = sort_cell(fr, load_point(pts, i));
        cell[i] = c;
        atomicAdd(hist + c, 1u);
    }
}

// exclusive scan of the cell counters in place, one block of 1024 threads (256 counters per thread, moved as
// 64 independent 128-bit loads so that the single block is not serialised on L2 latency)
__global__ void __launch_bounds__(1024) sort_scan_kernel(uint32_t *__restrict__ hist, int n_cells) {
    __shared__ uint32_t warp_sum[32];
    const int per4 = n_cells / 1024 / 4;              // uint4 per thread (n_cells is a power of two >= 4096)
    uint4 *mine = reinterpret_cast<uint4 *>(hist) + (size_t)threadIdx.x * per4;
    uint32_t s = 0;
#pragma unroll 16
    for (int j = 0; j < per4; ++j) {
        const uint4 v = mine[j];
        s += v.x + v.y + v.z + v.w;
    }
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((threadIdx.x & 31) >= o) incl += t;
    }
    if ((threadIdx.x & 31) == 31) warp_sum[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t w = warp_sum[threadIdx.x], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (threadIdx.x >= o) wi += t;
        }
        warp_sum[threadIdx.x] = wi - w;
    }
    __syncthreads();
    uint32_t run = warp_sum[threadIdx.x >> 5] + (incl - s);
#pragma unroll 16
    for (int j = 0; j < per4; ++j) {
        const uint4 v = mine[j];
        uint4 o;
        o.x = run; o.y = run + v.x; o.z = o.y + v.y; o.w = o.z + v.z;
        run = o.w + v.w;
        mine[j] = o;
    }
}

// Scatter into binned order.  The tree-walk kernels then read their queries as ONE coalesced 16-byte record
// {x, y, z, original index} per lane and write their results as one coalesced 16-byte record {d, gx, gy, gz} into a
// staging buffer in binned order; unpermute_kernel brings them home with coalesced writes.  (Round 1 walked through an
// index permutation: 12-byte point loads and 4/12-byte result stores at random addresses, 32-byte sectors half used
// and read-modify-written -- many times the algorithmic bytes in DRAM traffic.)
// `cell_inv` holds the cell id of point i on entry and its binned position on exit (same thread reads, then writes).
__global__ void sort_scatter_kernel(uint32_t *__restrict__ cell_inv, const float *__restrict__ pts, long long n,
                                    uint32_t *__restrict__ offs, float4 *__restrict__ sorted) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t pos = atomicAdd(offs + cell_inv[i], 1u);
        const f3 p = load_point(pts, i);
        sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float((int)i));
        cell_inv[i] = pos;
    }
}

// results from binned order back to the callers' slots: coalesced writes, 16-byte gathers
__global__ void unpermute_kernel(const uint32_t *__restrict__ inv, const float4 *__restrict__ stage, long long n,
                                 float *__restrict__ out_dist, float *__restrict__ out_grad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float4 r = __ldg(stage + inv[i]);
        out_dist[i] = r.x;
        out_grad[3 * i] = r.y; out_grad[3 * i + 1] = r.z; out_grad[3 * i + 2] = r.w;
    }
}

struct SortedQueries {
    const float4 *sorted;     // {x, y, z, original index} in binned order; nullptr = not binned
    const uint32_t *inv;      // original index -> binned position
    float4 *stage;            // result staging, binned order
};

static size_t sort_workspace_bytes(long long n) {
    // counters | cell id / inverse permutation | binned points | result staging, each 16-byte aligned
    const size_t n4 = ((size_t)n * 4 + 15) / 16 * 16;
    return ((size_t)4 << (3 * sort_bits_for(n))) + n4 + (size_t)n * 16 * 2;
}

// ================================================================ mesh query
constexpr int kMeshThreads = 256;
#ifndef PVB_MESH_MINB
#define PVB_MESH_MINB 4   // 64 registers, 4 CTAs per SM: occupancy over registers for the latency-bound tree walk
#endif

__global__ void __launch_bounds__(kMeshThreads, PVB_MESH_MINB)
mesh_query_kernel(const pvb_sdf_desc m, const float *__restrict__ pts, long long n,
                  const float4 *__restrict__ sorted, float4 *__restrict__ stage, int run, uint32_t mode, int n_stage_max,
                  float *__restrict__ out_dist, float *__restrict__ out_grad, float *__restrict__ out_closest,
                  int *__restrict__ out_face, float *__restrict__ out_normal) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar;
    const NodeStage st = stage_nodes(m.nodes, m.n_nodes, n_stage_max, smem_raw, &bar);
    // Each thread owns runs of `run` CONSECUTIVE queries of the (binned) order: the closest point of the previous
    // query lies on the surface, so its distance to the next query bounds that query's answer from above and the
    // walk starts with a tight radius instead of infinity (neighbouring queries are centimetres apart).
    const long long threads = (long long)gridDim.x * blockDim.x;
    for (long long base = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * run; base < n; base += threads * run) {
        f3 prev_q = mk3(0.f, 0.f, 0.f);
        bool have_prev = false;
        for (int r = 0; r < run; ++r) {
            const long long j = base + r;
            if (j >= n) break;
            long long i = j;
            f3 p;
            if (sorted) {           // spatially binned order: one coalesced 16-byte record, original slot in .w
                const float4 sp = __ldg(sorted + j);
                p = mk3(sp.x, sp.y, sp.z);
                i = (long long)__float_as_int(sp.w);
            } else {
                p = load_point(pts, i);
            }
            float init_d2 = PVB_INF;
            if (have_prev) {
                const f3 e = prev_q - p;
                init_d2 = dot(e, e) * 1.0001f + 1e-12f;
            }
            f3 q;
            int face;
            SdfOut o = mesh_eval(m, st, p, mode, (uint64_t)i, &q, &face, init_d2);
            if (face < 0) o = mesh_eval(m, st, p, mode, (uint64_t)i, &q, &face);   // rounding: retry unbounded
            prev_q = q;
            have_prev = true;
            if (stage) {
                stage[j] = make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
            } else {
                out_dist[i] = o.val;
                out_grad[3 * i] = o.grad.x; out_grad[3 * i + 1] = o.grad.y; out_grad[3 * i + 2] = o.grad.z;
            }
            if (out_closest) { out_closest[3 * i] = q.x; out_closest[3 * i + 1] = q.y; out_closest[3 * i + 2] = q.z; }
            if (out_face) out_face[i] = face;
            if (out_normal) {
                const float *fn = m.face_normals + 3 * (size_t)max(face, 0);
                out_normal[3 * i] = __ldg(fn); out_normal[3 * i + 1] = __ldg(fn + 1); out_normal[3 * i + 2] = __ldg(fn + 2);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// EXTENSION (sign_mode="winding"): second pass over the result of an UNSIGNED mesh_query_kernel launch.  Keeps the
// hot kernel free of the third tree walk: inside/outside from the generalized winding number, then the reference's
// epilogue (sign of the distance, direction of the gradient, face normal inside the 1e-3 shell; sdf.py:154-164).
__global__ void __launch_bounds__(256)
mesh_winding_kernel(const pvb_sdf_desc m, const float *__restrict__ pts, long long n,
                    const float4 *__restrict__ sorted, float4 *__restrict__ stage, uint32_t mode,
                    float *__restrict__ dist, float *__restrict__ grad, const int *__restrict__ face) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const float4 *nodes = reinterpret_cast<const float4 *>(m.nodes);
    const float4 *tris = reinterpret_cast<const float4 *>(m.tris);
    const float4 *wn = reinterpret_cast<const float4 *>(m.wn_nodes);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        long long i = j;
        f3 p;
        if (sorted) {
            const float4 sp = __ldg(sorted + j);
            p = mk3(sp.x, sp.y, sp.z);
            i = (long long)__float_as_int(sp.w);
        } else {
            p = load_point(pts, i);
        }
        // consistently oriented surface: w = +1 inside for outward normals, -1 for inward ones
        const bool inside = fabsf(bvh_winding(nodes, wn, st, tris, p)) > 0.5f;
        float d;                                         // unsigned pass: d >= 0, gradient points away from the surface
        f3 g;
        if (stage) {
            const float4 r = stage[j];
            d = r.x; g = mk3(r.y, r.z, r.w);
        } else {
            d = dist[i]; g = mk3(grad[3 * i], grad[3 * i + 1], grad[3 * i + 2]);
        }
        if (inside) { d = -d; g = mk3(-g.x, -g.y, -g.z); }
        if ((mode & PVB_MESH_SURFACE_NORMAL) && fabsf(d) < 1e-3f && face[i] >= 0) {
            const float *fn = m.face_normals + 3 * (size_t)face[i];
            g = mk3(__ldg(fn), __ldg(fn + 1), __ldg(fn + 2));
        }
        if (stage) {
            stage[j] = make_float4(d, g.x, g.y, g.z);
        } else {
            dist[i] = d;
            grad[3 * i] = g.x; grad[3 * i + 1] = g.y; grad[3 * i + 2] = g.z;
        }
    }
}

// =============================================================== grid lookup
// Streaming kernel: 28 B of compulsory HBM traffic per point (12 in, 16 out);
// the table (16 B/voxel, interleaved {val,gx,gy,gz}) stays L2 resident.
constexpr int kGridThreads = 256;

// 4 points per thread and per quad: three 128-bit loads cover 4 xyz triples, results leave as one float4 of values
// and three float4 of gradients.  PVB_GRID_UNROLL quads are in flight per thread (all loads issued before any
// dependent work) so that enough bytes are outstanding to cover HBM latency at the occupancy the register count
// allows.
#ifndef PVB_GRID_UNROLL
#define PVB_GRID_UNROLL 2
#endif
#ifndef PVB_GRID_MINB
#define PVB_GRID_MINB 4
#endif

template <bool kMesh>
__device__ __forceinline__ void grid_quad(const pvb_sdf_desc &g, const NodeStage &st, long long t, float4 a, float4 b,
                                          float4 c, uint32_t mesh_mode, float4 *__restrict__ out_val4,
                                          float4 *__restrict__ out_grad4, uchar4 *__restrict__ out_outside4,
                                          float surface_level, longlong2 *__restrict__ out_index2) {
    const f3 p[4] = {mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), mk3(b.z, b.w, c.x), mk3(c.y, c.z, c.w)};
    SdfOut o[4];
    long long key[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = grid_eval<kMesh>(g, st, p[k], mesh_mode, (uint64_t)(4 * t + k), &key[k]);
    if (out_val4) __stcs(out_val4 + t, make_float4(o[0].val, o[1].val, o[2].val, o[3].val));
    if (out_grad4) {
        __stcs(out_grad4 + 3 * t, make_float4(o[0].grad.x, o[0].grad.y, o[0].grad.z, o[1].grad.x));
        __stcs(out_grad4 + 3 * t + 1, make_float4(o[1].grad.y, o[1].grad.z, o[2].grad.x, o[2].grad.y));
        __stcs(out_grad4 + 3 * t + 2, make_float4(o[2].grad.z, o[3].grad.x, o[3].grad.y, o[3].grad.z));
    }
    if (out_outside4) {   // outside_surface: out of range => outside (sdf.py:600-601)
        uchar4 m;
        m.x = key[0] < 0 ? 1 : (o[0].val > surface_level);
        m.y = key[1] < 0 ? 1 : (o[1].val > surface_level);
        m.z = key[2] < 0 ? 1 : (o[2].val > surface_level);
        m.w = key[3] < 0 ? 1 : (o[3].val > surface_level);
        out_outside4[t] = m;
    }
    if (out_index2) {
        out_index2[2 * t] = make_longlong2(key[0], key[1]);
        out_index2[2 * t + 1] = make_longlong2(key[2], key[3]);
    }
}

template <bool kMesh>
__global__ void __launch_bounds__(kGridThreads, PVB_GRID_MINB)
grid_lookup_vec4_kernel(const pvb_sdf_desc g, const float4 *__restrict__ pts4, long long n_quads, uint32_t mesh_mode,
                        float4 *__restrict__ out_val4, float4 *__restrict__ out_grad4,
                        uchar4 *__restrict__ out_outside4, float surface_level, longlong2 *__restrict__ out_index2) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; t + (PVB_GRID_UNROLL - 1) * stride < n_quads; t += PVB_GRID_UNROLL * stride) {
        float4 a[PVB_GRID_UNROLL], b[PVB_GRID_UNROLL], c[PVB_GRID_UNROLL];
#pragma unroll
        for (int u = 0; u < PVB_GRID_UNROLL; ++u) {
            const float4 *src = pts4 + 3 * (t + u * stride);
            a[u] = __ldcs(src); b[u] = __ldcs(src + 1); c[u] = __ldcs(src + 2);
        }
#pragma unroll
        for (int u = 0; u < PVB_GRID_UNROLL; ++u)
            grid_quad<kMesh>(g, st, t + u * stride, a[u], b[u], c[u], mesh_mode, out_val4, out_grad4, out_outside4,
                             surface_level, out_index2);
    }
    for (; t < n_quads; t += stride) {
        const float4 *src = pts4 + 3 * t;
        const float4 a = __ldcs(src), b = __ldcs(src + 1), c = __ldcs(src + 2);
        grid_quad<kMesh>(g, st, t, a, b, c, mesh_mode, out_val4, out_grad4, out_outside4, surface_level, out_index2);
    }
}

// ---------------------------------------------------------------------------------------------------------
// TMA-streamed variant (the C2 headline path).  Random table gathers cost ~2 L1 wavefront-cycles per lane and
// cannot be coalesced, so the LSU is the scarce resource of this kernel; the AoS point / gradient streams (48-byte
// lane stride = 12 cache lines per warp instruction) would spend as much LSU time again.  They are therefore
// moved by the bulk-copy engine instead: one cp.async.bulk brings a tile of TILE points into shared memory
// (double buffered, mbarrier completion), threads read their 4 points with three conflict-free LDS.128, results
// are staged in shared memory and leave with cp.async.bulk shared->global stores (bulk groups).  The LSU then
// only executes the gathers.
#ifndef PVB_TMA_THREADS
#define PVB_TMA_THREADS 256
#endif
constexpr int kTmaThreads = PVB_TMA_THREADS;
constexpr int kTmaTile = kTmaThreads * 4;              // points per tile
struct __align__(128) GridTmaSmem {
    float in[2][kTmaTile * 3];                         // 2 x 12 KB
    float outv[2][kTmaTile];                           // 2 x  4 KB
    float outg[2][kTmaTile * 3];                       // 2 x 12 KB
    uint64_t full[2];
};

__global__ void __launch_bounds__(kTmaThreads)
grid_lookup_tma_kernel(const pvb_sdf_desc g, const float *__restrict__ pts, long long n_pts /* multiple of 4 */,
                       float *__restrict__ out_val, float *__restrict__ out_grad) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    GridTmaSmem &s = *reinterpret_cast<GridTmaSmem *>(smem_raw);
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_tiles = (n_pts + kTmaTile - 1) / kTmaTile;
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&s.full[0], 1);
        mbar_init(&s.full[1], 1);
    }
    __syncthreads();
    auto tile_points = [&](long long tile) -> uint32_t {
        const long long left = n_pts - tile * kTmaTile;
        return (uint32_t)(left < kTmaTile ? left : kTmaTile);
    };
    long long tile = blockIdx.x;
    if (tid == 0 && tile < n_tiles) {
        const uint32_t bytes = tile_points(tile) * 12u;
        mbar_expect_tx(&s.full[0], bytes);
        bulk_g2s(s.in[0], pts + tile * kTmaTile * 3, bytes, &s.full[0]);
    }
    for (int it = 0; tile < n_tiles; ++it, tile += gridDim.x) {
        const int buf = it & 1;
        const long long next = tile + gridDim.x;
        if (tid == 0 && next < n_tiles) {      // in[buf^1] was released by the __syncthreads of the previous iteration
            const uint32_t bytes = tile_points(next) * 12u;
            mbar_expect_tx(&s.full[buf ^ 1], bytes);
            bulk_g2s(s.in[buf ^ 1], pts + next * kTmaTile * 3, bytes, &s.full[buf ^ 1]);
        }
        mbar_wait(&s.full[buf], (uint32_t)((it >> 1) & 1));
        const uint32_t npt = tile_points(tile);
        const bool active = (uint32_t)(4 * tid) < npt;
        SdfOut o[4];
        if (active) {
            const float4 *src = reinterpret_cast<const float4 *>(s.in[buf]) + 3 * tid;
            const float4 a = src[0], b = src[1], c = src[2];
            const f3 p[4] = {mk3(a.x, a.y, a.z), mk3(a.w, b.x, b.y), mk3(b.z, b.w, c.x), mk3(c.y, c.z, c.w)};
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = grid_eval<false>(g, st, p[k], 0u, 0ull, nullptr);
        }
        // out[buf] was handed to the bulk-store engine two iterations ago: wait until it has been read
        if (tid == 0) bulk_wait_read<1>();
        __syncthreads();
        if (active) {
            reinterpret_cast<float4 *>(s.outv[buf])[tid] = make_float4(o[0].val, o[1].val, o[2].val, o[3].val);
            float4 *dg = reinterpret_cast<float4 *>(s.outg[buf]) + 3 * tid;
            dg[0] = make_float4(o[0].grad.x, o[0].grad.y, o[0].grad.z, o[1].grad.x);
            dg[1] = make_float4(o[1].grad.y, o[1].grad.z, o[2].grad.x, o[2].grad.y);
            dg[2] = make_float4(o[2].grad.z, o[3].grad.x, o[3].grad.y, o[3].grad.z);
        }
        fence_async_smem();       // generic-proxy smem writes -> visible to the async (bulk copy) proxy
        __syncthreads();          // also releases in[buf] for the load issued in the next iteration
        if (tid == 0) {
            bulk_s2g(out_val + tile * kTmaTile, s.outv[buf], npt * 4u);
            bulk_s2g(out_grad + tile * kTmaTile * 3, s.outg[buf], npt * 12u);
            bulk_commit();
        }
    }
    if (tid == 0) bulk_wait_read<0>();
}

// ---------------------------------------------------------------------------------------------------------
// EXTENSION, opt-in (CachedSDF(interpolation="trilinear")): the trilinear interpolant of the value table and its
// analytic gradient, grid_trilinear_eval (pvb_device.cuh) per point.  Every other kernel in this section reproduces
// the reference's nearest-voxel rule.
__global__ void __launch_bounds__(256)
grid_trilinear_kernel(const pvb_sdf_desc g, const float *__restrict__ pts, long long n, float *__restrict__ out_val,
                      float *__restrict__ out_grad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const SdfOut o = grid_trilinear_eval(g, load_point(pts, i));
        out_val[i] = o.val;
        out_grad[3 * i] = o.grad.x; out_grad[3 * i + 1] = o.grad.y; out_grad[3 * i + 2] = o.grad.z;
    }
}

// scalar variant for the tail and for unaligned views
template <bool kMesh>
__global__ void __launch_bounds__(kGridThreads)
grid_lookup_scalar_kernel(const pvb_sdf_desc g, const float *__restrict__ pts, long long first, long long n,
                          uint32_t mesh_mode, float *__restrict__ out_val, float *__restrict__ out_grad,
                          uint8_t *__restrict__ out_outside, float surface_level, long long *__restrict__ out_index) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = first + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const f3 p = load_point(pts, i);
        long long key;
        const SdfOut o = grid_eval<kMesh>(g, st, p, mesh_mode, (uint64_t)i, &key);
        if (out_val) out_val[i] = o.val;
        if (out_grad) { out_grad[3 * i] = o.grad.x; out_grad[3 * i + 1] = o.grad.y; out_grad[3 * i + 2] = o.grad.z; }
        if (out_outside) out_outside[i] = key < 0 ? 1 : (o.val > surface_level);
        if (out_index) out_index[i] = key;
    }
}

// ==================================================================== sphere
__global__ void sphere_kernel(float radius, const float *__restrict__ pts, long long n, float *__restrict__ out_val,
                              float *__restrict__ out_grad) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const SdfOut o = sphere_eval(radius, load_point(pts, i));
        out_val[i] = o.val;
        out_grad[3 * i] = o.grad.x; out_grad[3 * i + 1] = o.grad.y; out_grad[3 * i + 2] = o.grad.z;
    }
}

// ============================================================ composed query
// One thread per (configuration, 1 or 4 points): walks the S sub-SDFs in registers -- transform into the sub-frame,
// evaluate, keep the running min (first index on ties, as torch.argmin), rotate the winning gradient back -- and
// writes (val, grad) once.  The S*|A|*P*3 intermediates of sdf.py:399-415 never exist.
//
// Where the time goes is the LSU: a random 16-byte table gather costs L1 wavefront-cycles per lane
// (scripts/ubench_gather.cu measures how many), and so does every warp-uniform LDS/LDG.  Hence
//   * the descriptors travel as a __grid_constant__ kernel parameter (constant bank, uniform datapath, no LSU);
//     the first version staged them in shared memory and spent more LSU cycles on descriptor fields than on gathers
//   * 4 points per thread: one broadcast read of a link transform serves 4 points; points / results move as
//     128-bit coalesced loads and stores
//   * exact pruning: a sub-SDF whose AABB lower bound already exceeds the running min cannot be the argmin
//     (margin measured on the table at build time), compared on squared distances (no MUFU)
constexpr int kCompThreads = 256;
constexpr int kCompSmemXf = 64;
#ifndef PVB_COMP_PTS
#define PVB_COMP_PTS 2        // points per thread on the vector path (1, 2 or 4)
#endif
#ifndef PVB_COMP_MINB
#define PVB_COMP_MINB 4
#endif
#ifndef PVB_COMPMESH_MINB
#define PVB_COMPMESH_MINB 4   // CTAs per SM of the mesh instantiation (C3, 16 drills): occupancy hides the tree walk
#endif

// `order` is the sequence in which the sub-SDFs are visited: the bit-reversal permutation of 0..n-1.  Along a
// kinematic chain the distance to consecutive links changes monotonically for most points, so index order makes
// almost every link a new running minimum (4.5 lookups per (configuration, point) on the C4 arm); the coarse-to-fine
// bit-reversed order reaches a tight bound early (3.1 lookups, measured with the AABB bounds on the host).  The
// argmin keeps torch's first-index tie rule explicitly, so the visiting order never changes a result.
template <int MAXS>
struct DescPack {
    pvb_sdf_desc d[MAXS];
    unsigned char order[MAXS];
};

template <int MAXS>
static void fill_order(DescPack<MAXS> &pack, int n) {
    int bits = 0;
    while ((1 << bits) < n) ++bits;
    int m = 0;
    for (int i = 0; i < (1 << bits); ++i) {
        int r = 0;
        for (int b = 0; b < bits; ++b) r |= ((i >> b) & 1) << (bits - 1 - b);
        if (r < n) pack.order[m++] = (unsigned char)r;
    }
    static const int plain = [] { const char *e = getenv("PVB_COMP_INDEX_ORDER"); return e ? atoi(e) : 0; }();
    if (plain) for (int i = 0; i < n; ++i) pack.order[i] = (unsigned char)i;
}

// Destinations of the multi-target variants (kMulti): the local result buffer and the peer-mapped buffers of the
// other ranks, each already advanced to this rank's configuration slab.  Stores to peer memory travel over NVLink
// while the kernel keeps evaluating, so a configuration-sharded RobotSDF result is re-assembled on every rank
// without a trailing all-gather.
struct OutTargets {
    float *val[PVB_MAX_TARGETS];
    float *grad[PVB_MAX_TARGETS];
    int n;
    int vec;        // all pointers 16-byte aligned and n_pts % 4 == 0: rows may be stored as float4
    int mc;         // val[0] / grad[0] are MULTICAST addresses (NVLS): one multimem.st reaches every bound GPU
};

template <bool kMesh, int PTS, int MAXS, bool kMulti, bool kExt>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : (PTS > 1 ? PVB_COMP_MINB : 1)))
composed_query_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf, const float *__restrict__ xforms,
                      int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long first_pt,
                      long long n_pts, uint32_t mesh_mode, float *__restrict__ out_val, float *__restrict__ out_grad,
                      int *__restrict__ out_which, const __grid_constant__ OutTargets tg, int nearest_first,
                      float margin_max) {
    __shared__ __align__(16) float s_xf[kCompSmemXf][12];
    const bool use_smem = n_sdf <= kCompSmemXf;
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_items = (n_pts - first_pt) / PTS;     // work items of PTS consecutive points
    for (int c = blockIdx.y; c < cfg_count; c += gridDim.y) {
        const int cfg = cfg_begin + c;
        __syncthreads();
        if (use_smem) {
            for (int w = threadIdx.x; w < n_sdf * 12; w += blockDim.x) {
                const int s = w / 12, e = w % 12;
                s_xf[s][e] = xforms[((size_t)s * n_cfg + cfg) * 16 + e];
            }
        }
        __syncthreads();
        const long long stride = (long long)gridDim.x * blockDim.x;
        for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_items; t += stride) {
            const long long i0 = first_pt + t * PTS;
            f3 p[PTS];
            if constexpr (PTS == 4) {
                const float4 *src = reinterpret_cast<const float4 *>(pts + 3 * i0);
                const float4 a = __ldg(src), b = __ldg(src + 1), cc = __ldg(src + 2);
                p[0] = mk3(a.x, a.y, a.z); p[1] = mk3(a.w, b.x, b.y); p[2] = mk3(b.z, b.w, cc.x);
                p[3] = mk3(cc.y, cc.z, cc.w);
            } else if constexpr (PTS == 2) {
                const float2 *src = reinterpret_cast<const float2 *>(pts + 3 * i0);
                const float2 a = __ldg(src), b = __ldg(src + 1), cc = __ldg(src + 2);
                p[0] = mk3(a.x, a.y, b.x); p[1] = mk3(b.y, cc.x, cc.y);
            } else {
                p[0] = load_point(pts, i0);
            }
            float best[PTS];
            f3 bg[PTS];
            int bs[PTS];
#pragma unroll
            for (int k = 0; k < PTS; ++k) { best[k] = PVB_INF; bg[k] = mk3(0.f, 0.f, 0.f); bs[k] = -1; }

            auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
                if (use_smem) {
                    const float4 *row = reinterpret_cast<const float4 *>(s_xf[s]);      // 3 x LDS.128 broadcast
                    r0 = row[0]; r1 = row[1]; r2 = row[2];
                } else {
                    const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
                    r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
                }
            };
            // every sub-SDF in visiting order, skipped when provably not the argmin (composed_consider,
            // pvb_device.cuh).  (Evaluating the sub-SDF with the smallest AABB lower bound first -- an extra pass
            // over all of them without table access -- saves lookups but adds issue slots to a kernel that is
            // issue-bound.)
            // ... except when sub-SDFs are MESHES (kMesh, one point per thread): an evaluation is a tree walk of
            // thousands of instructions, so one cheap pass computes every sub-SDF's AABB lower bound and the thread
            // then evaluates them NEAREST BOUND FIRST, stopping as soon as the smallest remaining bound exceeds the
            // running minimum.  A fixed order evaluates every sub-SDF that is a running record when its turn comes
            // (~H_16 = 3.4 of 16 at C3, plus those inside the slack); nearest-first evaluates the winner and its near
            // ties.  Exact for the same reason as the fixed order: bounds are conservative and the argmin keeps
            // torch's first-index rule explicitly.
            bool ordered = false;
            if constexpr (kMesh && PTS == 1) {
                if (n_sdf <= 32 && nearest_first) {
                    ordered = true;
                    float key[32];                           // squared lower bound; -1 = no valid bound (evaluate)
                    unsigned todo = n_sdf >= 32 ? 0xffffffffu : ((1u << n_sdf) - 1u);
                    for (int s = 0; s < n_sdf; ++s) {
                        const pvb_sdf_desc &d = descs.d[s];
                        float4 r0, r1, r2;
                        load_xf(s, r0, r1, r2);
                        const bool bounded = (d.kind == PVB_KIND_GRID || (kExt && d.kind != PVB_KIND_MESH))
                                                 ? (d.flags & PVB_GRID_PRUNE_OK) != 0
                                                 : (d.kind == PVB_KIND_MESH && (d.flags & PVB_MESH_CLOSED) && (mesh_mode & PVB_MESH_SIGNED));
                        const float lb2 = bounded ? composed_aabb_lb2(d, composed_xform(r0, r1, r2, p[0])) : -1.f;
                        // a closed mesh is bounded only from OUTSIDE its box (composed_consider): inside it, its value may be
                        // as deep as the mesh itself, far below -prune_margin, so a query in the box has no bound
                        key[s] = (d.kind == PVB_KIND_MESH && !(lb2 > 0.f)) ? -1.f : lb2;
                    }
                    while (todo) {
                        int s = -1;
                        float kmin = PVB_INF;
                        for (int t = 0; t < n_sdf; ++t)
                            if ((todo >> t) & 1u) { if (key[t] < kmin) { kmin = key[t]; s = t; } }
                        if (s < 0) break;
                        todo &= ~(1u << s);
                        const pvb_sdf_desc &d = descs.d[s];
                        if (bs[0] >= 0 && kmin >= 0.f) {
                            // every remaining bound is at least kmin: when even the most generous margin cannot bring
                            // it under the running minimum, nothing left can win (margins are per sub-SDF: test this one
                            // exactly, and stop the loop only on the margin-free comparison)
                            const float thr = best[0] + d.prune_margin;
                            if (thr < 0.f || kmin > thr * thr) {
                                if (best[0] + margin_max < 0.f || kmin > (best[0] + margin_max) * (best[0] + margin_max)) break;
                                continue;
                            }
                        }
                        float4 r0, r1, r2;
                        load_xf(s, r0, r1, r2);
                        const uint64_t idx = ((uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i0) * (uint64_t)n_sdf + (uint64_t)s;
                        composed_consider<kMesh, kExt>(d, st, s, composed_xform(r0, r1, r2, p[0]), mesh_mode, idx, best[0], bg[0], bs[0]);
                    }
                }
            }
            for (int si = 0; si < (ordered ? 0 : n_sdf); ++si) {
                const int s = descs.order[si];
                const pvb_sdf_desc &d = descs.d[s];
                float4 r0, r1, r2;
                load_xf(s, r0, r1, r2);
#pragma unroll
                for (int k = 0; k < PTS; ++k) {
                    const uint64_t idx = ((uint64_t)cfg * (uint64_t)n_pts + (uint64_t)(i0 + k)) * (uint64_t)n_sdf + (uint64_t)s;   // absolute cfg: sharding-independent jitter
                    composed_consider<kMesh, kExt>(d, st, s, composed_xform(r0, r1, r2, p[k]), mesh_mode, idx, best[k], bg[k],
                                                   bs[k]);
                }
            }
            f3 go[PTS];
#pragma unroll
            for (int k = 0; k < PTS; ++k) {
                float4 r0, r1, r2;
                load_xf(max(bs[k], 0), r0, r1, r2);
                go[k] = composed_rotate_back(r0, r1, r2, bg[k]);
            }
            const long long o_i = (long long)c * n_pts + i0;
            auto emit = [&](float *ov, float *og) {
                if constexpr (PTS == 4) {
                    __stcs(reinterpret_cast<float4 *>(ov + o_i), make_float4(best[0], best[1], best[2], best[3]));
                    float4 *dg = reinterpret_cast<float4 *>(og + 3 * o_i);
                    __stcs(dg, make_float4(go[0].x, go[0].y, go[0].z, go[1].x));
                    __stcs(dg + 1, make_float4(go[1].y, go[1].z, go[2].x, go[2].y));
                    __stcs(dg + 2, make_float4(go[2].z, go[3].x, go[3].y, go[3].z));
                } else if constexpr (PTS == 2) {
                    __stcs(reinterpret_cast<float2 *>(ov + o_i), make_float2(best[0], best[1]));
                    float2 *dg = reinterpret_cast<float2 *>(og + 3 * o_i);
                    __stcs(dg, make_float2(go[0].x, go[0].y));
                    __stcs(dg + 1, make_float2(go[0].z, go[1].x));
                    __stcs(dg + 2, make_float2(go[1].y, go[1].z));
                } else {
                    ov[o_i] = best[0];
                    og[3 * o_i] = go[0].x; og[3 * o_i + 1] = go[0].y; og[3 * o_i + 2] = go[0].z;
                }
            };
            if constexpr (kMulti) {
                for (int t = 0; t < tg.n; ++t) emit(tg.val[t], tg.grad[t]);
            } else {
                emit(out_val, out_grad);
            }
            if (out_which) {
                if constexpr (PTS == 4) *reinterpret_cast<int4 *>(out_which + o_i) = make_int4(bs[0], bs[1], bs[2], bs[3]);
                else if constexpr (PTS == 2) *reinterpret_cast<int2 *>(out_which + o_i) = make_int2(bs[0], bs[1]);
                else out_which[o_i] = bs[0];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// Paired query: configuration c is evaluated at its OWN points pts[c][0 .. n_pts) instead of the point set all
// configurations share (trajectory steps against per-step obstacles, MPC rollouts, batched environments):
// cfg_count * n_pts pairs instead of the cfg_count x (cfg_count * n_pts) cross product.  One thread per pair
// t = c * n_pts + i, running composed_point with the jitter index of the absolute configuration, so the result equals
// pvb_composed_query(pts[c], cfg_begin + c, 1) bit for bit.  The transform rows are read per thread with __ldg rather
// than staged per block like composed_query_kernel does: with few points per configuration one block spans many
// configurations, and the lanes of one configuration read the same rows (L1 broadcasts).
template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
composed_paired_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf, const float *__restrict__ xforms,
                       int n_cfg, int cfg_begin, const float *__restrict__ pts, long long n_pts, long long n_pairs,
                       uint32_t mesh_mode, float *__restrict__ out_val, float *__restrict__ out_grad,
                       int *__restrict__ out_which, int nearest_first, float margin_max) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_pairs; t += stride) {
        long long c, i;
        paired_index(t, n_pts, c, i);
        const int cfg = cfg_begin + (int)c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
            const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
            r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
        };
        const ComposedOut o = composed_point<kMesh, kExt>(descs.d, descs.order, n_sdf, load_xf, st, load_point(pts, t),
                                                          mesh_mode, (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i,
                                                          nearest_first, margin_max);
        out_val[t] = o.val;
        out_grad[3 * t] = o.grad.x; out_grad[3 * t + 1] = o.grad.y; out_grad[3 * t + 2] = o.grad.z;
        if (out_which) out_which[t] = o.which;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Swept query, every sub-SDF set the composed query accepts (meshes, PVB_GRID_OOB_GT, 9-128 sub-SDFs): the minimum
// over the configurations cfg_begin .. cfg_begin + cfg_count - 1 at every point, in the order of swept_fold
// (pvb_device.cuh).  One thread per point walks the configurations in ascending order through composed_point with the
// jitter index of the absolute configuration, as composed_paired_kernel does, so every configuration's result is the
// per-configuration query's bit for bit.  out_cfg: the absolute configuration of the result.
template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
composed_swept_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf, const float *__restrict__ xforms,
                      int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_pts,
                      uint32_t mesh_mode, float *__restrict__ out_val, float *__restrict__ out_grad,
                      int *__restrict__ out_cfg, int *__restrict__ out_which, int nearest_first, float margin_max) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pts; i += stride) {
        const f3 p = load_point(pts, i);
        SweptBest b;
        b.val = PVB_INF; b.grad = mk3(0.f, 0.f, 0.f); b.cfg = -1; b.which = -1;
        for (int c = 0; c < cfg_count; ++c) {
            const int cfg = cfg_begin + c;
            auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
                const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
                r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
            };
            const ComposedOut o = composed_point<kMesh, kExt>(descs.d, descs.order, n_sdf, load_xf, st, p, mesh_mode,
                                                              (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i,
                                                              nearest_first, margin_max);
            swept_fold(b, o.val, o.grad, cfg, o.which);
        }
        out_val[i] = b.val;
        out_grad[3 * i] = b.grad.x; out_grad[3 * i + 1] = b.grad.y; out_grad[3 * i + 2] = b.grad.z;
        if (out_cfg) out_cfg[i] = b.cfg;
        if (out_which) out_which[i] = b.which;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Clearance query, every sub-SDF set the composed query accepts (meshes, PVB_GRID_OOB_GT, 9-128 sub-SDFs): for every
// configuration c of the slab and every segment b of seg_len points, the smallest clearance_key (pvb_device.cuh) over
// the segment's points, left in keys[c * n_seg + b] (which holds ~0 on entry).  One thread per (configuration, point)
// pair t = c * n_pts + i runs composed_point with the absolute configuration and the flat point index, the jitter
// inputs of the per-configuration query.  The lanes of a warp cover consecutive pairs, so lanes of the same key form
// runs: a segmented shuffle reduction leaves each run's minimum in its first lane, which issues one atomicMin.
// kPaired (composed_paired_clearance_kernel, pvb_composed_query_paired_clearance): configuration c has its own points,
// the point of pair t is pts[t] instead of pts[i]; the jitter index stays cfg * n_pts + i, that of the
// per-configuration query on pts[c].  (The flag sits on the inlined body, so that composed_clearance_kernel keeps its
// name and its code.)
template <bool kMesh, bool kExt, int MAXS, bool kPaired>
__device__ __forceinline__ void clearance_pairs(const DescPack<MAXS> &descs, int n_sdf, const float *__restrict__ xforms,
                                                int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts,
                                                long long n_seg, long long seg_len, uint32_t mesh_mode,
                                                unsigned long long *__restrict__ keys, int nearest_first,
                                                float margin_max) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const int lane = threadIdx.x & 31;
    const long long n_pts = n_seg * seg_len, total = (long long)cfg_count * n_pts;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // warp-uniform loop: every lane takes part in the shuffles below
    for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < total; base += stride) {
        const long long t = base + lane;
        unsigned long long k = ~0ull;
        long long tgt = -1;
        if (t < total) {
            long long c, i;
            paired_index(t, n_pts, c, i);
            const long long b = i / seg_len;
            const int cfg = cfg_begin + (int)c;
            auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
                const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
                r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
            };
            const ComposedOut o = composed_point<kMesh, kExt>(descs.d, descs.order, n_sdf, load_xf, st,
                                                              load_point(pts, kPaired ? t : i), mesh_mode,
                                                              (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i,
                                                              nearest_first, margin_max);
            k = clearance_key(o.val, (uint32_t)(i - b * seg_len));
            tgt = c * n_seg + b;
        }
        // after step `off`, lane l holds the minimum over lanes l .. l + 2 off - 1 of its own run
        for (int off = 1; off < 32; off <<= 1) {
            const unsigned long long ok = __shfl_down_sync(0xffffffffu, k, off);
            const long long ot = __shfl_down_sync(0xffffffffu, tgt, off);
            if (lane + off < 32 && ot == tgt && ok < k) k = ok;
        }
        const long long prev = __shfl_up_sync(0xffffffffu, tgt, 1);
        if (tgt >= 0 && (lane == 0 || prev != tgt)) atomicMin(keys + tgt, k);
    }
}

template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
composed_clearance_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf, const float *__restrict__ xforms,
                          int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_seg,
                          long long seg_len, uint32_t mesh_mode, unsigned long long *__restrict__ keys,
                          int nearest_first, float margin_max) {
    clearance_pairs<kMesh, kExt, MAXS, false>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                              mesh_mode, keys, nearest_first, margin_max);
}

template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
composed_paired_clearance_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf,
                                 const float *__restrict__ xforms, int n_cfg, int cfg_begin, int cfg_count,
                                 const float *__restrict__ pts, long long n_seg, long long seg_len, uint32_t mesh_mode,
                                 unsigned long long *__restrict__ keys, int nearest_first, float margin_max) {
    clearance_pairs<kMesh, kExt, MAXS, true>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                             mesh_mode, keys, nearest_first, margin_max);
}

// The result of a clearance query: one thread per (configuration c, segment b) decodes the point i* of its key and
// evaluates that single pair with composed_point -- the same descriptors, absolute configuration and flat point index
// as the per-configuration query -- into the value, world gradient, i* and sub-SDF.  Whichever kernel produced the
// key, its value is this pair's per-configuration value (robot_clearance_kernel's visits give composed_point's bits
// for every link kind: tests/test_clearance_cpu.py).  kPaired (paired_clearance_finish_kernel): the point of (c, b) is
// pts[c * n_pts + i], as in composed_paired_clearance_kernel.
template <bool kMesh, bool kExt, int MAXS, bool kPaired>
__device__ __forceinline__ void clearance_finish(const DescPack<MAXS> &descs, int n_sdf,
                                                 const float *__restrict__ xforms, int n_cfg, int cfg_begin,
                                                 int cfg_count, const float *__restrict__ pts, long long n_seg,
                                                 long long seg_len, uint32_t mesh_mode,
                                                 const unsigned long long *__restrict__ keys,
                                                 float *__restrict__ out_val, float *__restrict__ out_grad,
                                                 int *__restrict__ out_point, int *__restrict__ out_which,
                                                 int nearest_first, float margin_max) {
    NodeStage st; st.smem = nullptr; st.n = 0;
    const long long n_pts = n_seg * seg_len, total = (long long)cfg_count * n_seg;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        long long c, b;
        paired_index(t, n_seg, c, b);
        const int ip = (int)(uint32_t)keys[t];
        const long long i = b * seg_len + ip;
        const int cfg = cfg_begin + (int)c;
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) {
            const float4 *row = xf_rows(xforms, n_cfg, s, cfg);
            r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
        };
        const ComposedOut o = composed_point<kMesh, kExt>(descs.d, descs.order, n_sdf, load_xf, st,
                                                          load_point(pts, kPaired ? c * n_pts + i : i), mesh_mode,
                                                          (uint64_t)cfg * (uint64_t)n_pts + (uint64_t)i,
                                                          nearest_first, margin_max);
        out_val[t] = o.val;
        out_grad[3 * t] = o.grad.x; out_grad[3 * t + 1] = o.grad.y; out_grad[3 * t + 2] = o.grad.z;
        if (out_point) out_point[t] = ip;
        if (out_which) out_which[t] = o.which;
    }
}

template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
clearance_finish_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf, const float *__restrict__ xforms,
                        int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_seg,
                        long long seg_len, uint32_t mesh_mode, const unsigned long long *__restrict__ keys,
                        float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_point,
                        int *__restrict__ out_which, int nearest_first, float margin_max) {
    clearance_finish<kMesh, kExt, MAXS, false>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                               mesh_mode, keys, out_val, out_grad, out_point, out_which,
                                               nearest_first, margin_max);
}

template <bool kMesh, bool kExt, int MAXS>
__global__ void __launch_bounds__(kCompThreads, (kMesh ? PVB_COMPMESH_MINB : 1))
paired_clearance_finish_kernel(const __grid_constant__ DescPack<MAXS> descs, int n_sdf,
                               const float *__restrict__ xforms, int n_cfg, int cfg_begin, int cfg_count,
                               const float *__restrict__ pts, long long n_seg, long long seg_len, uint32_t mesh_mode,
                               const unsigned long long *__restrict__ keys, float *__restrict__ out_val,
                               float *__restrict__ out_grad, int *__restrict__ out_point, int *__restrict__ out_which,
                               int nearest_first, float margin_max) {
    clearance_finish<kMesh, kExt, MAXS, true>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                              mesh_mode, keys, out_val, out_grad, out_point, out_which, nearest_first,
                                              margin_max);
}

// ------------------------------------------------------------------------------------------------------------
// Configuration-major variant for RobotSDF-style batches (many joint configurations, shared points).
//
// Lanes of a warp are 32 CONFIGURATIONS of the same point instead of 32 points of the same configuration:
// neighbouring configurations place every link almost identically, so (a) the prune / evaluate decisions of a
// warp agree (the point-major kernel ran at 24/32 active lanes and evaluated nearly all 8 links per warp because
// some lane always needed them), (b) the 32 table gathers of a warp instruction fall into a handful of cache lines
// instead of 32, and (c) a cheap first-stage bound becomes worthwhile: the link's bounding sphere, carried into
// the OBJECT frame once per (configuration, link), rejects a link with 9 instructions and without transforming
// the point.  Results are bit-identical to the point-major kernel (same transform / lookup arithmetic; pruning is
// exact).  A block owns a tile of 32 configurations x 32 points; results are transposed through shared memory so
// that global stores stay coalesced along the point axis.
// (Visiting the link with the nearest bounding sphere first is not done here: the extra pass costs more than the
// lookups it saves in this configuration-major layout.)
constexpr int kCmCfg = 32;
constexpr int kCmWarps = 8;
constexpr int kCmPts = 4;                         // points per thread
constexpr int kCmTilePts = kCmWarps * kCmPts;     // 32
constexpr int kCmMaxS = 16;
struct __align__(16) CmSmem {
    float4 xf[kCmCfg][3 * kCmMaxS + 1];           // row stride = 49 float4: conflict-free LDS.128 across lanes
    float4 sph[kCmCfg][kCmMaxS + 1];              // bounding sphere (object frame) per (cfg, link); stride 17
    float4 out[kCmCfg][kCmTilePts + 1];           // {val, gx, gy, gz}; stride 33
    int which[kCmCfg][kCmTilePts + 1];
};

template <bool kMulti, bool kExt>
__global__ void __launch_bounds__(kCmCfg * kCmWarps, 3)
composed_cfgmajor_kernel(const __grid_constant__ DescPack<kCmMaxS> descs, int n_sdf, const float *__restrict__ xforms,
                         int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_pts,
                         float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_which,
                         const __grid_constant__ OutTargets tg) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    CmSmem &sm = *reinterpret_cast<CmSmem *>(smem_raw);
    NodeStage st; st.smem = nullptr; st.n = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = blockIdx.y * kCmCfg;                       // first configuration (relative to cfg_begin)
    const int ncfg = min(kCmCfg, cfg_count - c0);
    // ---- stage the transforms of this configuration tile and the object-frame bounding spheres ----
    for (int item = threadIdx.x; item < kCmCfg * n_sdf; item += blockDim.x) {
        const int ci = item % kCmCfg, s = item / kCmCfg;
        const pvb_sdf_desc &d = descs.d[s];
        float4 r0 = make_float4(1.f, 0.f, 0.f, 0.f), r1 = make_float4(0.f, 1.f, 0.f, 0.f),
               r2 = make_float4(0.f, 0.f, 1.f, 0.f);
        if (ci < ncfg) {
            const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg_begin + c0 + ci) * 16);
            r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
        }
        sm.xf[ci][3 * s] = r0; sm.xf[ci][3 * s + 1] = r1; sm.xf[ci][3 * s + 2] = r2;
        // sphere around the link AABB, centre carried to the object frame: c_obj = R^T (c_link - t)
        const f3 cl = mk3(0.5f * (d.bb_min[0] + d.bb_max[0]), 0.5f * (d.bb_min[1] + d.bb_max[1]),
                          0.5f * (d.bb_min[2] + d.bb_max[2]));
        const f3 hl = mk3(0.5f * (d.bb_max[0] - d.bb_min[0]), 0.5f * (d.bb_max[1] - d.bb_min[1]),
                          0.5f * (d.bb_max[2] - d.bb_min[2]));
        const f3 u = mk3(cl.x - r0.w, cl.y - r1.w, cl.z - r2.w);
        const f3 co = mk3(r0.x * u.x + r1.x * u.y + r2.x * u.z, r0.y * u.x + r1.y * u.y + r2.y * u.z,
                          r0.z * u.x + r1.z * u.y + r2.z * u.z);
        float rad = sqrtf(hl.x * hl.x + hl.y * hl.y + hl.z * hl.z) * 1.0001f + 1e-6f;
        // the bound needs an isometry: |R R^T - I| must vanish, otherwise this (cfg, link) never prunes in stage 1
        const float e00 = r0.x * r0.x + r0.y * r0.y + r0.z * r0.z - 1.f, e11 = r1.x * r1.x + r1.y * r1.y + r1.z * r1.z - 1.f,
                    e22 = r2.x * r2.x + r2.y * r2.y + r2.z * r2.z - 1.f;
        const float e01 = r0.x * r1.x + r0.y * r1.y + r0.z * r1.z, e02 = r0.x * r2.x + r0.y * r2.y + r0.z * r2.z,
                    e12 = r1.x * r2.x + r1.y * r2.y + r1.z * r2.z;
        const float dev = fmaxf(fmaxf(fmaxf(fabsf(e00), fabsf(e11)), fmaxf(fabsf(e22), fabsf(e01))),
                                fmaxf(fabsf(e02), fabsf(e12)));
        const bool ok = (d.kind == PVB_KIND_GRID || (kExt && d.kind != PVB_KIND_MESH)) && (d.flags & PVB_GRID_PRUNE_OK) &&
                        dev < 1e-5f;
        if (!ok) rad = PVB_INF;
        else rad += d.prune_margin;
        sm.sph[ci][s] = make_float4(co.x, co.y, co.z, rad);
    }
    __syncthreads();
    const bool lane_on = lane < ncfg;
    const long long n_tiles = (n_pts + kCmTilePts - 1) / kCmTilePts;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long pt0 = tile * kCmTilePts + warp * kCmPts;
        f3 p[kCmPts];
        bool pon[kCmPts];
#pragma unroll
        for (int k = 0; k < kCmPts; ++k) {
            pon[k] = lane_on && (pt0 + k < n_pts);
            p[k] = (pt0 + k < n_pts) ? load_point(pts, pt0 + k) : mk3(0.f, 0.f, 0.f);
        }
        float best[kCmPts];
        f3 bg[kCmPts];
        int bs[kCmPts];
#pragma unroll
        for (int k = 0; k < kCmPts; ++k) { best[k] = PVB_INF; bg[k] = mk3(0.f, 0.f, 0.f); bs[k] = -1; }
        // One sub-SDF visit for the points of this thread that still need it: transform, AABB bound, lookup
        // (same composed_xform / composed_consider as the point-major kernel: identical arithmetic, identical results)
        auto visit = [&](int s, const bool (&need)[kCmPts]) {
            const pvb_sdf_desc &d = descs.d[s];
            const float4 r0 = sm.xf[lane][3 * s], r1 = sm.xf[lane][3 * s + 1], r2 = sm.xf[lane][3 * s + 2];
#pragma unroll
            for (int k = 0; k < kCmPts; ++k) {
                if (!need[k]) continue;
                composed_consider<false, kExt>(d, st, s, composed_xform(r0, r1, r2, p[k]), 0u, 0ull, best[k], bg[k], bs[k]);
            }
        };
        for (int si = 0; si < n_sdf; ++si) {
            const int s = descs.order[si];
            const float4 sp = sm.sph[lane][s];
            bool need[kCmPts];
            bool any = false;
#pragma unroll
            for (int k = 0; k < kCmPts; ++k) {
                // stage 1: value >= |p - c_obj| - radius - margin (isometry); 0.9998 absorbs the 1e-5 non-rigidity
                const float thr = best[k] + sp.w;
                const float dx = p[k].x - sp.x, dy = p[k].y - sp.y, dz = p[k].z - sp.z;
                const float d2 = dx * dx + dy * dy + dz * dz;
                const bool pruned = bs[k] >= 0 && (thr < 0.f || d2 * 0.9998f > thr * thr);
                need[k] = pon[k] && !pruned;
                any |= need[k];
            }
            if (any) visit(s, need);
        }
        // rotate the winning gradients back (g @ M[:3,:3]) and park the results for the transposed store
#pragma unroll
        for (int k = 0; k < kCmPts; ++k) {
            const int sb = max(bs[k], 0);
            const f3 go = composed_rotate_back(sm.xf[lane][3 * sb], sm.xf[lane][3 * sb + 1], sm.xf[lane][3 * sb + 2], bg[k]);
            sm.out[lane][warp * kCmPts + k] = make_float4(best[k], go.x, go.y, go.z);
            if (out_which) sm.which[lane][warp * kCmPts + k] = bs[k];
        }
        __syncthreads();
        // transposed store: one configuration row (32 consecutive points) per warp instruction
        const long long pt = tile * kCmTilePts + lane;
        if (kMulti && tg.vec && tile * kCmTilePts + kCmTilePts <= n_pts) {
            // Peer destinations are not cached on this side of NVLink, so every store instruction should leave as
            // whole 32-byte sectors: a row is 128 B of values + 384 B of gradients, both contiguous -> lanes 0-7
            // carry the values, lanes 8-31 the gradients, ONE 16-byte store per lane and destination (instead of the
            // strided 4-byte stores of the single-destination path).
            for (int r = warp; r < ncfg; r += kCmWarps) {
                const float *row = reinterpret_cast<const float *>(&sm.out[r][0]);     // {val, gx, gy, gz} per point
                float w[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int e = (lane < 8 ? lane : lane - 8) * 4 + j;       // element of the value / gradient row
                    const int pp = lane < 8 ? e : e / 3;
                    const int cc = lane < 8 ? 0 : 1 + (e - 3 * pp);
                    w[j] = row[4 * pp + cc];
                }
                const float4 v4 = make_float4(w[0], w[1], w[2], w[3]);
                const long long o_row = (long long)(c0 + r) * n_pts + tile * kCmTilePts;
                for (int t = 0; t < tg.n; ++t) {
                    float4 *dst = lane < 8 ? reinterpret_cast<float4 *>(tg.val[t] + o_row) + lane
                                           : reinterpret_cast<float4 *>(tg.grad[t] + 3 * o_row) + (lane - 8);
                    __stcs(dst, v4);
                }
                if (out_which) out_which[o_row + lane] = sm.which[r][lane];
            }
        } else if (pt < n_pts) {
            for (int r = warp; r < ncfg; r += kCmWarps) {
                const float4 v = sm.out[r][lane];
                const long long o_i = (long long)(c0 + r) * n_pts + pt;
                auto emit = [&](float *ov, float *og) {
                    __stcs(ov + o_i, v.x);
                    __stcs(og + 3 * o_i, v.y); __stcs(og + 3 * o_i + 1, v.z); __stcs(og + 3 * o_i + 2, v.w);
                };
                if constexpr (kMulti) {
                    for (int t = 0; t < tg.n; ++t) emit(tg.val[t], tg.grad[t]);
                } else {
                    emit(out_val, out_grad);
                }
                if (out_which) out_which[o_i] = sm.which[r][lane];
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------
// RobotSDF kernel, second generation (round 2): the configuration-major scheme above, specialised to what a
// RobotSDF with cached links is -- every sub-SDF a GRID with the bounding-box out-of-range rule -- and rebuilt around
// what the first profile of composed_cfgmajor_kernel showed: 29 warp-instructions per
// (configuration, point) pair, 142 LDC + 183 MOV in the SASS because the descriptors were indexed with a run-time
// link number, 80 registers (3 CTAs per SM), four scalar stores per pair.
//   * the host passes the descriptors ALREADY in visiting order and the link loop is fully unrolled, so every
//     descriptor field is a constant-bank operand of the instruction that uses it (no LDC, no MOV, no index math);
//   * the transforms and bounding spheres are staged in visiting order as well: shared-memory addresses are
//     lane base + immediate;
//   * results leave through a row-major staging tile ([cfg][32 values], [cfg][96 gradient floats]) written with
//     conflict-free STS.128 and read back as whole 512-byte rows: ONE 16-byte store per lane and destination (lanes
//     0-7 the values, lanes 8-31 the gradients), for the local buffer, for peer buffers (kDest 1) and for a
//     multicast mapping (kDest 2: one multimem.st reaches every GPU of the NVSwitch domain);
//   * the four points of a thread are one 48-byte uniform vector load.
// Arithmetic is composed_xform / composed_aabb_lb2 / grid_eval / composed_rotate_back exactly as in the other two
// composed kernels, so results are bit-identical to them (tests/test_gpu_composed.py).
#ifndef PVB_ROBOT_PTS
#define PVB_ROBOT_PTS 4       // points per thread (4 or 2)
#endif
#ifndef PVB_ROBOT_MINB
#define PVB_ROBOT_MINB 3      // resident CTAs per SM the <= 8-link instantiation is compiled for: 80 registers, no spills (64 registers spill)
#endif
#ifndef PVB_ROBOT_UNROLL
#define PVB_ROBOT_UNROLL 0    // 1: fully unrolled link loop (descriptor fields become immediates, but the 8 x kRbPts inlined
#endif                        // visits overflow the instruction cache)
constexpr int kRbCfg = 32;                        // lanes = configurations
constexpr int kRbWarps = 8;
constexpr int kRbPts = PVB_ROBOT_PTS;             // points per thread
static_assert(kRbPts == 4 || kRbPts == 2, "PVB_ROBOT_PTS must be 2 or 4");
constexpr int kRbTilePts = kRbWarps * kRbPts;     // 32 (16): one output row of a tile
constexpr int kRbValStride = kRbTilePts + 4;      // floats; rows stay 16-byte aligned, vector STS conflict-free
constexpr int kRbGradStride = 3 * kRbTilePts + 4; // floats

template <int MAXS>
struct RobotPack {
    pvb_sdf_desc d[MAXS];       // visiting order
    int orig[MAXS];             // visiting position -> original sub-SDF index (transforms, tie rule, out_which)
    // robot_serial_kernel only (rs_link_consts in pvb_device.cuh): the link-only terms of its bounds, constant bank
    float sph_rad[MAXS];        // bounding-sphere radius + prune_margin; +inf: never rejected; -inf: slot beyond n_sdf
    float visit_margin[MAXS];   // prune_margin, +inf without PVB_GRID_PRUNE_OK: the AABB test then never rejects
};

template <int MAXS>
struct __align__(16) RobotSmem {
    float4 xf[kRbCfg][3 * MAXS + 1];              // row stride = odd number of float4: conflict-free LDS.128
    float4 sph[kRbCfg][MAXS + 1];
    float outv[kRbCfg][kRbValStride];
    float outg[kRbCfg][kRbGradStride];
};

__device__ __forceinline__ void st_mc_v4(float *mc, float4 v) {     // one store, every GPU of the multicast group
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void st_mc_f32(float *mc, float v) {
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc), "f"(v) : "memory");
}

// kDest: 0 = out_val / out_grad, 1 = every (val, grad) pair of tg, 2 = tg.val[0] / tg.grad[0] are multicast addresses
template <int MAXS, bool kUnroll, int kDest>
__global__ void __launch_bounds__(kRbCfg * kRbWarps, kUnroll ? PVB_ROBOT_MINB : 3)
robot_query_kernel(const __grid_constant__ RobotPack<MAXS> pk, int n_sdf, const float *__restrict__ xforms, int n_cfg,
                   int cfg_begin, int cfg_count, const float *__restrict__ pts, int n_pts, int vec,
                   float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_which,
                   const __grid_constant__ OutTargets tg) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RobotSmem<MAXS> &sm = *reinterpret_cast<RobotSmem<MAXS> *>(smem_raw);
    NodeStage st; st.smem = nullptr; st.n = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = blockIdx.y * kRbCfg;                       // first configuration (relative to cfg_begin)
    const int ncfg = min(kRbCfg, cfg_count - c0);
    // ---- stage transforms + object-frame bounding spheres of this configuration tile, in visiting order ----
    for (int item = threadIdx.x; item < kRbCfg * n_sdf; item += blockDim.x) {
        const int ci = item % kRbCfg, si = item / kRbCfg;
        const pvb_sdf_desc &d = pk.d[si];
        float4 r0 = make_float4(1.f, 0.f, 0.f, 0.f), r1 = make_float4(0.f, 1.f, 0.f, 0.f),
               r2 = make_float4(0.f, 0.f, 1.f, 0.f);
        if (ci < ncfg) {
            const float4 *row =
                reinterpret_cast<const float4 *>(xforms + ((size_t)pk.orig[si] * n_cfg + cfg_begin + c0 + ci) * 16);
            r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
        }
        sm.xf[ci][3 * si] = r0; sm.xf[ci][3 * si + 1] = r1; sm.xf[ci][3 * si + 2] = r2;
        // sphere around the link AABB, centre carried to the object frame: c_obj = R^T (c_link - t)
        const f3 cl = mk3(0.5f * (d.bb_min[0] + d.bb_max[0]), 0.5f * (d.bb_min[1] + d.bb_max[1]),
                          0.5f * (d.bb_min[2] + d.bb_max[2]));
        const f3 hl = mk3(0.5f * (d.bb_max[0] - d.bb_min[0]), 0.5f * (d.bb_max[1] - d.bb_min[1]),
                          0.5f * (d.bb_max[2] - d.bb_min[2]));
        const f3 u = mk3(cl.x - r0.w, cl.y - r1.w, cl.z - r2.w);
        const f3 co = mk3(r0.x * u.x + r1.x * u.y + r2.x * u.z, r0.y * u.x + r1.y * u.y + r2.y * u.z,
                          r0.z * u.x + r1.z * u.y + r2.z * u.z);
        float rad = sqrtf(hl.x * hl.x + hl.y * hl.y + hl.z * hl.z) * 1.0001f + 1e-6f;
        // the bound needs an isometry: |R R^T - I| must vanish, otherwise this (cfg, link) never prunes in stage 1
        const float e00 = r0.x * r0.x + r0.y * r0.y + r0.z * r0.z - 1.f, e11 = r1.x * r1.x + r1.y * r1.y + r1.z * r1.z - 1.f,
                    e22 = r2.x * r2.x + r2.y * r2.y + r2.z * r2.z - 1.f;
        const float e01 = r0.x * r1.x + r0.y * r1.y + r0.z * r1.z, e02 = r0.x * r2.x + r0.y * r2.y + r0.z * r2.z,
                    e12 = r1.x * r2.x + r1.y * r2.y + r1.z * r2.z;
        const float dev = fmaxf(fmaxf(fmaxf(fabsf(e00), fabsf(e11)), fmaxf(fabsf(e22), fabsf(e01))),
                                fmaxf(fabsf(e02), fabsf(e12)));
        const bool ok = (d.flags & PVB_GRID_PRUNE_OK) && dev < 1e-5f;
        rad = ok ? rad + d.prune_margin : PVB_INF;
        sm.sph[ci][si] = make_float4(co.x, co.y, co.z, rad);
    }
    __syncthreads();
    const bool lane_on = lane < ncfg;
    const int n_tiles = (n_pts + kRbTilePts - 1) / kRbTilePts;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int pt0 = tile * kRbTilePts + warp * kRbPts;
        const bool full_tile = tile * kRbTilePts + kRbTilePts <= n_pts;
        f3 p[kRbPts];
        // validity of the thread's points as a bit mask (bit k = point pt0 + k exists and this lane has a configuration)
        unsigned on_mask;
        if (vec && full_tile) {           // the thread's points are contiguous and the same for every lane: uniform vector loads
            if constexpr (kRbPts == 4) {
                const float4 *src = reinterpret_cast<const float4 *>(pts + 3 * (size_t)pt0);
                const float4 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2);
                p[0] = mk3(a.x, a.y, a.z); p[1] = mk3(a.w, b.x, b.y); p[2] = mk3(b.z, b.w, c.x); p[3] = mk3(c.y, c.z, c.w);
            } else {
                const float2 *src = reinterpret_cast<const float2 *>(pts + 3 * (size_t)pt0);
                const float2 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2);
                p[0] = mk3(a.x, a.y, b.x); p[1] = mk3(b.y, c.x, c.y);
            }
            on_mask = lane_on ? ((1u << kRbPts) - 1u) : 0u;
        } else {
            on_mask = 0u;
#pragma unroll
            for (int k = 0; k < kRbPts; ++k) {
                const bool in = pt0 + k < n_pts;
                if (lane_on && in) on_mask |= 1u << k;
                p[k] = in ? load_point(pts, pt0 + k) : mk3(0.f, 0.f, 0.f);
            }
        }
        float best[kRbPts];
        f3 bg[kRbPts];
        int bs[kRbPts];
#pragma unroll
        for (int k = 0; k < kRbPts; ++k) { best[k] = PVB_INF; bg[k] = mk3(0.f, 0.f, 0.f); bs[k] = -1; }

        // One link: stage 1 (object-frame bounding sphere against the running minimum, no transform), then for the
        // points that survive: transform, AABB bound, nearest-voxel lookup, running argmin (first index on ties).
        auto link = [&](const int si) {
            const pvb_sdf_desc &d = pk.d[si];
            const int s = pk.orig[si];
            const float4 sp = sm.sph[lane][si];
            unsigned need = 0u;
#pragma unroll
            for (int k = 0; k < kRbPts; ++k) {
                // value >= |p - c_obj| - radius - margin (isometry); 0.9998 absorbs the 1e-5 non-rigidity
                const float thr = best[k] + sp.w;
                const float dx = p[k].x - sp.x, dy = p[k].y - sp.y, dz = p[k].z - sp.z;
                const float d2 = dx * dx + dy * dy + dz * dz;
                const bool pruned = bs[k] >= 0 && (thr < 0.f || d2 * 0.9998f > thr * thr);
                if (!pruned) need |= 1u << k;
            }
            need &= on_mask;
            if (need == 0u) return;
            const float4 r0 = sm.xf[lane][3 * si], r1 = sm.xf[lane][3 * si + 1], r2 = sm.xf[lane][3 * si + 2];
#pragma unroll
            for (int k = 0; k < kRbPts; ++k) {
                if (!(need & (1u << k))) continue;
                const f3 q = composed_xform(r0, r1, r2, p[k]);
                if ((d.flags & PVB_GRID_PRUNE_OK) && bs[k] >= 0) {
                    const float thr = best[k] + d.prune_margin;
                    if (thr < 0.f || composed_aabb_lb2(d, q) > thr * thr) continue;
                }
                const float4 o = robot_lookup(d, q);
                if (bs[k] < 0 || o.x < best[k] || (o.x == best[k] && s < bs[k])) {
                    best[k] = o.x; bg[k] = mk3(o.y, o.z, o.w); bs[k] = s;
                }
            }
        };
        if constexpr (kUnroll && PVB_ROBOT_UNROLL) {
#pragma unroll
            for (int si = 0; si < MAXS; ++si) {
                if (si < n_sdf) link(si);
            }
        } else {
#pragma unroll 1
            for (int si = 0; si < n_sdf; ++si) link(si);
        }
        // ---- winning gradients back to the object frame (g @ M[:3,:3]) ----
        float gout[3 * kRbPts];
#pragma unroll
        for (int k = 0; k < kRbPts; ++k) {
            // visiting position of the winner: the transforms are staged in visiting order
            int sb = 0;
#pragma unroll
            for (int si = 0; si < MAXS; ++si)
                if (si < n_sdf && pk.orig[si] == bs[k]) sb = si;
            const f3 go = composed_rotate_back(sm.xf[lane][3 * sb], sm.xf[lane][3 * sb + 1], sm.xf[lane][3 * sb + 2], bg[k]);
            gout[3 * k] = go.x; gout[3 * k + 1] = go.y; gout[3 * k + 2] = go.z;
        }
        if (out_which) {            // diagnostic output (tests): strided, not on the fast path
#pragma unroll
            for (int k = 0; k < kRbPts; ++k)
                if (on_mask & (1u << k)) out_which[(size_t)(c0 + lane) * n_pts + pt0 + k] = bs[k];
        }
        if constexpr (kDest == 0) {
            // One destination in local memory: every lane owns kRbPts consecutive points of its configuration's row,
            // 16 B of values + 48 B of gradients, and stores them itself -- no staging, no block barrier in the tile
            // loop (the barriers of the staged path cost a large share of the warps' time: warps of a block finish
            // their points at different moments).  The 16-byte pieces of neighbouring warps complete each other's sectors in L2.
            const size_t o = (size_t)(c0 + lane) * n_pts + pt0;
            if (vec && full_tile) {
                if (lane_on) {
                    if constexpr (kRbPts == 4) {
                        __stcs(reinterpret_cast<float4 *>(out_val + o), make_float4(best[0], best[1], best[2], best[3]));
                        float4 *dg = reinterpret_cast<float4 *>(out_grad + 3 * o);
                        __stcs(dg, make_float4(gout[0], gout[1], gout[2], gout[3]));
                        __stcs(dg + 1, make_float4(gout[4], gout[5], gout[6], gout[7]));
                        __stcs(dg + 2, make_float4(gout[8], gout[9], gout[10], gout[11]));
                    } else {
                        __stcs(reinterpret_cast<float2 *>(out_val + o), make_float2(best[0], best[1]));
                        float2 *dg = reinterpret_cast<float2 *>(out_grad + 3 * o);
                        __stcs(dg, make_float2(gout[0], gout[1]));
                        __stcs(dg + 1, make_float2(gout[2], gout[3]));
                        __stcs(dg + 2, make_float2(gout[4], gout[5]));
                    }
                }
            } else {
#pragma unroll
                for (int k = 0; k < kRbPts; ++k) {
                    if (on_mask & (1u << k)) {
                        __stcs(out_val + o + k, best[k]);
                        __stcs(out_grad + 3 * (o + k), gout[3 * k]);
                        __stcs(out_grad + 3 * (o + k) + 1, gout[3 * k + 1]);
                        __stcs(out_grad + 3 * (o + k) + 2, gout[3 * k + 2]);
                    }
                }
            }
            continue;
        }
        // ---- several destinations / multicast: park the thread's values + gradient floats in the row-major staging
        // tile so that every destination receives whole 512-byte rows ----
        if constexpr (kRbPts == 4) {
            *reinterpret_cast<float4 *>(&sm.outv[lane][warp * kRbPts]) = make_float4(best[0], best[1], best[2], best[3]);
            float4 *dg = reinterpret_cast<float4 *>(&sm.outg[lane][3 * warp * kRbPts]);
            dg[0] = make_float4(gout[0], gout[1], gout[2], gout[3]);
            dg[1] = make_float4(gout[4], gout[5], gout[6], gout[7]);
            dg[2] = make_float4(gout[8], gout[9], gout[10], gout[11]);
        } else {
            *reinterpret_cast<float2 *>(&sm.outv[lane][warp * kRbPts]) = make_float2(best[0], best[1]);
            float2 *dg = reinterpret_cast<float2 *>(&sm.outg[lane][3 * warp * kRbPts]);
            dg[0] = make_float2(gout[0], gout[1]);
            dg[1] = make_float2(gout[2], gout[3]);
            dg[2] = make_float2(gout[4], gout[5]);
        }
        __syncthreads();
        if (vec && full_tile) {
            // one configuration row of the tile = kRbTilePts values + 3 * kRbTilePts gradient floats, both contiguous
            // in the output = kRbTilePts 16-byte chunks (the first quarter values, the rest gradients): one 16-byte
            // store per lane and destination, whole sectors; 32 / kRbTilePts rows per warp instruction
            constexpr int kRowsPerInstr = 32 / kRbTilePts;
            const int chunk = lane % kRbTilePts;
            const bool is_val = chunk < kRbTilePts / 4;
            for (int r = warp * kRowsPerInstr + lane / kRbTilePts; r < ncfg; r += kRbWarps * kRowsPerInstr) {
                const float4 v4 = is_val ? *reinterpret_cast<const float4 *>(&sm.outv[r][4 * chunk])
                                         : *reinterpret_cast<const float4 *>(&sm.outg[r][4 * (chunk - kRbTilePts / 4)]);
                const size_t o_row = (size_t)(c0 + r) * n_pts + (size_t)tile * kRbTilePts;
                const size_t off = is_val ? o_row + 4 * chunk : 3 * o_row + 4 * (chunk - kRbTilePts / 4);
                if constexpr (kDest == 0) {
                    __stcs(reinterpret_cast<float4 *>((is_val ? out_val : out_grad) + off), v4);
                } else if constexpr (kDest == 1) {
                    for (int t = 0; t < tg.n; ++t)
                        __stcs(reinterpret_cast<float4 *>((is_val ? tg.val[t] : tg.grad[t]) + off), v4);
                } else {
                    st_mc_v4((is_val ? tg.val[0] : tg.grad[0]) + off, v4);
                }
            }
        } else {
            const int pt = tile * kRbTilePts + lane;
            if (pt < n_pts) {
                for (int r = warp; r < ncfg; r += kRbWarps) {
                    const float v = sm.outv[r][lane];
                    const float gx = sm.outg[r][3 * lane], gy = sm.outg[r][3 * lane + 1], gz = sm.outg[r][3 * lane + 2];
                    const size_t o_i = (size_t)(c0 + r) * n_pts + pt;
                    if constexpr (kDest == 0) {
                        __stcs(out_val + o_i, v);
                        __stcs(out_grad + 3 * o_i, gx); __stcs(out_grad + 3 * o_i + 1, gy); __stcs(out_grad + 3 * o_i + 2, gz);
                    } else if constexpr (kDest == 1) {
                        for (int t = 0; t < tg.n; ++t) {
                            __stcs(tg.val[t] + o_i, v);
                            __stcs(tg.grad[t] + 3 * o_i, gx); __stcs(tg.grad[t] + 3 * o_i + 1, gy);
                            __stcs(tg.grad[t] + 3 * o_i + 2, gz);
                        }
                    } else {
                        st_mc_f32(tg.val[0] + o_i, v);
                        st_mc_f32(tg.grad[0] + 3 * o_i, gx); st_mc_f32(tg.grad[0] + 3 * o_i + 1, gy);
                        st_mc_f32(tg.grad[0] + 3 * o_i + 2, gz);
                    }
                }
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------
// RobotSDF kernel, third generation: point-serial, nearest-sphere-first.
// What the profiles of robot_query_kernel said: most instructions go to link visits, which run for 5.3 of the 8 links
// per (point, 32 configurations) although a lane needs 3.1 -- a fixed visiting order lets the running minimum tighten
// slowly, and "any lane needs it" makes the whole warp pay; the next share goes to the bounding-sphere tests of all
// 8 links x 4 points; 16-byte stores to 32 different rows per instruction load the L1; 80 registers limit the
// resident warps, and gather latency is the top stall.
//   * one point at a time per warp (lanes = 32 configurations), so the state of a point is 8 registers, not 32;
//   * the (configuration, link) bounding spheres sit in shared memory, one LDS.128 per link and point (keeping them in
//     32 registers costs occupancy, see below); per point one pass turns them into lower bounds lb_s <= value_s,
//     kept in 8 registers;
//   * the link with the smallest bound (lane 0's, shuffled: neighbouring configurations agree) is visited FIRST, so
//     the running minimum is tight at once and `lb_s > best` (one compare) rejects most other links for most lanes;
//     ties keep torch.argmin's first-index rule explicitly, so the order never changes a result;
//   * results of 8 consecutive points are parked in a per-WARP staging tile and leave as whole sectors (32 B of
//     values + 96 B of gradients per configuration row), one 16-byte store per lane and destination -- local
//     buffer, peer buffers or multicast -- with __syncwarp only: no block barrier anywhere in the loop.
// Pruning stays exact (bounds are conservative), arithmetic of a visit is unchanged: bit-identical to the other kernels.
// Instruction diet: the nearest sphere from a 5-instruction
// min over keys that carry the link index in their low mantissa bits (was compare + select per link), no per-link tests
// of `point exists` / `si < n_sdf` (slots beyond n_sdf carry a +inf bound), a division-free flush index and per-lane
// staging pointers: 640 -> 557 warp instructions per (point, 32 configurations).  What is left is L1 data-pipe
// wavefronts (~158 per point: 24 sphere-centre reads, ~54 transform rows, ~66 table gathers of 32 distinct sectors,
// 12 staging) and issue slots.
// The link-only terms of the bounds (sphere radius + margin, the visit's margin) sit in the constant bank
// (RobotPack::sph_rad / visit_margin), so the per-lane shared data is the 8 centres alone: 6 LDS.128 per point instead
// of 8, and the visits test no descriptor flags.  Tighter per-lane bounds were modelled on the host
// (scripts/c4_bound_model.py, 64 configurations x 2e4 C4 points, per warp step): the sphere costs 3.39 warp visits,
// 2.13 lookups per lane and 0.48 visits in which no lane passes the exact AABB test; max(sphere, slab of the thinnest
// AABB axis) 3.30 / 2.14 / 0.39; even the exact AABB test itself as the pre-bound 2.90 / 2.11 / 0.  The slab saves
// 0.09 visits (about 1 wavefront and 3 instructions) per point for 8 more dot products and 8 more floats per lane, so
// the bound stays a sphere.
constexpr int kRsWarps = 8;
#ifndef PVB_RS_CHUNK
#define PVB_RS_CHUNK 8
#endif
constexpr int kRsChunk = PVB_RS_CHUNK;            // consecutive points per warp between two flushes (8, or 4: tuning builds)
constexpr int kRsMaxS = 8;
constexpr int kRsValStride = kRsChunk + 1;        // 9: conflict-free STS.32 across lanes
constexpr int kRsGradStride = 3 * kRsChunk + 1;   // 25

// (The lane's 8 bounding spheres kept in 32 registers instead of shared memory -- no LDS in the bound pass, but 80
// registers / 3 CTAs per SM -- is the slower form; so are 48 registers / 5 CTAs with spills and 80 registers without.)
// (More than 4 blocks per SM needs <= 48 registers AND <= 45 KB of shared memory per block, i.e. 4-point staging tiles
// (PVB_RS_CHUNK=4: 35.8 KB); the spills then go through the L1 data pipe that already bounds the kernel.
// PVB_RS_MINB / PVB_RS_CHUNK are build macros so that the choice can be re-measured.)
#ifndef PVB_RS_MINB
#define PVB_RS_MINB 4
#endif

// The configuration tile of the block-level robot-family kernels: per configuration (lane), its transform rows and the
// object-frame centres of its links' bounding spheres.
struct __align__(16) RsTile {
    float4 xf[kRbCfg][3 * kRsMaxS + 1];
    // {x, y, z} of the 8 links back to back: 6 LDS.128 (24 wavefronts) per point instead of one 16-byte record per link
    // (32); + 1 float4: odd row stride, conflict-free
    float4 sph[kRbCfg][3 * kRsMaxS / 4 + 1];
};

// The `link` of rs_swept_pair on staged rows xf (link si at xf[3 si .. 3 si + 2]): rs_link_visit.
template <bool kExt>
__device__ __forceinline__ auto rs_staged_link(const RobotPack<kRsMaxS> &pk, const float4 *xf, const f3 &p) {
    return [&pk, xf, &p](const int si, const float thr, float4 &o) -> bool {
        return rs_link_visit<kExt>(pk.d[si], pk.visit_margin[si], xf[3 * si], xf[3 * si + 1], xf[3 * si + 2], p, thr,
                                   o);
    };
}

// the smallest clearance key over the lanes that differ from this one in lane bits off .. 16 (off a power of two)
__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long k, int off) {
    for (int o = 16; o >= off; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, k, o);
        k = v < k ? v : k;
    }
    return k;
}

// the minimum of v over the warp
__device__ __forceinline__ float warp_min(float v) {
    for (int off = 16; off > 0; off >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

struct __align__(16) RsSmem : RsTile {
    // per-warp staging, LC rows x (8 * 32/LC values + 1) resp. (24 * 32/LC gradient floats + 1): at most 32 x 9 / 32 x 25
    float sv[kRsWarps][kRbCfg][kRsValStride];
    float sg[kRsWarps][kRbCfg][kRsGradStride];
};

// (configuration tiles and the flush index arithmetic: rs_tile / rs_flush_piece in pvb_device.cuh, checked on the CPU tier)
// kExt: some links carry PVB_GRID_TRILINEAR or are analytic primitives (SPHERE / BOX / CYLINDER); each visit then picks
// its evaluation by the link's kind and flag (uniform across the lanes of a point group), so nearest, trilinear and
// primitive links mix.  The bounds are unchanged: they read only bb_min / bb_max, prune_margin and PVB_GRID_PRUNE_OK,
// and prune_margin holds for the interpolant and the primitives as well.  kExt = false is the nearest-voxel kernel as
// it always was.
template <int kDest, bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, PVB_RS_MINB)
robot_serial_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf, const float *__restrict__ xforms,
                    int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, int n_pts, int vec,
                    int chunk_log2, float *__restrict__ out_val, float *__restrict__ out_grad,
                    int *__restrict__ out_which, const __grid_constant__ OutTargets tg) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RsSmem &sm = *reinterpret_cast<RsSmem *>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int c0, lc_log2;
    rs_tile(cfg_count, blockIdx.y, c0, lc_log2);              // first configuration (relative to cfg_begin), log2(lanes per point)
    const int LC = 1 << lc_log2;                              // configurations of this tile = lanes per point group
    const int sub_log2 = 5 - lc_log2, SUB = 1 << sub_log2;    // point groups per warp
    const int cl = lane & (LC - 1), sub = lane >> lc_log2;    // this lane's configuration / point group
    // points per point group between two flushes: 8 (whole 32-byte sectors of values per row), or 4 when the launch has
    // so few steps per resident warp that the serial chain of one step (8 points x ~4 dependent gathers) is the critical
    // path -- the 25-configuration slab of an 8-GPU split
    const int npt = 1 << chunk_log2;                          // points per point group and step (4 or 8)
    const int pts_per_step = npt * SUB;                     // points a warp finishes between two flushes
    const int n_chunks = (n_pts + pts_per_step - 1) / pts_per_step;
    // Blocks stride over the tile's steps; small tiles need fewer blocks than the grid is wide (uniform per block).
    // (Not a balanced persistent schedule -- every warp exactly ceil(total steps / resident warp slots) steps: the
    // cost of a point varies, and many short-lived blocks of an oversubscribed grid let the hardware scheduler even it
    // out.)
    const int gx_tile = min((int)gridDim.x, (n_chunks + kRsWarps - 1) / kRsWarps);
    if ((int)blockIdx.x >= gx_tile) return;
    // ---- stage the transforms of this configuration tile ----
    for (int item = threadIdx.x; item < LC * n_sdf; item += blockDim.x) {
        const int ci = item & (LC - 1), si = item >> lc_log2;
        const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)si * n_cfg + cfg_begin + c0 + ci) * 16);
        sm.xf[ci][3 * si] = __ldg(row); sm.xf[ci][3 * si + 1] = __ldg(row + 1); sm.xf[ci][3 * si + 2] = __ldg(row + 2);
    }
    __syncthreads();
    // ---- bounding-sphere centres (object frame) of every (configuration, link) of the tile (rs_sphere_centre); the
    // radii are per link, in pk.sph_rad.  Slots beyond n_sdf: centre 0 and radius -inf, so that their bound is +inf --
    // never the nearest, never visited ----
    for (int item = threadIdx.x; item < LC * kRsMaxS; item += blockDim.x) {
        const int ci = item & (LC - 1), si = item >> lc_log2;
        const f3 co = si < n_sdf ? rs_sphere_centre(pk.d[si], sm.xf[ci][3 * si], sm.xf[ci][3 * si + 1],
                                                    sm.xf[ci][3 * si + 2])
                                 : mk3(0.f, 0.f, 0.f);
        float *c = reinterpret_cast<float *>(&sm.sph[ci][0]) + 3 * si;
        c[0] = co.x; c[1] = co.y; c[2] = co.z;
    }
    __syncthreads();
    // Staging tile.  One destination in local memory (kDest 0): every warp owns a tile of LC rows x its own
    // pts_per_step points and flushes it alone (__syncwarp only).  Remote destinations (peer buffers, multicast): the 8
    // warps of the block share ONE tile of LC rows x 8 pts_per_step points and flush it together, so that a row leaves
    // as 256 contiguous bytes of values + 768 of gradients -- stores into peer memory are faster in segments of 128
    // bytes and up than in 32- or 64-byte ones (scripts/ubench_peer_store.cu); the two block barriers per step are the
    // price.
    constexpr bool kCoop = kDest != 0;
    constexpr int w_log2 = kCoop ? 3 : 0;                                   // log2(warps sharing a tile)
    float *sv = kCoop ? &sm.sv[0][0][0] : &sm.sv[warp][0][0];
    float *sg = kCoop ? &sm.sg[0][0][0] : &sm.sg[warp][0][0];
    const int row_pts = pts_per_step << w_log2;                             // points per row of the tile
    const int vstride = row_pts + 1, gstride = 3 * row_pts + 1;             // odd: conflict-free STS.32 across lanes
    const int col0 = (kCoop ? warp * pts_per_step : 0) + sub * npt;         // this lane's first column
    const int low3_off = rs_low3_off(n_sdf);   // (bits & ~7) | si is then ONE LOP3 with the immediate si
    float *const sv_lane = sv + cl * vstride + col0, *const sg_lane = sg + cl * gstride + 3 * col0;
    const int n_super = (n_chunks + kRsWarps - 1) / kRsWarps;
    for (int sup = blockIdx.x; sup < n_super; sup += gx_tile) {
        const int chunk = sup * kRsWarps + warp;
        const bool active = chunk < n_chunks;                               // uniform per warp
        const int pt_base = chunk * pts_per_step;
        const int tile_base = kCoop ? sup * kRsWarps * pts_per_step : pt_base;
        const bool full = tile_base + row_pts <= n_pts;                     // every point of the tile exists
#pragma unroll 1
        for (int k = 0; k < (active ? npt : 0); ++k) {
            const int pt = pt_base + sub * npt + k;
            const bool on = pt < n_pts;
            if (!full && !__any_sync(0xffffffffu, on)) break;
            const f3 p = on ? load_point(pts, pt) : mk3(0.f, 0.f, 0.f);     // the same for the LC lanes of a point group
            // ---- lower bounds of every link's value from its bounding sphere (rs_sphere_lb): value_s >= lb_s.
            // radius = inf (bound not valid) gives -inf, a NaN centre (not an isometry) NaN: never rejected.
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[cl], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            // one visiting order per point group: its first lane's nearest sphere (neighbouring configurations agree;
            // rs_nearest in pvb_device.cuh: any link is a valid first visit, the order never changes a result)
            const int pred = __shfl_sync(0xffffffffu, rs_nearest(key, n_sdf), sub << lc_log2);
            float best = PVB_INF;
            f3 bg = mk3(0.f, 0.f, 0.f);
            int bs = -1;
            // one link: transform, AABB bound against the running minimum, nearest-voxel lookup, running argmin.  The
            // first visit (nothing evaluated yet) always looks up and takes the result; every later one has bs >= 0.
            // visit_margin is +inf for a link without PVB_GRID_PRUNE_OK, so the AABB test never rejects it.
            auto visit = [&](const pvb_sdf_desc &d, const int si, const bool first) {
                const float4 r0 = sm.xf[cl][3 * si], r1 = sm.xf[cl][3 * si + 1], r2 = sm.xf[cl][3 * si + 2];
                const f3 q = composed_xform(r0, r1, r2, p);
                if (!first) {
                    const float thr = best + pk.visit_margin[si];
                    if (thr < 0.f || composed_aabb_lb2(d, q) > thr * thr) return;
                }
                // (the three-way choice of rs_link_eval, written out: through the helper, ptxas allocates the kExt
                // instantiations' registers differently)
                const float4 o = (kExt && d.kind != PVB_KIND_GRID)         ? robot_primitive(&d, q.x, q.y, q.z)
                                 : (kExt && (d.flags & PVB_GRID_TRILINEAR)) ? robot_lookup_trilinear(d, q)
                                                                            : robot_lookup(d, q);
                if (first || o.x < best || (o.x == best && si < bs)) {
                    best = o.x; bg = mk3(o.y, o.z, o.w); bs = si;
                }
            };
            // (lanes past the last point work on p = 0 and are not stored: no `on` in the conditions below)
            visit(pk.d[pred], pred, true);
#pragma unroll
            for (int si = 0; si < kRsMaxS; ++si) {
                // reject when the sphere bound already exceeds the running minimum (exact: lb <= value); best is finite
                // after the first visit, so the +inf bound of a slot beyond n_sdf never passes
                if (si != pred && !(lb[si] > best)) visit(pk.d[si], si, false);
            }
            // (Rotating the gradient inside the visit, while the rows are in registers, saves these 3 LDS.128 -- 12 of the
            // ~166 L1 wavefronts a point costs -- but runs the 9 multiply-adds once per visit instead of once per point.)
            const int sb = max(bs, 0);
            const f3 go = composed_rotate_back(sm.xf[cl][3 * sb], sm.xf[cl][3 * sb + 1], sm.xf[cl][3 * sb + 2], bg);
            sv_lane[k] = best;
            sg_lane[3 * k] = go.x;
            sg_lane[3 * k + 1] = go.y;
            sg_lane[3 * k + 2] = go.z;
            if (out_which && on) out_which[(size_t)(c0 + cl) * n_pts + pt] = bs;
        }
        if constexpr (kCoop) __syncthreads(); else __syncwarp();
        // ---- flush: LC configuration rows x (row_pts values | 3 row_pts gradient floats), whole sectors ----
        if (vec && full) {
            // LC * row_pts pieces of 16 B per tile: the first quarter values, the rest gradients; the tile's threads take
            // consecutive pieces (one row segment per warp instruction), npt pieces each
            const int me = kCoop ? (int)threadIdx.x : lane;
            constexpr int kGroup = kCoop ? kRbCfg * kRsWarps : 32;
#pragma unroll 1
            for (int j = 0; j < npt; ++j) {
                bool is_val;
                int row, part;
                rs_flush_piece(me + kGroup * j, chunk_log2, sub_log2, w_log2, is_val, row, part);
                const float *src = is_val ? sv + row * vstride + 4 * part : sg + row * gstride + 4 * part;
                const float4 v4 = make_float4(src[0], src[1], src[2], src[3]);
                const size_t o_row = (size_t)(c0 + row) * n_pts + tile_base;
                const size_t off = is_val ? o_row + 4 * part : 3 * o_row + 4 * part;
                if constexpr (kDest == 0) {
                    __stcs(reinterpret_cast<float4 *>((is_val ? out_val : out_grad) + off), v4);
                } else if constexpr (kDest == 1) {
                    for (int t = 0; t < tg.n; ++t)
                        __stcs(reinterpret_cast<float4 *>((is_val ? tg.val[t] : tg.grad[t]) + off), v4);
                } else {
                    st_mc_v4((is_val ? tg.val[0] : tg.grad[0]) + off, v4);
                }
            }
        } else if (active) {
            for (int k = 0; k < npt; ++k) {
                const int col = col0 + k;
                const int pt = pt_base + sub * npt + k;
                if (pt >= n_pts) break;
                const float v = sv[cl * vstride + col];
                const float gx = sg[cl * gstride + 3 * col], gy = sg[cl * gstride + 3 * col + 1],
                            gz = sg[cl * gstride + 3 * col + 2];
                const size_t o_i = (size_t)(c0 + cl) * n_pts + pt;
                if constexpr (kDest == 0) {
                    __stcs(out_val + o_i, v);
                    __stcs(out_grad + 3 * o_i, gx); __stcs(out_grad + 3 * o_i + 1, gy); __stcs(out_grad + 3 * o_i + 2, gz);
                } else if constexpr (kDest == 1) {
                    for (int t = 0; t < tg.n; ++t) {
                        __stcs(tg.val[t] + o_i, v);
                        __stcs(tg.grad[t] + 3 * o_i, gx); __stcs(tg.grad[t] + 3 * o_i + 1, gy);
                        __stcs(tg.grad[t] + 3 * o_i + 2, gz);
                    }
                } else {
                    st_mc_f32(tg.val[0] + o_i, v);
                    st_mc_f32(tg.grad[0] + 3 * o_i, gx); st_mc_f32(tg.grad[0] + 3 * o_i + 1, gy);
                    st_mc_f32(tg.grad[0] + 3 * o_i + 2, gz);
                }
            }
        }
        if constexpr (kCoop) __syncthreads(); else __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------------------
// Swept query on the sets robot_serial_kernel takes (<= 8 GRID links with the bounding-box rule, nearest or
// trilinear, or primitives): the minimum over the configuration slab at every point (swept_fold, pvb_device.cuh),
// without materialising the cfg_count x n_pts cross product.
//   * A block owns blk_pts consecutive points and walks the slab's configuration tiles (rs_tile) in ascending order.
//     Per tile it stages the transforms and the object-frame sphere centres once, as robot_serial_kernel does, and its
//     point groups (LC lanes = the tile's configurations of one point) take the block's points in turn.
//   * Each point's running result (value, link-frame gradient, configuration, link) stays in shared memory across the
//     tiles.  A lane prunes against the smaller of its own running value and the point's best from earlier tiles
//     (rs_swept_pair): (configuration, link) pairs that cannot beat an earlier configuration are skipped as well.
//   * After the pair, a lexicographic (value, configuration) shuffle reduction within the point group names the
//     tile's winner, which folds itself into the point's result.
//   * The gradient is rotated back once per point, at the end, with the winner's transform: the same
//     composed_rotate_back on the same operands as the per-configuration query.  Outputs are written once per point.
// Transform, bounds, lookups and primitives are those of robot_serial_kernel, so every configuration's candidate is
// its per-configuration result bit for bit whenever it can win.
constexpr int kSwMaxPts = 128;                    // points per block at most (blk_pts: 32, 64 or 128)

struct __align__(16) SwSmem : RsTile {
    SweptBest best[kSwMaxPts];                    // cfg relative to cfg_begin
};

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, PVB_RS_MINB)
robot_swept_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf, const float *__restrict__ xforms,
                   int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, int n_pts, int blk_pts,
                   float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_cfg,
                   int *__restrict__ out_which) {
    __shared__ SwSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long base = (long long)blockIdx.x * blk_pts;
    const int npb = (int)min((long long)blk_pts, (long long)n_pts - base);     // points of this block
    for (int j = threadIdx.x; j < npb; j += blockDim.x) {
        sm.best[j].val = PVB_INF; sm.best[j].cfg = -1;
    }
    const int low3_off = rs_low3_off(n_sdf);
    const int n_tiles = (cfg_count >> 5) + __popc((unsigned)(cfg_count & 31));
    for (int t = 0; t < n_tiles; ++t) {
        int c0, lc_log2;
        rs_tile(cfg_count, t, c0, lc_log2);
        const int LC = 1 << lc_log2, sub_log2 = 5 - lc_log2;
        const int cl = lane & (LC - 1), sub = lane >> lc_log2;
        __syncthreads();                                     // the previous tile's staging is no longer read
        for (int item = threadIdx.x; item < LC * n_sdf; item += blockDim.x) {
            const int ci = item & (LC - 1), si = item >> lc_log2;
            const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)si * n_cfg + cfg_begin + c0 + ci) * 16);
            sm.xf[ci][3 * si] = __ldg(row); sm.xf[ci][3 * si + 1] = __ldg(row + 1); sm.xf[ci][3 * si + 2] = __ldg(row + 2);
        }
        __syncthreads();
        for (int item = threadIdx.x; item < LC * kRsMaxS; item += blockDim.x) {
            const int ci = item & (LC - 1), si = item >> lc_log2;
            const f3 co = si < n_sdf ? rs_sphere_centre(pk.d[si], sm.xf[ci][3 * si], sm.xf[ci][3 * si + 1],
                                                        sm.xf[ci][3 * si + 2])
                                     : mk3(0.f, 0.f, 0.f);
            float *c = reinterpret_cast<float *>(&sm.sph[ci][0]) + 3 * si;
            c[0] = co.x; c[1] = co.y; c[2] = co.z;
        }
        __syncthreads();
        const int groups = kRsWarps << sub_log2;             // point groups of the block
        const int gid = (warp << sub_log2) + sub;
#pragma unroll 1
        for (int j0 = 0; j0 < npb; j0 += groups) {
            const int j = j0 + gid;
            const bool on = j < npb;
            if (!__any_sync(0xffffffffu, on)) break;         // uniform per warp: the warp's groups are all past the end
            const f3 p = on ? load_point(pts, base + j) : mk3(0.f, 0.f, 0.f);
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[cl], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            const int pred = __shfl_sync(0xffffffffu, rs_nearest(key, n_sdf), sub << lc_log2);
            const float bp = on ? sm.best[j].val : PVB_INF;
            auto link = [&](const int si, const float thr, float4 &o) -> bool {
                const pvb_sdf_desc &d = pk.d[si];
                const float4 r0 = sm.xf[cl][3 * si], r1 = sm.xf[cl][3 * si + 1], r2 = sm.xf[cl][3 * si + 2];
                return rs_link_visit<kExt>(d, pk.visit_margin[si], r0, r1, r2, p, thr, o);
            };
            float best;
            f3 bg;
            int bs;
            rs_swept_pair(lb, pred, bp, link, best, bg, bs);
            // the tile's winner for this point: lexicographic (value, configuration) over the LC lanes of the group
            float wv = best;
            int wl = cl;
            for (int off = 1; off < LC; off <<= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, wv, off);
                const int ol = __shfl_xor_sync(0xffffffffu, wl, off);
                if (swept_before(ov, ol, wv, wl)) { wv = ov; wl = ol; }
            }
            if (on && cl == wl) swept_fold(sm.best[j], best, bg, c0 + cl, bs);
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < npb; j += blockDim.x) {
        const SweptBest b = sm.best[j];
        const int cfg = cfg_begin + b.cfg;
        const float4 *row = xf_rows(xforms, n_cfg, max(b.which, 0), cfg);
        const f3 go = composed_rotate_back(__ldg(row), __ldg(row + 1), __ldg(row + 2), b.grad);
        const long long i = base + j;
        out_val[i] = b.val;
        out_grad[3 * i] = go.x; out_grad[3 * i + 1] = go.y; out_grad[3 * i + 2] = go.z;
        if (out_cfg) out_cfg[i] = cfg;
        if (out_which) out_which[i] = b.which;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Clearance query on the sets robot_serial_kernel takes (<= 8 GRID links with the bounding-box rule, nearest or
// trilinear, or primitives): for every configuration of the slab and every segment of seg_len points, the smallest
// clearance_key (pvb_device.cuh) over the segment, left in keys[c * n_seg + b] (~0 on entry); clearance_finish_kernel
// turns it into the result.  Nothing per pair leaves the SM.
//   * Orientation and tiles of robot_serial_kernel: grid row blockIdx.y is configuration tile rs_tile(blockIdx.y), its
//     transforms and sphere centres staged once per block; lanes are the LC configurations of one point, and a warp
//     holds 32 / LC point groups.
//   * Work unit: (tile, chunk), a chunk being `chunk` consecutive points of ONE segment; blocks stride over the chunks.
//     The point groups of the block take the chunk's points in turn.
//   * Each lane keeps its configuration's running key over the points it has seen.  It evaluates a point through
//     rs_swept_pair with bp = min(its running value, the seed): a (point, link) pair is skipped only when a lower bound
//     of its value is STRICTLY above a value that some point of the segment attains, so ties are always evaluated, and
//     a candidate can only be inexact when its value is above bp -- then it loses to the key that attains bp.
//   * Seed: at the start of a chunk each lane reads its (configuration, segment) key from global memory -- the best
//     that earlier blocks have found -- and prunes against its value (a NaN or ~0 key: no pruning).
//   * End of a chunk: the lanes holding the same configuration (the point groups of a warp, then the 8 warps) reduce
//     their keys, and one atomicMin per configuration leaves the block.
struct __align__(16) ClSmem : RsTile {
    unsigned long long red[kRsWarps][kRbCfg];
};

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, PVB_RS_MINB)
robot_clearance_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf, const float *__restrict__ xforms,
                       int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_seg,
                       int seg_len, int chunk, int chunks_per_seg, unsigned long long *__restrict__ keys) {
    __shared__ ClSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int c0, lc_log2;
    rs_tile(cfg_count, blockIdx.y, c0, lc_log2);
    const int LC = 1 << lc_log2, sub_log2 = 5 - lc_log2;
    const int cl = lane & (LC - 1), sub = lane >> lc_log2;
    for (int item = threadIdx.x; item < LC * n_sdf; item += blockDim.x) {
        const int ci = item & (LC - 1), si = item >> lc_log2;
        const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)si * n_cfg + cfg_begin + c0 + ci) * 16);
        sm.xf[ci][3 * si] = __ldg(row); sm.xf[ci][3 * si + 1] = __ldg(row + 1); sm.xf[ci][3 * si + 2] = __ldg(row + 2);
    }
    __syncthreads();
    for (int item = threadIdx.x; item < LC * kRsMaxS; item += blockDim.x) {
        const int ci = item & (LC - 1), si = item >> lc_log2;
        const f3 co = si < n_sdf ? rs_sphere_centre(pk.d[si], sm.xf[ci][3 * si], sm.xf[ci][3 * si + 1],
                                                    sm.xf[ci][3 * si + 2])
                                 : mk3(0.f, 0.f, 0.f);
        float *c = reinterpret_cast<float *>(&sm.sph[ci][0]) + 3 * si;
        c[0] = co.x; c[1] = co.y; c[2] = co.z;
    }
    __syncthreads();
    const int low3_off = rs_low3_off(n_sdf);
    const int groups = kRsWarps << sub_log2;                 // point groups of the block
    const int gid = (warp << sub_log2) + sub;
    const long long n_work = n_seg * chunks_per_seg;
    for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
        const long long b = w / chunks_per_seg;
        const int i0 = (int)(w - b * chunks_per_seg) * chunk;
        const int len = min(chunk, seg_len - i0);
        const long long pt0 = b * seg_len + i0;
        unsigned long long *const kp = keys + (size_t)(c0 + cl) * n_seg + b;
        const unsigned long long seed_key = __ldcg(kp);
        const float seed = clearance_key_value(seed_key);
        unsigned long long run = ~0ull;                      // this lane's running key
        float rv = PVB_INF;                                  // and its value
#pragma unroll 1
        for (int j0 = 0; j0 < len; j0 += groups) {
            const int j = j0 + gid;
            const bool on = j < len;
            if (!__any_sync(0xffffffffu, on)) break;         // uniform per warp: the warp's groups are all past the end
            const f3 p = on ? load_point(pts, pt0 + j) : mk3(0.f, 0.f, 0.f);
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[cl], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            const int pred = __shfl_sync(0xffffffffu, rs_nearest(key, n_sdf), sub << lc_log2);
            const auto link = rs_staged_link<kExt>(pk, sm.xf[cl], p);
            float best;
            f3 bg;
            int bs;
            rs_swept_pair(lb, pred, fminf(rv, seed), link, best, bg, bs);
            if (on && bs >= 0) {
                const unsigned long long k = clearance_key(best, (uint32_t)(i0 + j));
                if (k < run) { run = k; rv = best; }
            }
        }
        // the configuration's minimum over the block: the point groups of this warp, then the warps
        for (int off = LC; off < 32; off <<= 1) {
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, run, off);
            run = o < run ? o : run;
        }
        if (sub == 0) sm.red[warp][cl] = run;
        __syncthreads();
        if (threadIdx.x < LC) {                              // warp 0, point group 0: cl == threadIdx.x
            unsigned long long m = sm.red[0][cl];
            for (int v = 1; v < kRsWarps; ++v) m = sm.red[v][cl] < m ? sm.red[v][cl] : m;
            if (m < seed_key) atomicMin(kp, m);
        }
        __syncthreads();                                     // red is rewritten by the next chunk
    }
}

// ------------------------------------------------------------------------------------------------------------
// Paired clearance query on the sets robot_serial_kernel takes: configuration c against its OWN points, pts
// [cfg_count][n_seg][seg_len][3].  For every configuration of the slab and every segment b of its points, the smallest
// clearance_key over the segment, left in keys[c * n_seg + b] (~0 on entry); paired_clearance_finish_kernel turns it
// into the result.  robot_clearance_kernel cannot serve here: its lanes are the configurations of one shared point.
//   * Work unit: (configuration, segment, chunk of `chunk` consecutive points), owned by one warp.  Units are numbered
//     chunk-major -- unit w is chunk w / (cfg_count * n_seg) of pair w % (cfg_count * n_seg) -- and the warps of a 1-D
//     grid stride over them, so any cfg_count fits, and the later chunks of a segment start after its earlier ones.
//   * The lanes are points of the unit's one configuration: its transform rows and sphere centres are staged once per
//     unit in the warp's slot of shared memory, and every lane reads the same words (broadcasts).
//   * Per lane: the 8 sphere bounds, then rs_swept_pair with the lane's own nearest link first (the visiting order
//     never changes a result) and bp = min(running value, seed), the seed being the pair's key read when the unit
//     starts.  A (point, link) pair is skipped only when its bound is STRICTLY above a value the segment attains.
//   * After every step of 32 points the running value is the minimum over the warp: every lane holds the same
//     configuration and segment, so each prunes against the best point the warp has seen (5 shuffles per step).
//   * End of unit: a warp key minimum, one atomicMin per unit.
// (Measured on the 8-link arm, DESIGN.md §4: a whole block per unit -- shared staging, 8 warps on one chunk -- was 1.2x
// to 3.8x slower, most at 64 points per configuration where 192 of its 256 threads idle; without the per-step warp
// minimum the unit was 1.12-1.27x slower at 4096 x 2048 and 65 536 x 64.)
struct __align__(16) PclSmem {
    float4 xf[kRsWarps][3 * kRsMaxS];
    float4 sph[kRsWarps][3 * kRsMaxS / 4];
};

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, PVB_RS_MINB)
robot_paired_clearance_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf,
                              const float *__restrict__ xforms, int n_cfg, int cfg_begin, int cfg_count,
                              const float *__restrict__ pts, long long n_seg, int seg_len, int chunk, long long n_units,
                              unsigned long long *__restrict__ keys) {
    __shared__ PclSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int low3_off = rs_low3_off(n_sdf);
    const long long pairs = (long long)cfg_count * n_seg;
    // uniform per warp: every lane takes part in the shuffles
    for (long long w = (long long)blockIdx.x * kRsWarps + warp; w < n_units; w += (long long)gridDim.x * kRsWarps) {
        const long long k = w / pairs, cb = w - k * pairs;   // chunk index; c * n_seg + b
        const int cfg = cfg_begin + (int)(cb / n_seg);
        const int i0 = (int)k * chunk;
        const int len = min(chunk, seg_len - i0);
        const long long pt0 = cb * seg_len + i0;             // pts[c][b][i0]
        __syncwarp();                                        // the previous unit's staging is no longer read
        if (lane < 3 * n_sdf) {
            const int si = lane / 3;
            sm.xf[warp][lane] = __ldg(xf_rows(xforms, n_cfg, si, cfg) + (lane - 3 * si));
        }
        __syncwarp();
        if (lane < kRsMaxS) rs_centre_slot(pk.d, lane, n_sdf, sm.xf[warp], sm.sph[warp]);
        __syncwarp();
        unsigned long long *const kp = keys + cb;
        const unsigned long long seed_key = __ldcg(kp);
        const float seed = clearance_key_value(seed_key);
        unsigned long long run = ~0ull;                      // this lane's running key
        float rv = PVB_INF;                                  // the warp's running value
#pragma unroll 1
        for (int j0 = 0; j0 < len; j0 += 32) {
            const int j = j0 + lane;
            const bool on = j < len;
            const f3 p = on ? load_point(pts, pt0 + j) : mk3(0.f, 0.f, 0.f);
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[warp], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            float best;
            f3 bg;
            int bs;
            // lanes past the end prune everything that has a bound (bp = -inf); their result is not used
            rs_swept_pair(lb, rs_nearest(key, n_sdf), on ? fminf(rv, seed) : -PVB_INF,
                          rs_staged_link<kExt>(pk, sm.xf[warp], p), best, bg, bs);
            if (on && bs >= 0) {
                const unsigned long long kk = clearance_key(best, (uint32_t)(i0 + j));
                if (kk < run) { run = kk; rv = best; }
            }
            rv = warp_min(rv);
        }
        run = warp_min_key(run, 1);
        if (lane == 0 && run < seed_key) atomicMin(kp, run);
    }
}

// ------------------------------------------------------------------------------------------------------------
// Self-clearance query on the sets robot_paired_clearance_kernel takes (pvb_device.cuh: self_clearance_key): for every
// configuration of the slab, the smallest self_clearance_key over its sources' link points against their allowed
// sub-SDFs, left in keys[c] (~0 on entry); self_clearance_finish_kernel turns it into the result.
//   * Work unit: (configuration, source sub-SDF i, chunk of `chunk` consecutive link points of i), owned by one warp.
//     Only sources with a non-empty row are numbered (rows.src); units are numbered chunk-major -- unit w is chunk
//     w / (cfg_count * n_src) of (configuration, source) w % (cfg_count * n_src) -- and the warps of a 1-D grid stride
//     over them.
//   * The lanes are link points of the unit's one configuration: its transform rows, W_i's three rows and the sphere
//     centres are staged once per unit in the warp's slot of shared memory.  A lane loads link_pts[i][k] (the same for
//     every configuration: L2-resident) and poses it with composed_xform.
//   * Masked links get a bound of +inf AND are refused inside the visit: rs_swept_pair visits its first link whenever
//     the bound is not strictly above bp, and bp is +inf until a value has been reached.
//   * Pruning, the per-step warp minimum and the one atomicMin per unit are robot_paired_clearance_kernel's, against
//     the configuration's one key: every source prunes against the best value any source of it has reached.
struct SclRows {
    unsigned char src[kRsMaxS];     // the sources with a non-empty row, ascending
    unsigned char mask[kRsMaxS];    // by sub-SDF index: bit j allows (i, j); the diagonal is cleared
};

struct __align__(16) SclSmem {
    float4 xf[kRsWarps][3 * kRsMaxS];
    float4 inv[kRsWarps][4];
    float4 sph[kRsWarps][3 * kRsMaxS / 4];
};

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, PVB_RS_MINB)
robot_self_clearance_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf,
                            const float *__restrict__ xforms, const float *__restrict__ inv_xforms, int n_cfg,
                            int cfg_begin, int cfg_count, const float *__restrict__ link_pts, int K,
                            const __grid_constant__ SclRows rows, int n_src, int chunk, long long n_units,
                            unsigned long long *__restrict__ keys) {
    __shared__ SclSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int low3_off = rs_low3_off(n_sdf);
    const long long pairs = (long long)cfg_count * n_src;
    // uniform per warp: every lane takes part in the shuffles
    for (long long w = (long long)blockIdx.x * kRsWarps + warp; w < n_units; w += (long long)gridDim.x * kRsWarps) {
        const long long kc = w / pairs, r = w - kc * pairs;  // chunk index; c * n_src + source position
        const int c = (int)(r / n_src);
        const int i = rows.src[r - (long long)c * n_src];
        const unsigned mask = rows.mask[i];
        const int cfg = cfg_begin + c;
        const int k0 = (int)kc * chunk;
        const int len = min(chunk, K - k0);
        __syncwarp();                                        // the previous unit's staging is no longer read
        if (lane < 3 * n_sdf) {
            const int si = lane / 3;
            sm.xf[warp][lane] = __ldg(xf_rows(xforms, n_cfg, si, cfg) + (lane - 3 * si));
        } else if (lane >= 3 * kRsMaxS && lane < 3 * kRsMaxS + 3) {
            sm.inv[warp][lane - 3 * kRsMaxS] = __ldg(xf_rows(inv_xforms, n_cfg, i, cfg) + (lane - 3 * kRsMaxS));
        }
        __syncwarp();
        if (lane < kRsMaxS) {
            const f3 co = lane < n_sdf ? rs_sphere_centre(pk.d[lane], sm.xf[warp][3 * lane], sm.xf[warp][3 * lane + 1],
                                                          sm.xf[warp][3 * lane + 2])
                                       : mk3(0.f, 0.f, 0.f);
            float *cc = reinterpret_cast<float *>(&sm.sph[warp][0]) + 3 * lane;
            cc[0] = co.x; cc[1] = co.y; cc[2] = co.z;
        }
        __syncwarp();
        unsigned long long *const kp = keys + c;
        const unsigned long long seed_key = __ldcg(kp);
        const float seed = clearance_key_value(seed_key);
        const float4 w0 = sm.inv[warp][0], w1 = sm.inv[warp][1], w2 = sm.inv[warp][2];
        unsigned long long run = ~0ull;                      // this lane's running key
        float rv = PVB_INF;                                  // the warp's running value
#pragma unroll 1
        for (int j0 = 0; j0 < len; j0 += 32) {
            const int j = j0 + lane;
            const bool on = j < len;
            const f3 p = composed_xform(w0, w1, w2,
                                        on ? load_point(link_pts, (long long)i * K + k0 + j) : mk3(0.f, 0.f, 0.f));
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[warp], pk.sph_rad, p, low3_off, mask, lb, key);
            auto link = [&](const int si, const float thr, float4 &o) -> bool {
                if (!((mask >> si) & 1u)) return false;
                const pvb_sdf_desc &d = pk.d[si];
                const float4 r0 = sm.xf[warp][3 * si], r1 = sm.xf[warp][3 * si + 1], r2 = sm.xf[warp][3 * si + 2];
                return rs_link_visit<kExt>(d, pk.visit_margin[si], r0, r1, r2, p, thr, o);
            };
            float best;
            f3 bg;
            int bs;
            // lanes past the end prune everything that has a bound (bp = -inf) and refuse the rest; unused
            rs_swept_pair(lb, rs_nearest(key, n_sdf), on ? fminf(rv, seed) : -PVB_INF, link, best, bg, bs);
            if (on && bs >= 0) {
                const unsigned long long kk = self_clearance_key(best, i, k0 + j);
                if (kk < run) { run = kk; rv = best; }
            }
            rv = warp_min(rv);
        }
        run = warp_min_key(run, 1);
        if (lane == 0 && run < seed_key) atomicMin(kp, run);
    }
}

// The result of a self-clearance query: one thread per configuration, self_clearance_finish_one (pvb_device.cuh) with
// the visit arithmetic of robot_self_clearance_kernel.  Whichever route produced the key, the output is what the
// composition route's finish (composed_point of the allowed sub-composition at the posed point) gives, bit for bit.
template <bool kExt>
__global__ void __launch_bounds__(kCompThreads)
self_clearance_finish_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf,
                             const float *__restrict__ xforms, const float *__restrict__ inv_xforms, int n_cfg,
                             int cfg_begin, int cfg_count, const float *__restrict__ link_pts, int K,
                             const __grid_constant__ SclRows rows, const unsigned long long *__restrict__ keys,
                             float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_src,
                             int *__restrict__ out_point, int *__restrict__ out_which) {
    const int stride = gridDim.x * blockDim.x;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cfg_count; c += stride) {
        const int cfg = cfg_begin + c;
        auto rows_of = [&](const float *m, int s, float4 &r0, float4 &r1, float4 &r2) {
            const float4 *row = xf_rows(m, n_cfg, s, cfg);
            r0 = __ldg(row); r1 = __ldg(row + 1); r2 = __ldg(row + 2);
        };
        auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { rows_of(xforms, s, r0, r1, r2); };
        auto load_inv = [&](int s, float4 &r0, float4 &r1, float4 &r2) { rows_of(inv_xforms, s, r0, r1, r2); };
        auto load_pt = [&](int i, int k) { return load_point(link_pts, (long long)i * K + k); };
        auto eval = [&](int s, f3 q) { return rs_link_eval<kExt>(pk.d[s], q); };
        const SelfClearanceOut o = self_clearance_finish_one(__ldcg(keys + c), rows.mask, n_sdf, load_xf, load_inv,
                                                             load_pt, eval);
        out_val[c] = o.val;
        out_grad[3 * c] = o.grad.x; out_grad[3 * c + 1] = o.grad.y; out_grad[3 * c + 2] = o.grad.z;
        if (out_src) out_src[c] = o.src;
        if (out_point) out_point[c] = o.point;
        if (out_which) out_which[c] = o.which;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Collision-cost query on the sets robot_serial_kernel takes (pvb_device.cuh: collision_cost_term): for every
// configuration of the slab, every segment and every chunk of the segment (collision_cost_chunk), the chunk's partial
// sums -- cost and the 6 n_sdf twist components -- left in partial[((c * n_seg + b) * chunks_per_seg + kc) * E + e],
// E = 1 + 6 n_sdf (e = 0: cost; 1 + 6 s + k: component k of sub-SDF s).  collision_cost_finish_kernel adds the chunks.
//   * Orientation of robot_clearance_kernel: the lanes are 32 configurations of one shared point, whose transform rows
//     and sphere centres the block stages once per work unit.  Tiles are always 32 configurations wide (tile t starts
//     at slab configuration 32 t; lanes past cfg_count evaluate the slab's last configuration and are never stored),
//     so that no configuration's summation order depends on the slab.
//   * Work unit: (tile, segment, chunk), one block; units are numbered tile-fastest (the tiles of a chunk read the same
//     points) and the blocks of a 1-D grid stride over them.  Warp w takes the chunk's points w, w + 8, ... in order.
//   * A point is skipped by the whole warp when no lane has a link whose sphere bound is below m; otherwise each lane
//     runs rs_swept_pair with bp = m: a link is skipped only when a lower bound of its value is above min(running
//     value, m), so whenever the configuration's value at the point is below m, (d, g, s) is its per-configuration
//     result bit for bit (the gradient rotated back with the winner's rows, as robot_serial_kernel does).
//   * Accumulators: the cost in a register, the twist sums in the lane's column of its warp's slab of shared memory,
//     acc[warp][1 + 6 s + k][lane] (row stride 33: conflict-free for the end-of-unit reads down a column).  8 x 6
//     registers per lane would be the alternative; a contributing lane touches only its argmin link's 6 slots.
//   * End of unit: one thread per (configuration, slot) adds the 8 warps' values in order in fp64 and stores the
//     partial rounded to fp32.  No atomics anywhere: the result does not depend on the grid or on block scheduling.
constexpr int kCcLaneStride = kRbCfg + 1;
// RsTile, then the accumulators: kCcWarps x (1 + 6 n_sdf) rows of kCcLaneStride floats
static int cc_smem_bytes(int n_sdf) {
    return (int)sizeof(RsTile) + kCcWarps * (1 + 6 * n_sdf) * kCcLaneStride * (int)sizeof(float);
}

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kCcWarps, 3)
robot_collision_cost_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf, const float *__restrict__ xforms,
                            int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ pts, long long n_seg,
                            int seg_len, int chunk, int chunks_per_seg, float margin, long long n_units,
                            float *__restrict__ partial) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RsTile &sm = *reinterpret_cast<RsTile *>(smem_raw);
    float *const acc_all = reinterpret_cast<float *>(smem_raw + sizeof(RsTile));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = 1 + 6 * n_sdf;
    float *const acc = acc_all + warp * E * kCcLaneStride + lane;       // this lane's column
    const int n_tiles = (cfg_count + 31) >> 5;
    const int low3_off = rs_low3_off(n_sdf);
    const float m = margin;
    for (long long u = blockIdx.x; u < n_units; u += gridDim.x) {
        const long long sc = u / n_tiles;                               // segment * chunks_per_seg + chunk
        const int c0 = (int)(u - sc * n_tiles) << 5;
        const long long b = sc / chunks_per_seg;
        const int kc = (int)(sc - b * chunks_per_seg);
        const int i0 = kc * chunk;
        const int len = min(chunk, seg_len - i0);
        const long long pt0 = b * seg_len + i0;
        __syncthreads();                                                // the previous unit is no longer read
        for (int item = threadIdx.x; item < kRbCfg * n_sdf; item += blockDim.x) {
            const int ci = item & 31, si = item >> 5;
            const int cfg = cfg_begin + min(c0 + ci, cfg_count - 1);
            const float4 *row = xf_rows(xforms, n_cfg, si, cfg);
            sm.xf[ci][3 * si] = __ldg(row); sm.xf[ci][3 * si + 1] = __ldg(row + 1); sm.xf[ci][3 * si + 2] = __ldg(row + 2);
        }
        for (int e = 0; e < E; ++e) acc[e * kCcLaneStride] = 0.f;
        __syncthreads();
        for (int item = threadIdx.x; item < kRbCfg * kRsMaxS; item += blockDim.x) {
            const int ci = item & 31, si = item >> 5;
            const f3 co = si < n_sdf ? rs_sphere_centre(pk.d[si], sm.xf[ci][3 * si], sm.xf[ci][3 * si + 1],
                                                        sm.xf[ci][3 * si + 2])
                                     : mk3(0.f, 0.f, 0.f);
            float *c = reinterpret_cast<float *>(&sm.sph[ci][0]) + 3 * si;
            c[0] = co.x; c[1] = co.y; c[2] = co.z;
        }
        __syncthreads();
        float cost = 0.f;
#pragma unroll 1
        for (int j = warp; j < len; j += kCcWarps) {                    // uniform per warp
            const f3 p = load_point(pts, pt0 + j);
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[lane], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            if (!__any_sync(0xffffffffu, collision_cost_near(lb, m))) continue;
            const int pred = __shfl_sync(0xffffffffu, rs_nearest(key, n_sdf), 0);
            const auto link = rs_staged_link<kExt>(pk, sm.xf[lane], p);
            float best;
            f3 bg;
            int bs;
            rs_swept_pair(lb, pred, m, link, best, bg, bs);
            if (bs >= 0 && best < m) {
                const f3 g = composed_rotate_back(sm.xf[lane][3 * bs], sm.xf[lane][3 * bs + 1], sm.xf[lane][3 * bs + 2],
                                                  bg);
                const CollisionTerm t = collision_cost_term(m, best, g, p);
                cost += t.cost;
                float *const a = acc + (1 + 6 * bs) * kCcLaneStride;
#pragma unroll
                for (int k = 0; k < 6; ++k) a[k * kCcLaneStride] += t.tw[k];
            }
        }
        acc[0] = cost;
        __syncthreads();
        const int active = min(kRbCfg, cfg_count - c0);
        for (int item = threadIdx.x; item < active * E; item += blockDim.x) {
            const int ci = item / E, e = item - ci * E;
            double s = 0.0;
            for (int w = 0; w < kCcWarps; ++w) s += (double)acc_all[(w * E + e) * kCcLaneStride + ci];
            partial[(((size_t)(c0 + ci) * n_seg + b) * chunks_per_seg + kc) * E + e] = (float)s;
        }
    }
}

// The result of a collision-cost query: one thread per (configuration, segment, slot) adds the chunks' partials in
// order in fp64.  Without chunks (seg_len == 0) every output is 0.
__global__ void __launch_bounds__(kCompThreads)
collision_cost_finish_kernel(const float *__restrict__ partial, long long n_rows, int chunks_per_seg, int E,
                             float *__restrict__ out_cost, float *__restrict__ out_twist) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_rows * E; t += stride) {
        const long long r = t / E;
        const int e = (int)(t - r * E);
        const float *src = partial + (size_t)r * chunks_per_seg * E + e;
        double s = 0.0;
        for (int kc = 0; kc < chunks_per_seg; ++kc) s += (double)__ldg(src + (size_t)kc * E);
        if (e == 0) out_cost[r] = (float)s;
        else out_twist[(size_t)r * (E - 1) + (e - 1)] = (float)s;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Paired collision-cost query on the sets robot_collision_cost_kernel takes: configuration c against its OWN points,
// pts [cfg_count][n_seg][seg_len][3].  The same partials as robot_collision_cost_kernel, in the same layout and with
// the same summation order (pvb_device.cuh: collision_cost_chunk), so that collision_cost_finish_kernel completes them
// and row c * n_seg + b is the shared-cloud kernel's row of configuration cfg_begin + c over points[c], bit for bit.
// robot_collision_cost_kernel cannot serve here: its lanes are the configurations of one shared point.
//   * Work unit: (configuration, segment, chunk), owned by one warp, numbered chunk-major as in
//     robot_paired_clearance_kernel; the warps of a 1-D grid stride over them, so any cfg_count fits.
//   * Staging as robot_paired_clearance_kernel: the configuration's transform rows and sphere centres once per unit in
//     the warp's slot of shared memory, __syncwarp only.
//   * A 32-point step is skipped by the whole warp when no lane has a link whose sphere bound is below m; otherwise
//     each lane runs rs_swept_pair on its own point with its own nearest link first and bp = m, so every (d, g, s)
//     below m is the per-pair query's bit for bit (the visiting order never changes it).
//   * Accumulators: chunk point j belongs to accumulator j mod 8 = lane & 7 (j0 is a multiple of 32), kept in column
//     lane & 7 of the warp's acc[e][8].  Accumulator w must take its points in ascending order, i.e. lanes w, w + 8,
//     w + 16, w + 24 in turn: four ordered sub-steps, lanes 8r .. 8r + 7 adding in sub-step r, __syncwarp between
//     them.  A lane that does not contribute adds nothing, as in robot_collision_cost_kernel.  The terms go in through
//     collision_cost_add: the products fused into the sums as that kernel's compiled code fuses them.
//   * End of unit: lane e adds row e's 8 accumulators in order in fp64 and stores the partial rounded to fp32.  No
//     atomics anywhere.
struct __align__(16) PccSmem {
    float4 xf[kRsWarps][3 * kRsMaxS];
    float4 sph[kRsWarps][3 * kRsMaxS / 4];
    float acc[kRsWarps][1 + 6 * kRsMaxS][kCcWarps];
};

template <bool kExt>
__global__ void __launch_bounds__(kRbCfg * kRsWarps, 3)
robot_paired_collision_cost_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf,
                                   const float *__restrict__ xforms, int n_cfg, int cfg_begin, int cfg_count,
                                   const float *__restrict__ pts, long long n_seg, int seg_len, int chunk,
                                   int chunks_per_seg, float margin, long long n_units, float *__restrict__ partial) {
    __shared__ PccSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int low3_off = rs_low3_off(n_sdf);
    const int E = 1 + 6 * n_sdf;
    const float m = margin;
    const long long pairs = (long long)cfg_count * n_seg;
    float *const acc_all = &sm.acc[warp][0][0];
    float *const acc = acc_all + (lane & (kCcWarps - 1));    // this lane's accumulator column
    // uniform per warp: every lane takes part in the votes and __syncwarp
    for (long long w = (long long)blockIdx.x * kRsWarps + warp; w < n_units; w += (long long)gridDim.x * kRsWarps) {
        const long long kc = w / pairs, cb = w - kc * pairs;  // chunk index; c * n_seg + b
        const int cfg = cfg_begin + (int)(cb / n_seg);
        const int i0 = (int)kc * chunk;
        const int len = min(chunk, seg_len - i0);
        const long long pt0 = cb * seg_len + i0;             // pts[c][b][i0]
        __syncwarp();                                        // the previous unit is no longer read
        if (lane < 3 * n_sdf) {
            const int si = lane / 3;
            sm.xf[warp][lane] = __ldg(xf_rows(xforms, n_cfg, si, cfg) + (lane - 3 * si));
        }
        for (int e = lane; e < E * kCcWarps; e += 32) acc_all[e] = 0.f;
        __syncwarp();
        if (lane < kRsMaxS) {
            const f3 co = lane < n_sdf ? rs_sphere_centre(pk.d[lane], sm.xf[warp][3 * lane], sm.xf[warp][3 * lane + 1],
                                                          sm.xf[warp][3 * lane + 2])
                                       : mk3(0.f, 0.f, 0.f);
            float *c = reinterpret_cast<float *>(&sm.sph[warp][0]) + 3 * lane;
            c[0] = co.x; c[1] = co.y; c[2] = co.z;
        }
        __syncwarp();
#pragma unroll 1
        for (int j0 = 0; j0 < len; j0 += 32) {
            const int j = j0 + lane;
            const bool on = j < len;
            const f3 p = on ? load_point(pts, pt0 + j) : mk3(0.f, 0.f, 0.f);
            float lb[kRsMaxS], key[kRsMaxS];
            rs_point_bounds(sm.sph[warp], pk.sph_rad, p, low3_off, 0xffu, lb, key);
            if (!__any_sync(0xffffffffu, on && collision_cost_near(lb, m))) continue;
            const auto link = rs_staged_link<kExt>(pk, sm.xf[warp], p);
            float best;
            f3 bg;
            int bs;
            // lanes past the end prune everything that has a bound (bp = -inf); their result is not used
            rs_swept_pair(lb, rs_nearest(key, n_sdf), on ? m : -PVB_INF, link, best, bg, bs);
            const bool add = on && bs >= 0 && best < m;
#pragma unroll 1
            for (int r = 0; r < kRbCfg / kCcWarps; ++r) {
                if (lane / kCcWarps == r && add) {
                    const f3 g = composed_rotate_back(sm.xf[warp][3 * bs], sm.xf[warp][3 * bs + 1],
                                                      sm.xf[warp][3 * bs + 2], bg);
                    collision_cost_add(m, best, g, p, acc, acc + (1 + 6 * bs) * kCcWarps, kCcWarps);
                }
                __syncwarp();
            }
        }
        __syncwarp();
        for (int e = lane; e < E; e += 32) {
            double s = 0.0;
            for (int v = 0; v < kCcWarps; ++v) s += (double)acc_all[e * kCcWarps + v];
            partial[((size_t)cb * chunks_per_seg + kc) * E + e] = (float)s;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// Self-collision-cost query on the sets robot_self_clearance_kernel takes (pvb_device.cuh: the definition and the
// summation order): for every configuration of the slab, cost and the 6 n_sdf twist components, stored once each.
//   * Work unit: one configuration, owned by one warp; the warps of a 1-D grid stride over the slab.  No workspace
//     and no finish kernel.
//   * Staging as robot_self_clearance_kernel: the configuration's transform rows and sphere centres once, W_i's three
//     rows once per source (sources with a non-empty row, ascending).  A lane loads link_pts[i][k] and poses it with
//     composed_xform.
//   * A 32-point step is skipped by the whole warp when no lane has an allowed link whose sphere bound is below m;
//     otherwise each lane runs rs_swept_pair with bp = m, so every (d, g, j) below m is the per-point result of the
//     allowed sub-composition bit for bit.  Masked links get a +inf bound and are refused inside the visit.
//   * Accumulators: acc[warp][e][lane] (e = 0: cost; 1 + 6 s + k: component k of sub-SDF s), row stride
//     kCcLaneStride, each lane owning its column; a contributing pair adds collision_cost_term to its target's slots
//     and subtracts it from its source's.  End of configuration: lane e adds row e over the 32 lanes in order in fp64.
//     No atomics anywhere.
constexpr int kSccWarps = 4;
struct __align__(16) SccSmem {
    float4 xf[kSccWarps][3 * kRsMaxS];
    float4 inv[kSccWarps][4];
    float4 sph[kSccWarps][3 * kRsMaxS / 4];
    float acc[kSccWarps][1 + 6 * kRsMaxS][kCcLaneStride];
};

template <bool kExt>
__global__ void __launch_bounds__(kSccLanes * kSccWarps, 8)
robot_self_collision_cost_kernel(const __grid_constant__ RobotPack<kRsMaxS> pk, int n_sdf,
                                 const float *__restrict__ xforms, const float *__restrict__ inv_xforms, int n_cfg,
                                 int cfg_begin, int cfg_count, const float *__restrict__ link_pts, int K,
                                 const __grid_constant__ SclRows rows, int n_src, float margin,
                                 float *__restrict__ out_cost, float *__restrict__ out_twist) {
    __shared__ SccSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int low3_off = rs_low3_off(n_sdf);
    const int E = 1 + 6 * n_sdf;
    const float m = margin;
    float *const acc = &sm.acc[warp][0][lane];                 // this lane's column
    // uniform per warp: every lane takes part in the shuffles
    for (int c = blockIdx.x * kSccWarps + warp; c < cfg_count; c += gridDim.x * kSccWarps) {
        const int cfg = cfg_begin + c;
        __syncwarp();                                        // the previous configuration is no longer read
        if (lane < 3 * n_sdf) {
            const int si = lane / 3;
            sm.xf[warp][lane] = __ldg(xf_rows(xforms, n_cfg, si, cfg) + (lane - 3 * si));
        }
        for (int e = 0; e < E; ++e) acc[e * kCcLaneStride] = 0.f;
        __syncwarp();
        if (lane < kRsMaxS) rs_centre_slot(pk.d, lane, n_sdf, sm.xf[warp], sm.sph[warp]);
#pragma unroll 1
        for (int t = 0; t < n_src; ++t) {
            const int i = rows.src[t];
            const unsigned mask = rows.mask[i];
            __syncwarp();                                    // the previous source's W_i is no longer read
            if (lane < 3)
                sm.inv[warp][lane] = __ldg(xf_rows(inv_xforms, n_cfg, i, cfg) + lane);
            __syncwarp();
            const float4 w0 = sm.inv[warp][0], w1 = sm.inv[warp][1], w2 = sm.inv[warp][2];
            float *const acc_i = acc + (1 + 6 * i) * kCcLaneStride;
#pragma unroll 1
            for (int j0 = 0; j0 < K; j0 += 32) {
                const int k = j0 + lane;
                const bool on = k < K;
                const f3 p = composed_xform(w0, w1, w2,
                                            on ? load_point(link_pts, (long long)i * K + k) : mk3(0.f, 0.f, 0.f));
                float lb[kRsMaxS], key[kRsMaxS];
                rs_point_bounds(sm.sph[warp], pk.sph_rad, p, low3_off, mask, lb, key);
                if (!__any_sync(0xffffffffu, on && collision_cost_near(lb, m))) continue;
                auto link = [&](const int si, const float thr, float4 &o) -> bool {
                    if (!((mask >> si) & 1u)) return false;
                    const pvb_sdf_desc &d = pk.d[si];
                    const float4 r0 = sm.xf[warp][3 * si], r1 = sm.xf[warp][3 * si + 1], r2 = sm.xf[warp][3 * si + 2];
                    return rs_link_visit<kExt>(d, pk.visit_margin[si], r0, r1, r2, p, thr, o);
                };
                float best;
                f3 bg;
                int bs;
                // lanes past the end prune everything that has a bound (bp = -inf) and refuse the rest; unused
                rs_swept_pair(lb, rs_nearest(key, n_sdf), on ? m : -PVB_INF, link, best, bg, bs);
                if (on && bs >= 0 && best < m) {
                    const f3 g = composed_rotate_back(sm.xf[warp][3 * bs], sm.xf[warp][3 * bs + 1],
                                                      sm.xf[warp][3 * bs + 2], bg);
                    const CollisionTerm tm = collision_cost_term(m, best, g, p);
                    acc[0] += tm.cost;
                    float *const acc_j = acc + (1 + 6 * bs) * kCcLaneStride;
#pragma unroll
                    for (int q = 0; q < 6; ++q) {
                        acc_j[q * kCcLaneStride] += tm.tw[q];
                        acc_i[q * kCcLaneStride] -= tm.tw[q];
                    }
                }
            }
        }
        __syncwarp();
        for (int e = lane; e < E; e += 32) {
            double s = 0.0;
            for (int l = 0; l < kSccLanes; ++l) s += (double)sm.acc[warp][e][l];
            if (e == 0) out_cost[c] = (float)s;
            else out_twist[(size_t)c * (E - 1) + (e - 1)] = (float)s;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// Scene queries (pvb_device.cuh: the definition and the summation order): every configuration's link points, posed by
// its W_i, against one static scene of grid (bounding-box rule) or primitive sub-SDFs, evaluated with composed_point
// -- the scene's own one-point sequence.  The robot's sub-SDFs are never evaluated, so their kinds and their number
// (up to kSceneMaxSources) do not matter.
//   * Work unit: one configuration, owned by one block of kSceneWarps warps; the blocks of a 1-D grid stride over the
//     slab.  Warp w takes the sources w, w + kSceneWarps, ... (a source not tested is skipped, or for the cost given
//     a zero row); lane l the points k = l, l + 32, ... of a source, in order.  W_i's three rows are read once per
//     source (the same address for every lane).
//   * The scene's transform rows are the same for every configuration: staged once per block in shared memory.
//   * No atomics, no workspace and no finish kernel: the block's reductions go through shared memory.
constexpr int kSceneWarps = 8;
struct SceneLinks {
    unsigned char on[kSceneMaxSources + 1];     // by source index: tested
};

// Clearance: per-lane running self_clearance_key, the warp minimum, the block minimum in shared memory; thread 0 then
// poses the winning (i, k) again and evaluates the scene there once for the gradient.
template <bool kExt, int MAXS>
__global__ void __launch_bounds__(kSceneLanes * kSceneWarps)
scene_clearance_kernel(const __grid_constant__ DescPack<MAXS> scene, int n_scene, const float *__restrict__ scene_xforms,
                       const float *__restrict__ inv_xforms, int n_sdf, int n_cfg, int cfg_begin, int cfg_count,
                       const float *__restrict__ link_pts, int K, const __grid_constant__ SceneLinks links,
                       float *__restrict__ out_val, float *__restrict__ out_grad, int *__restrict__ out_link,
                       int *__restrict__ out_point) {
    __shared__ float4 sxf[3 * MAXS];
    __shared__ unsigned long long wkey[kSceneWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < 3 * n_scene; t += blockDim.x) sxf[t] = __ldg(xf_rows(scene_xforms, 1, t / 3, 0) + t % 3);
    __syncthreads();
    NodeStage st; st.smem = nullptr; st.n = 0;
    auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { r0 = sxf[3 * s]; r1 = sxf[3 * s + 1]; r2 = sxf[3 * s + 2]; };
    for (int c = blockIdx.x; c < cfg_count; c += gridDim.x) {
        const int cfg = cfg_begin + c;
        unsigned long long run = ~0ull;
        for (int i = warp; i < n_sdf; i += kSceneWarps) {
            if (!links.on[i]) continue;
            const float4 *w = xf_rows(inv_xforms, n_cfg, i, cfg);
            const float4 w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
#pragma unroll 1
            for (int k = lane; k < K; k += 32) {
                const f3 x = composed_xform(w0, w1, w2, load_point(link_pts, (long long)i * K + k));
                const ComposedOut o = composed_point<false, kExt>(scene.d, scene.order, n_scene, load_xf, st, x, 0u,
                                                                  0ull, 0, 0.f);
                const unsigned long long kk = self_clearance_key(o.val, i, k);
                run = kk < run ? kk : run;
            }
        }
        run = warp_min_key(run, 1);
        if (lane == 0) wkey[warp] = run;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long best = wkey[0];
            for (int v = 1; v < kSceneWarps; ++v) best = wkey[v] < best ? wkey[v] : best;
            float val = PVB_INF;
            f3 g = mk3(0.f, 0.f, 0.f);
            int li = -1, pk = -1;
            if (best != ~0ull) {
                li = (int)((uint32_t)best >> 24); pk = (int)((uint32_t)best & 0xffffffu);
                const float4 *w = xf_rows(inv_xforms, n_cfg, li, cfg);
                const f3 x = composed_xform(__ldg(w), __ldg(w + 1), __ldg(w + 2),
                                            load_point(link_pts, (long long)li * K + pk));
                const ComposedOut o = composed_point<false, kExt>(scene.d, scene.order, n_scene, load_xf, st, x, 0u,
                                                                  0ull, 0, 0.f);
                val = o.val; g = o.grad;
            }
            out_val[c] = val;
            out_grad[3 * c] = g.x; out_grad[3 * c + 1] = g.y; out_grad[3 * c + 2] = g.z;
            if (out_link) out_link[c] = li;
            if (out_point) out_point[c] = pk;
        }
        __syncthreads();                                     // wkey is free for the next configuration
    }
}

// Collision cost: per-lane fp32 accumulators (collision_cost_add), a 32-point step skipped by the whole warp when
// scene_near clears every lane's point; at the end of a source the lanes' sums in lane order in fp64 (acc[warp] in
// shared memory, lane e adding row e), the twist row stored and the cost kept in shared memory by source; thread 0
// then adds the sources' costs in order in fp64.
struct __align__(16) SceneCostSmem {
    float acc[kSceneWarps][7][kSceneLanes + 1];
    double cost[kSceneMaxSources + 1];
};

template <bool kExt, int MAXS>
__global__ void __launch_bounds__(kSceneLanes * kSceneWarps)
scene_collision_cost_kernel(const __grid_constant__ DescPack<MAXS> scene, int n_scene,
                            const float *__restrict__ scene_xforms, const float *__restrict__ inv_xforms, int n_sdf,
                            int n_cfg, int cfg_begin, int cfg_count, const float *__restrict__ link_pts, int K,
                            const __grid_constant__ SceneLinks links, float margin, float *__restrict__ out_cost,
                            float *__restrict__ out_twist) {
    __shared__ float4 sxf[3 * MAXS];
    __shared__ SceneCostSmem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float m = margin;
    for (int t = threadIdx.x; t < 3 * n_scene; t += blockDim.x) sxf[t] = __ldg(xf_rows(scene_xforms, 1, t / 3, 0) + t % 3);
    __syncthreads();
    NodeStage st; st.smem = nullptr; st.n = 0;
    auto load_xf = [&](int s, float4 &r0, float4 &r1, float4 &r2) { r0 = sxf[3 * s]; r1 = sxf[3 * s + 1]; r2 = sxf[3 * s + 2]; };
    for (int c = blockIdx.x; c < cfg_count; c += gridDim.x) {
        const int cfg = cfg_begin + c;
        // uniform per warp: every lane takes part in the votes and __syncwarp
        for (int i = warp; i < n_sdf; i += kSceneWarps) {
            float *const row = out_twist + ((size_t)c * n_sdf + i) * 6;
            if (!links.on[i]) {
                if (lane < 6) row[lane] = 0.f;
                if (lane == 0) sm.cost[i] = 0.0;
                continue;
            }
            const float4 *w = xf_rows(inv_xforms, n_cfg, i, cfg);
            const float4 w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
            float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
            for (int j0 = 0; j0 < K; j0 += 32) {
                const int k = j0 + lane;
                const bool on = k < K;
                const f3 x = composed_xform(w0, w1, w2,
                                            on ? load_point(link_pts, (long long)i * K + k) : mk3(0.f, 0.f, 0.f));
                if (!__any_sync(0xffffffffu, on && scene_near(scene.d, n_scene, load_xf, x, m))) continue;
                if (!on) continue;
                const ComposedOut o = composed_point<false, kExt>(scene.d, scene.order, n_scene, load_xf, st, x, 0u,
                                                                  0ull, 0, 0.f);
                if (o.val < m) collision_cost_add(m, o.val, o.grad, x, acc, acc + 1, 1);
            }
#pragma unroll
            for (int e = 0; e < 7; ++e) sm.acc[warp][e][lane] = acc[e];
            __syncwarp();
            if (lane < 7) {
                double s = 0.0;
                for (int l = 0; l < kSceneLanes; ++l) s += (double)sm.acc[warp][lane][l];
                if (lane == 0) sm.cost[i] = s;
                else row[lane - 1] = (float)(0.0 - s);     // twist[a, i] -= tau; +0 when nothing contributed
            }
            __syncwarp();                                    // acc[warp] is free for the warp's next source
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = 0.0;
            for (int i = 0; i < n_sdf; ++i) s += sm.cost[i];
            out_cost[c] = (float)s;
        }
        __syncthreads();                                     // sm.cost is free for the next configuration
    }
}

// ========================================================== voxel containers
// VoxelGrid / ExpandingVoxelGrid / voxel_down_sample (voxel.py:42-171) and the value-range view they sit on
// (TorchMultidimView: sdf.py:264, voxel.py:55-64): the reference reads, writes and lists voxels with boolean-mask
// indexing, nonzero() and index_put on full-size temporaries.  Here: one index kernel (the nearest-cell rule
// round((p - min) / res), evaluated exactly in the dtype torch infers for the range -- fp64 for numpy ranges, fp32
// for Python floats -- half-to-even like torch.round; a cell is valid when every index lies in [0, dim)), a
// scatter-set, a gather, and an ordered stream compaction for "which cells hold something".
struct VoxelGeom {
    double min64[3], res64[3];
    float min32[3], res32[3];
    int dims[3];
    int d;              // 1..3 coordinates per point
    int fp32_mode;
};

__device__ __forceinline__ long long voxel_flat_index(const VoxelGeom &g, const float *__restrict__ p) {
    long long flat = 0;
#pragma unroll 3
    for (int a = 0; a < g.d; ++a) {
        double kf;
        if (g.fp32_mode) kf = (double)rintf(__fdiv_rn(p[a] - g.min32[a], g.res32[a]));
        else kf = rint(__ddiv_rn((double)p[a] - g.min64[a], g.res64[a]));
        if (!(kf >= 0.0 && kf < (double)g.dims[a])) return -1;        // also catches NaN
        flat = flat * g.dims[a] + (long long)kf;
    }
    return flat;
}

__global__ void voxel_index_kernel(const VoxelGeom g, const float *__restrict__ pts, long long n,
                                   long long *__restrict__ out_index) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float p[3] = {0.f, 0.f, 0.f};
        for (int a = 0; a < g.d; ++a) p[a] = __ldg(pts + i * g.d + a);
        out_index[i] = voxel_flat_index(g, p);
    }
}

// data[index(p_i)] = value_i (or the scalar) for the points that fall into the grid.  T = float or unsigned char
// (bool grids).  Duplicate cells: one of the writers wins, as with torch's index_put.
template <typename T>
__global__ void voxel_scatter_kernel(const VoxelGeom g, const float *__restrict__ pts, long long n,
                                     const T *__restrict__ values, T scalar, T *__restrict__ data) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float p[3] = {0.f, 0.f, 0.f};
        for (int a = 0; a < g.d; ++a) p[a] = __ldg(pts + i * g.d + a);
        const long long k = voxel_flat_index(g, p);
        if (k >= 0) data[k] = values ? values[i] : scalar;
    }
}

template <typename T>
__global__ void voxel_gather_kernel(const VoxelGeom g, const float *__restrict__ pts, long long n,
                                    const T *__restrict__ data, T invalid, T *__restrict__ out,
                                    unsigned char *__restrict__ out_valid) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float p[3] = {0.f, 0.f, 0.f};
        for (int a = 0; a < g.d; ++a) p[a] = __ldg(pts + i * g.d + a);
        const long long k = voxel_flat_index(g, p);
        out[i] = k >= 0 ? data[k] : invalid;
        if (out_valid) out_valid[i] = k >= 0;
    }
}

// Ordered compaction of the cells whose content differs from `empty`: (1) per-block counts, (2) exclusive scan of the
// block counts by one block, (3) every block re-evaluates its flags and writes its indices at its offset, in order.
constexpr int kCompactBlock = 1024;          // elements per block (256 threads x 4)

template <typename T>
__global__ void __launch_bounds__(256)
compact_count_kernel(const T *__restrict__ data, long long n, T empty, unsigned int *__restrict__ block_count) {
    __shared__ unsigned int s_cnt[8];
    const long long base = (long long)blockIdx.x * kCompactBlock + threadIdx.x * 4;
    unsigned int c = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (base + j < n && data[base + j] != empty) ++c;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int t = 0;
        for (int w = 0; w < 8; ++w) t += s_cnt[w];
        block_count[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024)
compact_scan_kernel(unsigned int *__restrict__ block_count, long long n_blocks, long long *__restrict__ total) {
    __shared__ unsigned long long s_warp[32];
    __shared__ unsigned long long s_carry;
    if (threadIdx.x == 0) s_carry = 0ull;
    __syncthreads();
    for (long long base = 0; base < n_blocks; base += 1024) {
        const long long i = base + threadIdx.x;
        const unsigned long long v = i < n_blocks ? block_count[i] : 0u;
        unsigned long long incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((threadIdx.x & 31) >= o) incl += t;
        }
        if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
        __syncthreads();
        if (threadIdx.x < 32) {
            unsigned long long w = s_warp[threadIdx.x], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long t = __shfl_up_sync(0xffffffffu, wi, o);
                if (threadIdx.x >= o) wi += t;
            }
            s_warp[threadIdx.x] = wi - w;
        }
        __syncthreads();
        const unsigned long long excl = s_carry + s_warp[threadIdx.x >> 5] + (incl - v);
        if (i < n_blocks) block_count[i] = (unsigned int)excl;       // offsets < 2^32: checked by the caller
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = (long long)s_carry;
}

template <typename T>
__global__ void __launch_bounds__(256)
compact_write_kernel(const T *__restrict__ data, long long n, T empty, const unsigned int *__restrict__ block_offset,
                     long long capacity, long long *__restrict__ out_index) {
    __shared__ unsigned int s_warp[8];
    const long long base = (long long)blockIdx.x * kCompactBlock + threadIdx.x * 4;
    bool f[4];
    unsigned int c = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) { f[j] = base + j < n && data[base + j] != empty; c += f[j]; }
    unsigned int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((threadIdx.x & 31) >= o) incl += t;
    }
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
    __syncthreads();
    unsigned int wbase = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wbase += s_warp[w];
    long long pos = (long long)block_offset[blockIdx.x] + wbase + (incl - c);
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (f[j]) { if (pos < capacity) out_index[pos] = base + j; ++pos; }
}

// ======================================================== forward kinematics
// RobotSDF.set_joint_configuration: the walk is pvb_device.cuh's fk_walk.  A chain (pvb_fk_serial) keeps its plan at
// 32 frames and 16 links; a tree (pvb_fk_tree) takes up to 64 of each and keeps its saved branch poses in shared
// memory, slot-major with one column per thread, sized by the plan's slot count.
using FkSerialPlan = FkPlan<PVB_FK_MAX_FRAMES, PVB_FK_MAX_LINKS>;
using FkTreePlanMax = FkTreePlan<PVB_FK_TREE_MAX_FRAMES, PVB_FK_TREE_MAX_LINKS>;
constexpr int kFkThreads = 64;
// a kernel's parameters may take up to 32764 bytes on sm_70+ with CUDA 12.1 or later; the plan travels by value
static_assert(sizeof(FkTreePlanMax) + 2 * sizeof(void *) + 2 * sizeof(int) <= 32764, "fk_tree_kernel parameters");

__global__ void fk_serial_kernel(const __grid_constant__ FkSerialPlan plan, const float *__restrict__ q, int n_cfg,
                                 int n_joints, float *__restrict__ out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_cfg) return;
    fk_walk<false>(plan, q, n_joints, n_cfg, a, out, nullptr, 0);
}

__global__ void __launch_bounds__(kFkThreads) fk_tree_kernel(const __grid_constant__ FkTreePlanMax plan,
                                                             const float *__restrict__ q, int n_cfg, int n_joints,
                                                             float *__restrict__ out) {
    extern __shared__ float fk_saved_poses[];
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_cfg) return;
    fk_walk<true>(plan, q, n_joints, n_cfg, a, out, fk_saved_poses + threadIdx.x, kFkThreads);
}

// =================================================================== chamfer
// grid = (tiles, transforms).  Each block: transform its points with W_b, unsigned distance (no sign pass: the value
// is squared, chamfer.py:92), sd = scale*d.  Thread t of block k sums fmaf(sd, sd, acc) over the points
// i = k*256 + t, i + stride, ... in that order; the block sums its 8 warps in order into one partial, and
// chamfer_finish_kernel adds the partials in fp64 in a fixed order and divides by N.  Every step of the sum is in a
// fixed order, so the result is a function of the inputs and the grid size only.
// A binned cloud (mesh, >= kSortMinPoints points) is walked in binned order for tree-walk locality, but the order
// within a Morton cell is set by the atomics of sort_scatter_kernel.  So that pass only stores sd (coalesced, at its
// binned position) and chamfer_sum_kernel then sums that scratch through the inverse permutation, with the unbinned
// assignment and order above: binned and unbinned results are equal bit for bit.
constexpr int kChamThreads = 256;
constexpr int kChamSdPass = 4;      // transforms per binned pass: 4 floats per point fit the 16-byte result staging

__device__ __forceinline__ void chamfer_block_partial(float acc, float *s_red, float *partial_slot) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kChamThreads / 32; ++w) s += s_red[w];
        *partial_slot = s;
    }
}

// sorted == nullptr: sums into partial.  Otherwise (binned order): stores sd to sd_out[blockIdx.y * n_pts + j].
__global__ void __launch_bounds__(kChamThreads)
chamfer_partial_kernel(const pvb_sdf_desc obj, const float *__restrict__ w2o, const float *__restrict__ pts,
                       long long n_pts, const float4 *__restrict__ sorted, float scale, int n_stage_max,
                       float *__restrict__ partial, float *__restrict__ sd_out) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar;
    __shared__ float s_red[kChamThreads / 32];
    NodeStage st; st.smem = nullptr; st.n = 0;
    if (obj.kind == PVB_KIND_MESH) st = stage_nodes(obj.nodes, obj.n_nodes, n_stage_max, smem_raw, &bar);
    const float *W = w2o + (size_t)blockIdx.y * 16;
    float xf[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) xf[e] = __ldg(W + e);
    float acc = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_pts; j += stride) {
        long long i = j;
        f3 p;
        if (sorted) {           // binned order, one coalesced 16-byte record per lane
            const float4 sp = __ldg(sorted + j);
            p = mk3(sp.x, sp.y, sp.z);
            i = (long long)__float_as_int(sp.w);
        } else {
            p = load_point(pts, i);
        }
        const f3 q = mk3(fmaf(xf[0], p.x, fmaf(xf[1], p.y, fmaf(xf[2], p.z, xf[3]))),
                         fmaf(xf[4], p.x, fmaf(xf[5], p.y, fmaf(xf[6], p.z, xf[7]))),
                         fmaf(xf[8], p.x, fmaf(xf[9], p.y, fmaf(xf[10], p.z, xf[11]))));
        float d;
        if (obj.kind == PVB_KIND_MESH) {
            const Closest c = bvh_closest(reinterpret_cast<const float4 *>(obj.nodes), st,
                                          reinterpret_cast<const float4 *>(obj.tris), q, PVB_INF);
            const f3 g = c.q - q;
            d = sqrtf(fmaf(g.x, g.x, fmaf(g.y, g.y, g.z * g.z)));
        } else if (obj.kind == PVB_KIND_GRID) {
            d = grid_eval<true>(obj, st, q, PVB_MESH_DEFAULT, (uint64_t)i, nullptr).val;
        } else {
            d = primitive_eval(obj, q).val;
        }
        const float sd = scale * d;
        if (sorted)
            sd_out[(size_t)blockIdx.y * n_pts + j] = sd;
        else
            acc = fmaf(sd, sd, acc);
    }
    if (sorted) return;
    chamfer_block_partial(acc, s_red, partial + (size_t)blockIdx.y * gridDim.x + blockIdx.x);
}

// the unbinned kernel's sum over the scratch of a binned pass (same grid, same assignment and order): point i's sd
// is at its binned position inv[i]
__global__ void __launch_bounds__(kChamThreads)
chamfer_sum_kernel(const float *__restrict__ sd, const uint32_t *__restrict__ inv, long long n_pts,
                   float *__restrict__ partial) {
    __shared__ float s_red[kChamThreads / 32];
    const float *row = sd + (size_t)blockIdx.y * n_pts;
    float acc = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_pts; j += stride) {
        const float s = __ldg(row + __ldg(inv + j));
        acc = fmaf(s, s, acc);
    }
    chamfer_block_partial(acc, s_red, partial + (size_t)blockIdx.y * gridDim.x + blockIdx.x);
}

__global__ void chamfer_finish_kernel(const float *__restrict__ partial, int n_blk, long long n_pts,
                                      float *__restrict__ out) {
    // one warp per transform, fixed summation order
    const int b = blockIdx.x;
    double s = 0.0;
    for (int k = threadIdx.x; k < n_blk; k += 32) s += (double)partial[(size_t)b * n_blk + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[b] = (float)(s / (double)n_pts);
}

// ==================================================================== sample
// Philox4x32-10 counter RNG (Salmon et al. 2011): sample i uses counter (i, 0, 0, 0).
__device__ __forceinline__ void philox_round(uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3, uint32_t k0,
                                             uint32_t k1) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}

__global__ void mesh_sample_kernel(const double *__restrict__ verts, const int *__restrict__ faces, long long n_faces,
                                   const long long *__restrict__ cum, long long n, unsigned long long seed,
                                   double *__restrict__ out_pts, int *__restrict__ out_face) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        // first face whose inclusive cumulative count exceeds i
        long long lo = 0, hi = n_faces - 1;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (cum[mid] > i) hi = mid; else lo = mid + 1;
        }
        const int f = (int)lo;
        uint32_t c0 = (uint32_t)i, c1 = (uint32_t)((unsigned long long)i >> 32), c2 = 0u, c3 = 0u;
        uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
        for (int r = 0; r < 10; ++r) {
            philox_round(c0, c1, c2, c3, k0, k1);
            k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
        }
        const double r1 = ((double)(((unsigned long long)c0 << 21) ^ (unsigned long long)(c1 >> 11)) + 0.5) * (1.0 / 9007199254740992.0);
        const double r2 = ((double)(((unsigned long long)c2 << 21) ^ (unsigned long long)(c3 >> 11)) + 0.5) * (1.0 / 9007199254740992.0);
        const double sr = sqrt(r1);
        const double a = 1.0 - sr, b = sr * (1.0 - r2), c = sr * r2;   // sdf.py:654 (Open3D area-uniform rule)
        const int i0 = faces[3 * (size_t)f], i1 = faces[3 * (size_t)f + 1], i2 = faces[3 * (size_t)f + 2];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            out_pts[3 * i + k] = a * verts[3 * (size_t)i0 + k] + b * verts[3 * (size_t)i1 + k] + c * verts[3 * (size_t)i2 + k];
        if (out_face) out_face[i] = f;
    }
}

// ======================================================== transform points
// out[t] = M_{t / n_pts} applied to pts[t % n_pts]: every transform to every point (the unfused composition).  One
// flat 64-bit index over the n_tf x n_pts pairs, so that no grid dimension bounds the transform count.
__global__ void transform_points_kernel(const float *__restrict__ xforms, const float *__restrict__ pts,
                                        long long n_pts, long long n, float *__restrict__ out) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        long long b, i;
        paired_index(t, n_pts, b, i);
        const float *xf = xforms + b * 16;
        const f3 p = load_point(pts, i);
        float *o = out + 3 * t;
        o[0] = fmaf(xf[0], p.x, fmaf(xf[1], p.y, fmaf(xf[2], p.z, xf[3])));
        o[1] = fmaf(xf[4], p.x, fmaf(xf[5], p.y, fmaf(xf[6], p.z, xf[7])));
        o[2] = fmaf(xf[8], p.x, fmaf(xf[9], p.y, fmaf(xf[10], p.z, xf[11])));
    }
}

// out[t] = M_{t / n_pts} applied to pts[t]: every transform to its own n_pts points (the unfused paired composition),
// with the arithmetic of composed_xform so that the sub-frame points equal what the fused kernels compute
__global__ void transform_points_paired_kernel(const float *__restrict__ xforms, const float *__restrict__ pts,
                                               long long n_pts, long long n, float *__restrict__ out) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        long long b, i;
        paired_index(t, n_pts, b, i);
        const float4 *row = reinterpret_cast<const float4 *>(xforms + b * 16);
        const f3 q = composed_xform(__ldg(row), __ldg(row + 1), __ldg(row + 2), load_point(pts, t));
        out[3 * t] = q.x; out[3 * t + 1] = q.y; out[3 * t + 2] = q.z;
    }
}

static int grid_for(long long work_items, int threads, int blocks_per_sm) {
    const long long want = (work_items + threads - 1) / threads;
    const long long cap = (long long)sm_count() * blocks_per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

// shared-memory budget for the staged top of the tree (PVB_STAGE_NODES overrides, for tuning)
constexpr int kStageNodesMax = 1536;   // 192 KB
static int stage_nodes_for(int n_nodes) {
    static int max_nodes = -1;
    if (max_nodes < 0) {
        // Shared memory taken from the SM's unified 256 KB L1 / shared array (up to 228 KB of it shared on H100) is L1
        // taken away from the triangles, the deeper nodes and the traversal stacks,
        // and the top of the tree is an L1 hit anyway; the bulk-copy staging path is kept (PVB_STAGE_NODES) but off.
        max_nodes = 0;
        if (const char *e = getenv("PVB_STAGE_NODES")) {
            const int v = atoi(e);
            if (v >= 0 && v <= kStageNodesMax) max_nodes = v;
        }
    }
    return n_nodes < max_nodes ? n_nodes : max_nodes;
}


}  // namespace pvb

using namespace pvb;

// ======================================================================= ABI
extern "C" int pvb_timing_enable(int on) {
    g_timing = on ? 1 : 0;
    return PVB_OK;
}

extern "C" int pvb_timing_last_ms(float *ms) {
    if (!ms) { pvb_set_error("pvb_timing_last_ms: null argument"); return PVB_ERR_INVALID; }
    const int dev = current_device();
    if (!g_ev_ok[dev] || !g_ev_set[dev]) {
        pvb_set_error("pvb_timing_last_ms: no timed launch on device %d (call pvb_timing_enable(1) first)", dev);
        return PVB_ERR_INVALID;
    }
    if (cudaEventSynchronize(g_ev[dev][1]) != cudaSuccess ||
        cudaEventElapsedTime(ms, g_ev[dev][0], g_ev[dev][1]) != cudaSuccess) {
        pvb_set_error("pvb_timing_last_ms: %s", cudaGetErrorString(cudaGetLastError()));
        return PVB_ERR_CUDA;
    }
    return PVB_OK;
}

static int check_mesh(const pvb_sdf_desc *m, const char *who) {
    if (!m->nodes || !m->tris || m->n_nodes < 1 || m->n_tris < 1) {
        pvb_set_error("%s: mesh part of the descriptor is empty", who);
        return PVB_ERR_INVALID;
    }
    return PVB_OK;
}

// Bins `n` points (optionally seen through the rigid transform xf_dev) over the padded AABB of `obj`; returns the
// binned records / inverse permutation / result staging inside `workspace`, or all-null when the batch is small / no
// workspace was given.
static SortedQueries sort_queries(const pvb_sdf_desc *obj, const float *pts, long long n, const float *xf_dev,
                                  void *workspace, size_t workspace_bytes, cudaStream_t stream, int *rc) {
    *rc = PVB_OK;
    SortedQueries sq{nullptr, nullptr, nullptr};
    static const int enabled = [] { const char *e = getenv("PVB_SORT_QUERIES"); return e ? atoi(e) : 1; }();
    // (the scan moves the counters as uint4: an unaligned scratch pointer simply means no binning)
    if (!enabled || !workspace || ((uintptr_t)workspace & 15) || n < kSortMinPoints || n >= (1ll << 31) ||
        workspace_bytes < sort_workspace_bytes(n))
        return sq;
    uint32_t *hist = reinterpret_cast<uint32_t *>(workspace);
    const int bits = sort_bits_for(n);
    const size_t n_cells = (size_t)1 << (3 * bits);
    uint32_t *cell = hist + n_cells;
    const size_t n4 = ((size_t)n * 4 + 15) / 16 * 16;
    float4 *sorted = reinterpret_cast<float4 *>(reinterpret_cast<unsigned char *>(cell) + n4);
    float4 *stage = sorted + n;
    SortFrame f;
    for (int a = 0; a < 3; ++a) {
        const float ext = obj->bb_max[a] - obj->bb_min[a];
        // queries beyond the padded box clamp to the border cells.  Mesh queries may lie anywhere around the object
        // (pad = half its extent); a chamfer cloud hugs the surface (xf_dev given): a tenth keeps the cells 1.7x finer
        const float pad = (xf_dev ? 0.1f : 0.5f) * ext + 1e-6f;
        f.lo[a] = obj->bb_min[a] - pad;
        f.scale[a] = (float)(1 << bits) / (ext + 2.f * pad);
    }
    f.use_xf = xf_dev != nullptr;
    f.bits = bits;
    for (int e = 0; e < 12; ++e) f.xf[e] = 0.f;
    if (cudaMemsetAsync(hist, 0, n_cells * 4, stream) != cudaSuccess) {
        pvb_set_error("sort_queries: cudaMemsetAsync failed");
        *rc = PVB_ERR_CUDA;
        return sq;
    }
    const int blocks = grid_for(n, 256, 8);
    sort_hist_kernel<<<blocks, 256, 0, stream>>>(f, pts, n, xf_dev, cell, hist);
    sort_scan_kernel<<<1, 1024, 0, stream>>>(hist, (int)n_cells);
    sort_scatter_kernel<<<blocks, 256, 0, stream>>>(cell, pts, n, hist, sorted);
    if (cudaGetLastError() != cudaSuccess) {
        pvb_set_error("sort_queries: launch failed");
        *rc = PVB_ERR_CUDA;
        return sq;
    }
    sq.sorted = sorted;
    sq.inv = cell;
    sq.stage = stage;
    return sq;
}

extern "C" int64_t pvb_query_workspace(int64_t n) {
    return n >= kSortMinPoints ? (int64_t)sort_workspace_bytes(n) : 0;
}

extern "C" int pvb_mesh_query(const pvb_sdf_desc *mesh, const float *pts, int64_t n, uint32_t mode, float *out_dist,
                              float *out_grad, float *out_closest, int32_t *out_face, float *out_normal,
                              void *workspace, int64_t workspace_bytes, void *stream) {
    if (!mesh || n < 0 || (n > 0 && (!pts || !out_dist || !out_grad))) {
        pvb_set_error("pvb_mesh_query: null argument");
        return PVB_ERR_INVALID;
    }
    if (int rc = check_mesh(mesh, "pvb_mesh_query")) return rc;
    if ((mode & PVB_MESH_SURFACE_NORMAL) && !mesh->face_normals) {
        pvb_set_error("pvb_mesh_query: face_normals required for PVB_MESH_SURFACE_NORMAL");
        return PVB_ERR_INVALID;
    }
    if (out_normal && !mesh->face_normals) {
        pvb_set_error("pvb_mesh_query: face_normals required for out_normal");
        return PVB_ERR_INVALID;
    }
    if (n == 0) return PVB_OK;
    const int n_stage = stage_nodes_for(mesh->n_nodes);
    const size_t smem = (size_t)n_stage * 128;
    if (!ensure_smem(mesh_query_kernel, kSlotMesh, kStageNodesMax * 128)) {
        pvb_set_error("pvb_mesh_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
        return PVB_ERR_CUDA;
    }
    int rc = PVB_OK;
    const SortedQueries sq = sort_queries(mesh, pts, n, nullptr, workspace,
                                          (size_t)(workspace_bytes < 0 ? 0 : workspace_bytes), (cudaStream_t)stream, &rc);
    if (rc != PVB_OK) return rc;
    // run length (PVB_MESH_RUN, default 1): the tighter start radius of a run does not pay for lanes being `run`
    // queries apart.
    static const int run_max = [] { const char *e = getenv("PVB_MESH_RUN"); return e ? atoi(e) : 1; }();
    long long run = n / ((long long)sm_count() * 2048);
    run = run < 1 ? 1 : (run > run_max ? run_max : run);
    const int blocks = grid_for((n + run - 1) / run, kMeshThreads, 8);
    const bool winding = (mode & PVB_MESH_WINDING) && (mode & PVB_MESH_SIGNED);
    if (winding && (!mesh->wn_nodes || !out_face)) {
        pvb_set_error("pvb_mesh_query: PVB_MESH_WINDING needs pvb_sdf_desc.wn_nodes and an out_face buffer");
        return PVB_ERR_INVALID;
    }
    // winding mode: unsigned first pass (distance >= 0, gradient away from the surface), sign in a second pass
    const uint32_t walk_mode = winding ? 0u : (mode & ~(uint32_t)PVB_MESH_WINDING);
    timing_mark(0, (cudaStream_t)stream);
    mesh_query_kernel<<<blocks, kMeshThreads, smem, (cudaStream_t)stream>>>(*mesh, pts, n, sq.sorted, sq.stage, (int)run,
                                                                            walk_mode, n_stage, out_dist, out_grad,
                                                                            out_closest, out_face, out_normal);
    timing_mark(1, (cudaStream_t)stream);
    PVB_CHECK_LAUNCH("pvb_mesh_query");
    if (winding) {
        mesh_winding_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(*mesh, pts, n, sq.sorted, sq.stage, mode,
                                                                                  out_dist, out_grad, out_face);
        PVB_CHECK_LAUNCH("pvb_mesh_query(winding)");
    }
    if (sq.stage) {
        unpermute_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(sq.inv, sq.stage, n, out_dist, out_grad);
        PVB_CHECK_LAUNCH("pvb_mesh_query(unpermute)");
    }
    return PVB_OK;
}

extern "C" int pvb_grid_lookup(const pvb_sdf_desc *grid, const float *pts, int64_t n, float *out_val, float *out_grad,
                               uint8_t *out_outside, float surface_level, int64_t *out_index, void *stream) {
    if (!grid || n < 0 || (n > 0 && !pts)) {
        pvb_set_error("pvb_grid_lookup: null argument");
        return PVB_ERR_INVALID;
    }
    if (!grid->table || grid->dims[0] < 1 || grid->dims[1] < 1 || grid->dims[2] < 1) {
        pvb_set_error("pvb_grid_lookup: grid part of the descriptor is empty");
        return PVB_ERR_INVALID;
    }
    if ((long long)grid->dims[0] * grid->dims[1] * grid->dims[2] >= (1ll << 31)) {
        pvb_set_error("pvb_grid_lookup: more than 2^31 voxels");
        return PVB_ERR_INVALID;
    }
    if (grid->flags & PVB_GRID_OOB_GT)
        if (int rc = check_mesh(grid, "pvb_grid_lookup(LOOKUP_GT_SDF)")) return rc;
    if (n == 0) return PVB_OK;
    const uint32_t mesh_mode = PVB_MESH_DEFAULT;
    const bool gt = (grid->flags & PVB_GRID_OOB_GT) != 0;
    if (grid->flags & PVB_GRID_TRILINEAR) {
        if (gt || out_outside || out_index || !out_val || !out_grad) {
            pvb_set_error("pvb_grid_lookup: PVB_GRID_TRILINEAR supports value + gradient output with the AABB rule only");
            return PVB_ERR_INVALID;
        }
        grid_trilinear_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(*grid, pts, n, out_val, out_grad);
        PVB_CHECK_LAUNCH("pvb_grid_lookup(trilinear)");
        return PVB_OK;
    }
    auto aligned = [](const void *p, size_t a) { return p == nullptr || ((uintptr_t)p % a) == 0; };
    const bool vec_ok = aligned(pts, 16) && aligned(out_val, 16) && aligned(out_grad, 16) && aligned(out_outside, 4) &&
                        aligned(out_index, 16);
    long long n_quads = vec_ok ? n / 4 : 0;
    static const int use_tma = [] { const char *e = getenv("PVB_GRID_TMA"); return e ? atoi(e) : 1; }();
    if (use_tma && n_quads >= 4 * kTmaTile && !gt && out_val && out_grad && !out_outside && !out_index) {
        if (!ensure_smem(grid_lookup_tma_kernel, kSlotGridTma, (int)sizeof(GridTmaSmem))) {
            pvb_set_error("pvb_grid_lookup: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
            return PVB_ERR_CUDA;
        }
        static const int ctas_per_sm = [] { const char *e = getenv("PVB_GRID_TMA_CTAS"); return e ? atoi(e) : 3; }();
        const long long n_tiles = (4 * n_quads + kTmaTile - 1) / kTmaTile;
        const long long cap = (long long)sm_count() * ctas_per_sm;
        const int blocks = (int)(n_tiles < cap ? n_tiles : cap);
        timing_mark(0, (cudaStream_t)stream);
        grid_lookup_tma_kernel<<<blocks, kTmaThreads, sizeof(GridTmaSmem), (cudaStream_t)stream>>>(
            *grid, pts, 4 * n_quads, out_val, out_grad);
        timing_mark(1, (cudaStream_t)stream);
        PVB_CHECK_LAUNCH("pvb_grid_lookup(tma)");
    } else if (n_quads > 0) {
        const int blocks = grid_for(n_quads, kGridThreads, 8);
        auto kern = gt ? grid_lookup_vec4_kernel<true> : grid_lookup_vec4_kernel<false>;
        timing_mark(0, (cudaStream_t)stream);
        kern<<<blocks, kGridThreads, 0, (cudaStream_t)stream>>>(
            *grid, reinterpret_cast<const float4 *>(pts), n_quads, mesh_mode, reinterpret_cast<float4 *>(out_val),
            reinterpret_cast<float4 *>(out_grad), reinterpret_cast<uchar4 *>(out_outside), surface_level,
            reinterpret_cast<longlong2 *>(out_index));
        timing_mark(1, (cudaStream_t)stream);
        PVB_CHECK_LAUNCH("pvb_grid_lookup(vec4)");
    }
    const long long first = 4 * n_quads;
    if (first < n) {
        const int blocks = grid_for(n - first, kGridThreads, 8);
        auto kern = gt ? grid_lookup_scalar_kernel<true> : grid_lookup_scalar_kernel<false>;
        kern<<<blocks, kGridThreads, 0, (cudaStream_t)stream>>>(
            *grid, pts, first, n, mesh_mode, out_val, out_grad, out_outside, surface_level, (long long *)out_index);
        PVB_CHECK_LAUNCH("pvb_grid_lookup(scalar)");
    }
    return PVB_OK;
}

extern "C" int pvb_sphere_query(float radius, const float *pts, int64_t n, float *out_val, float *out_grad,
                                void *stream) {
    if (n < 0 || (n > 0 && (!pts || !out_val || !out_grad))) {
        pvb_set_error("pvb_sphere_query: null argument");
        return PVB_ERR_INVALID;
    }
    if (n == 0) return PVB_OK;
    sphere_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(radius, pts, n, out_val, out_grad);
    PVB_CHECK_LAUNCH("pvb_sphere_query");
    return PVB_OK;
}

// The sub-SDFs of the generic composed kernels in their visiting order (fill_order).
template <int MAXS>
static DescPack<MAXS> desc_pack(const pvb_sdf_desc *descs, int n_sdf) {
    DescPack<MAXS> pack;
    memcpy(pack.d, descs, sizeof(pvb_sdf_desc) * (size_t)n_sdf);
    fill_order(pack, n_sdf);
    return pack;
}

// The scalar arguments every generic composed kernel takes after its outputs: whether mesh sub-SDFs are evaluated
// nearest-bound-first (PVB_COMP_NEAREST_FIRST=0 restores the fixed bit-reversed order) and the largest prune margin.
struct CompConsts {
    int nearest_first;
    float margin_max;
};

static CompConsts comp_consts(const pvb_sdf_desc *descs, int n_sdf) {
    static const int nearest_first = [] { const char *e = getenv("PVB_COMP_NEAREST_FIRST"); return e ? atoi(e) : 1; }();
    float margin_max = 0.f;
    for (int i = 0; i < n_sdf; ++i) margin_max = descs[i].prune_margin > margin_max ? descs[i].prune_margin : margin_max;
    return {nearest_first, margin_max};
}

// Calls f(kMesh, kExt, kMaxS), std::bool_constant / std::integral_constant values naming the instantiation of the
// generic composed kernels that serves the set: with mesh sub-SDFs or not, with trilinear or primitive sub-SDFs or
// not, and room for 16 or 128 sub-SDFs.
template <typename F>
static int comp_variant(bool mesh, bool ext, int n_sdf, F &&f) {
    auto by_maxs = [&](auto kMesh, auto kExt) {
        return n_sdf <= 16 ? f(kMesh, kExt, std::integral_constant<int, 16>{})
                           : f(kMesh, kExt, std::integral_constant<int, 128>{});
    };
    auto by_ext = [&](auto kMesh) { return ext ? by_maxs(kMesh, std::true_type{}) : by_maxs(kMesh, std::false_type{}); };
    return mesh ? by_ext(std::true_type{}) : by_ext(std::false_type{});
}

template <bool kMesh, int PTS, int MAXS, bool kExt>
static int launch_composed(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                           int cfg_count, const float *pts, long long n_pts, uint32_t mesh_mode, float *out_val,
                           float *out_grad, int *out_which, const OutTargets *tg, cudaStream_t stream) {
    const long long n_items = n_pts / PTS;
    if (n_items <= 0) return PVB_OK;
    const DescPack<MAXS> pack = desc_pack<MAXS>(descs, n_sdf);
    const CompConsts c = comp_consts(descs, n_sdf);
    const int gx = grid_for(n_items, kCompThreads, 8);
    int gy = cfg_count < 65535 ? cfg_count : 65535;
    const long long cap = (long long)sm_count() * 64;     // bound the block count for huge configuration batches
    if ((long long)gx * gy > cap) { gy = (int)(cap / gx); if (gy < 1) gy = 1; }
    dim3 grid((unsigned)gx, (unsigned)gy);
    auto k = tg ? composed_query_kernel<kMesh, PTS, MAXS, true, kExt>
                : composed_query_kernel<kMesh, PTS, MAXS, false, kExt>;
    timing_mark(0, stream);
    k<<<grid, kCompThreads, 0, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, 0, n_pts, mesh_mode,
                                         tg ? nullptr : out_val, tg ? nullptr : out_grad, out_which,
                                         tg ? *tg : OutTargets{}, c.nearest_first, c.margin_max);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query");
    return PVB_OK;
}

// Waves of resident blocks the point-form robot kernels aim their grid at.
static int robot_waves() {
    static const int waves = [] { const char *e = getenv("PVB_ROBOT_WAVES"); return e ? atoi(e) : 4; }();
    return waves;
}

// Launch robot_query_kernel (all sub-SDFs GRID with the bounding-box rule, <= 16 of them).
template <int MAXS, bool kUnroll>
static int launch_robot(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                        int cfg_count, const float *pts, long long n_pts, int vec, float *out_val, float *out_grad,
                        int *out_which, const OutTargets *tg, cudaStream_t stream) {
    RobotPack<MAXS> pack;
    memset(&pack, 0, sizeof(pack));
    DescPack<MAXS> order;               // only its visiting order is used
    fill_order(order, n_sdf);
    for (int si = 0; si < n_sdf; ++si) {
        pack.d[si] = descs[order.order[si]];
        pack.orig[si] = order.order[si];
    }
    for (int si = n_sdf; si < MAXS; ++si) pack.orig[si] = -1;
    const int kind = !tg ? 0 : (tg->mc ? 2 : 1);
    decltype(&robot_query_kernel<MAXS, kUnroll, 0>) const ks[3] = {
        robot_query_kernel<MAXS, kUnroll, 0>, robot_query_kernel<MAXS, kUnroll, 1>, robot_query_kernel<MAXS, kUnroll, 2>};
    const int smem = (int)sizeof(RobotSmem<MAXS>);
    const int slot0 = kUnroll ? kSlotRobot : kSlotRobotWide;
    for (int d = 0; d < 3; ++d)
        if (!ensure_smem(ks[d], slot0 + d, smem)) {
            pvb_set_error("pvb_composed_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
            return PVB_ERR_CUDA;
        }
    const int gy = (cfg_count + kRbCfg - 1) / kRbCfg;
    const long long n_tiles = (n_pts + kRbTilePts - 1) / kRbTilePts;
    long long gx = ((long long)sm_count() * (kUnroll ? 4 : 3) * robot_waves() + gy - 1) / gy;
    if (gx > n_tiles) gx = n_tiles;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, (unsigned)gy);
    timing_mark(0, stream);
    ks[kind]<<<grid, kRbCfg * kRbWarps, smem, stream>>>(
        pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts, vec, tg ? nullptr : out_val,
        tg ? nullptr : out_grad, out_which, tg ? *tg : OutTargets{});
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query(robot)");
    return PVB_OK;
}

// Launch robot_serial_kernel (<= 8 GRID sub-SDFs with the bounding-box rule or primitives; `ext`: some of them
// PVB_GRID_TRILINEAR or primitives).
// The pack of the robot-family kernels (robot_serial_kernel and the forms built on its tiles): the links in index
// order with their bound constants (rs_link_consts); slots beyond n_sdf get radius -inf, i.e. a bound of +inf.
static RobotPack<kRsMaxS> rs_pack(const pvb_sdf_desc *descs, int n_sdf) {
    RobotPack<kRsMaxS> pack;
    memset(&pack, 0, sizeof(pack));
    for (int si = 0; si < n_sdf; ++si) { pack.d[si] = descs[si]; pack.orig[si] = si; }
    for (int si = 0; si < kRsMaxS; ++si) {
        if (si < n_sdf) rs_link_consts(descs[si], pack.sph_rad[si], pack.visit_margin[si]);
        else pack.sph_rad[si] = -PVB_INF;       // empty slot: bound +inf
    }
    return pack;
}

// The links the robot-family kernels evaluate: GRID sub-SDFs with the bounding-box rule (nearest or trilinear) and
// primitives; no mesh and no LOOKUP_GT_SDF grid.
static bool rs_links_ok(const pvb_sdf_desc *descs, int n_sdf) {
    for (int i = 0; i < n_sdf; ++i)
        if (descs[i].kind == PVB_KIND_GRID ? (descs[i].flags & PVB_GRID_OOB_GT) : descs[i].kind == PVB_KIND_MESH)
            return false;
    return true;
}

static int launch_robot_serial(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                               int cfg_count, const float *pts, long long n_pts, int vec, float *out_val,
                               float *out_grad, int *out_which, const OutTargets *tg, bool ext, cudaStream_t stream) {
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const int kind = !tg ? 0 : (tg->mc ? 2 : 1);
    decltype(&robot_serial_kernel<0, false>) const ks[3] = {
        ext ? robot_serial_kernel<0, true> : robot_serial_kernel<0, false>,
        ext ? robot_serial_kernel<1, true> : robot_serial_kernel<1, false>,
        ext ? robot_serial_kernel<2, true> : robot_serial_kernel<2, false>};
    const int smem = (int)sizeof(RsSmem);
    const int slot0 = ext ? kSlotSerialExt : kSlotSerial;
    for (int d = 0; d < 3; ++d)
        if (!ensure_smem(ks[d], slot0 + d, smem)) {
            pvb_set_error("pvb_composed_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
            return PVB_ERR_CUDA;
        }
    // tiles: cfg_count / 32 of 32 configurations, then one per binary digit of the remainder (rs_tile)
    const int n_full = cfg_count >> 5, rem = cfg_count & 31;
    const int gy = n_full + __builtin_popcount((unsigned)rem);
    // steps per resident warp slot at 8 points per step; below PVB_ROBOT_FINE_STEPS the launch runs 4-point steps
    auto steps_of = [&](int lc_log2) { const long long per = (long long)kRsChunk << (5 - lc_log2); return (n_pts + per - 1) / per; };
    long long total_steps = (long long)n_full * steps_of(5);
    for (int b = 4; b >= 0; --b) if (rem & (1 << b)) total_steps += steps_of(b);
    // (small configuration slabs favour 4 points per step, the full C4 batch 8; PVB_ROBOT_FINE_STEPS moves the switch)
    static const int fine_below = [] { const char *e = getenv("PVB_ROBOT_FINE_STEPS"); return e ? atoi(e) : 12; }();
    const long long slots = (long long)sm_count() * PVB_RS_MINB * kRsWarps;
    const int chunk_log2 = (kRsChunk == 4 || total_steps < (long long)fine_below * slots) ? 2 : 3;
    const long long n_chunks = (n_pts + (1 << chunk_log2) - 1) >> chunk_log2;     // steps of a 32-configuration tile
    long long gx = ((long long)sm_count() * PVB_RS_MINB * robot_waves() + gy - 1) / gy;
    const long long gx_max = (n_chunks + kRsWarps - 1) / kRsWarps;
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    const long long spw = chunk_log2;
    dim3 grid((unsigned)gx, (unsigned)gy);
    timing_mark(0, stream);
    ks[kind]<<<grid, kRbCfg * kRsWarps, smem, stream>>>(
        pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts, vec, (int)spw, tg ? nullptr : out_val,
        tg ? nullptr : out_grad, out_which, tg ? *tg : OutTargets{});
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query(robot-serial)");
    return PVB_OK;
}

// Argument checks shared by the composed entry points (`fn` names the entry point in the error message); any_ext:
// some sub-SDF is PVB_GRID_TRILINEAR or a primitive (SPHERE / BOX / CYLINDER), so the kExt instantiations run.
static int composed_check_args(const char *fn, const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                               int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_pts,
                               const float *out_val, const float *out_grad, bool &any_ext) {
    if (!descs || !xforms || n_sdf < 1 || n_cfg < 1 || cfg_begin < 0 || cfg_count < 0 ||
        cfg_begin + cfg_count > n_cfg || n_pts < 0 || (n_pts > 0 && cfg_count > 0 && (!pts || !out_val || !out_grad))) {
        pvb_set_error("%s: invalid argument (n_sdf=%d n_cfg=%d cfg=[%d,+%d) n_pts=%lld)", fn, n_sdf, n_cfg,
                      cfg_begin, cfg_count, (long long)n_pts);
        return PVB_ERR_INVALID;
    }
    if (n_sdf > 128) {
        pvb_set_error("%s: at most 128 sub-SDFs per call (got %d)", fn, n_sdf);
        return PVB_ERR_INVALID;
    }
    any_ext = false;
    for (int i = 0; i < n_sdf; ++i) {
        if (descs[i].kind < PVB_KIND_GRID || descs[i].kind > PVB_KIND_CYLINDER) {
            pvb_set_error("%s: sub-SDF %d: unknown kind %d", fn, i, descs[i].kind);
            return PVB_ERR_INVALID;
        }
        if (descs[i].kind != PVB_KIND_MESH && descs[i].kind != PVB_KIND_GRID) any_ext = true;
        if (descs[i].kind != PVB_KIND_GRID || !(descs[i].flags & PVB_GRID_TRILINEAR)) continue;
        if (descs[i].flags & PVB_GRID_OOB_GT) {
            pvb_set_error("%s: sub-SDF %d: PVB_GRID_TRILINEAR supports the bounding-box rule only", fn, i);
            return PVB_ERR_INVALID;
        }
        any_ext = true;
    }
    return PVB_OK;
}

// tg == nullptr: one destination (out_val / out_grad); otherwise the kMulti instantiations store to every target
static int composed_dispatch(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                             int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_pts,
                             uint32_t mesh_mode, float *out_val, float *out_grad, int32_t *out_which,
                             const OutTargets *tg, void *stream) {
    bool any_ext;
    const int bad = composed_check_args("pvb_composed_query", descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts,
                                        n_pts, out_val, out_grad, any_ext);
    if (bad) return bad;
    if (n_pts == 0 || cfg_count == 0) return PVB_OK;
    // The robot and configuration-major kernels run one grid row per configuration tile (rs_tile_count).  A slab of
    // more tiles than a grid has rows runs as consecutive slabs, each of whole 32-configuration tiles but the last and
    // balanced so that each takes the route the whole would (none of them a small remainder).  A configuration's row
    // depends on nothing else of the slab, so the rows are bit for bit those of one call.
    if (rs_tile_count(cfg_count) > kRsMaxGridRows) {
        // at most kSlab configurations per slab: 65531 tiles of 32 and up to 4 remainder tiles fit in a grid
        constexpr int kSlab = (kRsMaxGridRows - 4) * kRbCfg;
        const int n_slab = (cfg_count - 1) / kSlab + 1;
        const int step = ((cfg_count - 1) / n_slab / kRbCfg + 1) * kRbCfg;      // <= kSlab, whole tiles
        for (long long b = 0; b < cfg_count; b += step) {
            const int cnt = (int)(cfg_count - b < step ? cfg_count - b : step);
            const size_t o = (size_t)b * (size_t)n_pts;
            OutTargets sub{};
            if (tg) {
                sub = *tg;
                for (int t = 0; t < sub.n; ++t) { sub.val[t] += o; sub.grad[t] += 3 * o; }
            }
            const int rc = composed_dispatch(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin + (int)b, cnt, pts, n_pts,
                                             mesh_mode, out_val ? out_val + o : nullptr,
                                             out_grad ? out_grad + 3 * o : nullptr, out_which ? out_which + o : nullptr,
                                             tg ? &sub : nullptr, stream);
            if (rc) return rc;
        }
        return PVB_OK;
    }
    cudaStream_t s = (cudaStream_t)stream;
    auto aligned16 = [](const void *p) { return p == nullptr || ((uintptr_t)p % 16) == 0; };
    // 4-points-per-thread vector path needs 16-byte aligned rows: every configuration slab starts at c * n_pts
    bool out_aligned = aligned16(out_val) && aligned16(out_grad);
    OutTargets tgv{};
    if (tg) {
        for (int t = 0; t < tg->n; ++t) out_aligned = out_aligned && aligned16(tg->val[t]) && aligned16(tg->grad[t]);
        tgv = *tg;
        tgv.vec = out_aligned && (n_pts % 4 == 0);
        tg = &tgv;
    }
    static const int cfg_major = [] { const char *e = getenv("PVB_COMP_CFGMAJOR"); return e ? atoi(e) : 1; }();
    static const int robot_kernel = [] { const char *e = getenv("PVB_ROBOT_KERNEL"); return e ? atoi(e) : 2; }();
    // every sub-SDF a GRID with the bounding-box rule (nearest or trilinear) or a primitive: the robot kernels'
    // precondition (primitives and trilinear grids then need the serial kernel, see serial_taken)
    const bool all_grid = !needs_mesh && n_sdf <= 16 && rs_int_pts_ok(n_pts) && rs_links_ok(descs, n_sdf);
    // the point-serial kernel has no fill problem (remainder configurations run in lane-split tiles): any batch of
    // PVB_ROBOT_MIN_CFG or more configurations takes it
    static const int serial_min_cfg = [] { const char *e = getenv("PVB_ROBOT_MIN_CFG"); return e ? atoi(e) : 8; }();
    const bool serial_ok = robot_kernel >= 2 && n_sdf <= kRsMaxS && cfg_count >= serial_min_cfg &&
                           rs_tile_count(cfg_count) <= kRsMaxGridRows;          // one grid row per tile
    // sets with trilinear or primitive links take the serial kernel where nearest sets would; robot_query_kernel (9-16
    // links) is nearest-voxel only, so otherwise they fall through to the configuration-major or point-major kernel
    const bool serial_taken = robot_kernel && cfg_major && all_grid && serial_ok;
    if (tg && tg->mc) {
        // multicast destinations exist only in the robot kernels: refuse anything that would fall through
        if (!all_grid || (any_ext && !serial_taken)) {
            pvb_set_error(any_ext ? "pvb_composed_query_multicast: trilinear and primitive sub-SDFs need <= %d GRID "
                                    "(bounding-box rule) or primitive sub-SDFs and >= PVB_ROBOT_MIN_CFG configurations"
                                  : "pvb_composed_query_multicast: needs <= 16 GRID sub-SDFs with the bounding-box rule",
                          kRsMaxS);
            return PVB_ERR_INVALID;
        }
    }
    const bool vec = !needs_mesh && aligned16(pts) && out_aligned && aligned16(out_which) && (n_pts % 4 == 0);
    // lanes = configurations: only worthwhile when the 32-wide configuration tiles are well filled (25 configurations
    // per rank on 8 GPUs would idle 22 % of the lanes, and point-major is faster there)
    const int cm_tiles = (cfg_count + kCmCfg - 1) / kCmCfg;
    // ... except with several destinations: the configuration-major epilogue owns whole rows and stores them as full
    // sectors, which is what the NVLink-bound re-assembly needs; idle lanes cost less than partial-sector packets
    const bool cm_filled = (cfg_count >= 16 && (double)cfg_count >= 0.85 * (double)(cm_tiles * kCmCfg)) ||
                           (tg && tg->vec && cfg_count >= 8);
    static const double robot_fill = [] { const char *e = getenv("PVB_ROBOT_MIN_FILL"); return e ? atof(e) : 0.85; }();
    const bool rb_filled = (cfg_count >= 16 && (double)cfg_count >= robot_fill * (double)(cm_tiles * kCmCfg)) ||
                           (tg && tg->vec && cfg_count >= 8) || (tg && tg->mc);
    // PVB_ROBOT_KERNEL: 2 (default) = point-serial nearest-sphere-first kernel for <= 8 links, 1 = the
    // 4-points-per-thread kernel, 0 = round 1's configuration-major kernel
    if (serial_taken)
        return launch_robot_serial(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                   (tg ? tg->vec : (out_aligned && (n_pts % 4 == 0))), out_val, out_grad, out_which,
                                   tg, any_ext, s);
    if (robot_kernel && cfg_major && all_grid && !any_ext && rb_filled) {
        const int vec_rows = (tg ? tg->vec : (out_aligned && (n_pts % 4 == 0))) && aligned16(pts);
        return n_sdf <= 8 ? launch_robot<8, true>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, vec_rows,
                                                  out_val, out_grad, out_which, tg, s)
                          : launch_robot<16, false>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                                    vec_rows, out_val, out_grad, out_which, tg, s);
    }
    if (cfg_major && !needs_mesh && n_sdf <= kCmMaxS && cm_filled) {
        auto kl = any_ext ? composed_cfgmajor_kernel<false, true> : composed_cfgmajor_kernel<false, false>;
        auto km = any_ext ? composed_cfgmajor_kernel<true, true> : composed_cfgmajor_kernel<true, false>;
        const int slot = any_ext ? kSlotCfgMajorExt : kSlotCfgMajor;
        if (!ensure_smem(kl, slot, (int)sizeof(CmSmem)) || !ensure_smem(km, slot + 1, (int)sizeof(CmSmem))) {
            pvb_set_error("pvb_composed_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
            return PVB_ERR_CUDA;
        }
        const DescPack<kCmMaxS> pack = desc_pack<kCmMaxS>(descs, n_sdf);
        const int gy = (cfg_count + kCmCfg - 1) / kCmCfg;
        const long long n_tiles = (n_pts + kCmTilePts - 1) / kCmTilePts;
        long long gx = ((long long)sm_count() * 3 * 4 + gy - 1) / gy;     // ~4 waves of resident CTAs
        if (gx > n_tiles) gx = n_tiles;
        if (gx < 1) gx = 1;
        dim3 grid((unsigned)gx, (unsigned)gy);
        timing_mark(0, s);
        (tg ? km : kl)<<<grid, kCmCfg * kCmWarps, sizeof(CmSmem), s>>>(
            pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, tg ? nullptr : out_val,
            tg ? nullptr : out_grad, out_which, tg ? *tg : OutTargets{});
        timing_mark(1, s);
        PVB_CHECK_LAUNCH("pvb_composed_query(cfg-major)");
        return PVB_OK;
    }
    // point-major; the 4-points-per-thread vector rows exist for sets without meshes only (vec implies !needs_mesh)
    return comp_variant(needs_mesh, any_ext, n_sdf, [&](auto kMesh, auto kExt, auto kMaxS) {
        if constexpr (kMesh)
            return launch_composed<true, 1, kMaxS, kExt>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                                         mesh_mode, out_val, out_grad, out_which, tg, s);
        else if (vec)
            return launch_composed<false, PVB_COMP_PTS, kMaxS, kExt>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count,
                                                                     pts, n_pts, mesh_mode, out_val, out_grad,
                                                                     out_which, tg, s);
        else
            return launch_composed<false, 1, kMaxS, kExt>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                                          mesh_mode, out_val, out_grad, out_which, tg, s);
    });
}

extern "C" int pvb_composed_query(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                                  int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                  const float *pts, int64_t n_pts, uint32_t mesh_mode, float *out_val, float *out_grad,
                                  int32_t *out_which, void *stream) {
    return composed_dispatch(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, mesh_mode,
                             out_val, out_grad, out_which, nullptr, stream);
}

template <bool kMesh, bool kExt, int MAXS>
static int launch_paired(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                         const float *pts, long long n_pts, long long n_pairs, uint32_t mesh_mode, float *out_val,
                         float *out_grad, int *out_which, cudaStream_t stream) {
    const DescPack<MAXS> pack = desc_pack<MAXS>(descs, n_sdf);
    const CompConsts c = comp_consts(descs, n_sdf);
    timing_mark(0, stream);
    composed_paired_kernel<kMesh, kExt, MAXS><<<grid_for(n_pairs, kCompThreads, 8), kCompThreads, 0, stream>>>(
        pack, n_sdf, xforms, n_cfg, cfg_begin, pts, n_pts, n_pairs, mesh_mode, out_val, out_grad, out_which,
        c.nearest_first, c.margin_max);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query_paired");
    return PVB_OK;
}

extern "C" int pvb_composed_query_paired(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                         const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                         const float *pts, int64_t n_pts, uint32_t mesh_mode, float *out_val,
                                         float *out_grad, int32_t *out_which, void *stream) {
    bool any_ext;
    const int bad = composed_check_args("pvb_composed_query_paired", descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count,
                                        pts, n_pts, out_val, out_grad, any_ext);
    if (bad) return bad;
    if (n_pts == 0 || cfg_count == 0) return PVB_OK;
    if (n_pts > INT64_MAX / cfg_count) {
        pvb_set_error("pvb_composed_query_paired: cfg_count * n_pts overflows int64 (cfg_count=%d n_pts=%lld)",
                      cfg_count, (long long)n_pts);
        return PVB_ERR_INVALID;
    }
    const long long n_pairs = (long long)cfg_count * n_pts;
    return comp_variant(needs_mesh, any_ext, n_sdf, [&](auto kMesh, auto kExt, auto kMaxS) {
        return launch_paired<kMesh, kExt, kMaxS>(descs, n_sdf, xforms, n_cfg, cfg_begin, pts, n_pts, n_pairs, mesh_mode,
                                                 out_val, out_grad, out_which, (cudaStream_t)stream);
    });
}

// Launch robot_swept_kernel.  Points per block: as many as keep >= 2 waves of resident blocks, so that the tile
// staging is shared by up to 128 points without leaving SMs idle at 10^5 points.
static int launch_robot_swept(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                              int cfg_count, const float *pts, long long n_pts, float *out_val, float *out_grad,
                              int *out_cfg, int *out_which, bool ext, cudaStream_t stream) {
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const long long slots = (long long)sm_count() * PVB_RS_MINB;
    int blk_pts = kSwMaxPts;
    while (blk_pts > 32 && n_pts < 2 * slots * blk_pts) blk_pts >>= 1;
    const long long gx = (n_pts + blk_pts - 1) / blk_pts;
    auto k = ext ? robot_swept_kernel<true> : robot_swept_kernel<false>;
    timing_mark(0, stream);
    k<<<(unsigned)gx, kRbCfg * kRsWarps, 0, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      blk_pts, out_val, out_grad, out_cfg, out_which);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query_swept(robot)");
    return PVB_OK;
}

template <bool kMesh, bool kExt, int MAXS>
static int launch_swept(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                        int cfg_count, const float *pts, long long n_pts, uint32_t mesh_mode, float *out_val,
                        float *out_grad, int *out_cfg, int *out_which, cudaStream_t stream) {
    const DescPack<MAXS> pack = desc_pack<MAXS>(descs, n_sdf);
    const CompConsts c = comp_consts(descs, n_sdf);
    timing_mark(0, stream);
    composed_swept_kernel<kMesh, kExt, MAXS><<<grid_for(n_pts, kCompThreads, 8), kCompThreads, 0, stream>>>(
        pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, mesh_mode, out_val, out_grad, out_cfg,
        out_which, c.nearest_first, c.margin_max);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query_swept");
    return PVB_OK;
}

extern "C" int pvb_composed_query_swept(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                        const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                        const float *pts, int64_t n_pts, uint32_t mesh_mode, float *out_val,
                                        float *out_grad, int32_t *out_cfg, int32_t *out_which, void *stream) {
    bool any_ext;
    const int bad = composed_check_args("pvb_composed_query_swept", descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count,
                                        pts, n_pts, out_val, out_grad, any_ext);
    if (bad) return bad;
    if (n_pts == 0) return PVB_OK;
    if (cfg_count < 1) {
        pvb_set_error("pvb_composed_query_swept: no minimum over an empty configuration slab (cfg_count=%d)", cfg_count);
        return PVB_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    // robot_serial_kernel's sets take the fused kernel: <= 8 GRID links with the bounding-box rule or primitives
    const bool fused = !needs_mesh && n_sdf <= kRsMaxS && n_pts < (1ll << 31) && rs_links_ok(descs, n_sdf);
    if (fused)
        return launch_robot_swept(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, out_val, out_grad,
                                  out_cfg, out_which, any_ext, s);
    return comp_variant(needs_mesh, any_ext, n_sdf, [&](auto kMesh, auto kExt, auto kMaxS) {
        return launch_swept<kMesh, kExt, kMaxS>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                                mesh_mode, out_val, out_grad, out_cfg, out_which, s);
    });
}

// The longest chunk of the clearance kernels: their point loops step j0 = 0, 32, 64, ... (robot_clearance_kernel: up to
// 256) past the chunk's end in int, so a chunk as long as a segment of nearly 2^31 points would wrap.  The chunking
// never changes a result (the keys name the first point attaining the minimum).
constexpr long long kRsMaxChunk = 1ll << 30;

// Argument rules of the clearance, self-clearance and collision-cost entry points (`fn` names the entry point in the
// error message).  Each entry point applies them in its own order: the first that fails decides the error.

// Segment sizes: seg_len < 2^31, n_seg * seg_len and cfg_count * n_seg below 2^63, and (`paired`: one point set per
// configuration) cfg_count * n_seg * seg_len below 2^63.
static int check_segments(const char *fn, long long n_seg, long long seg_len, int cfg_count, bool paired) {
    if (n_seg < 0 || seg_len < 0 || seg_len >= (1ll << 31) || (seg_len > 0 && n_seg > INT64_MAX / seg_len) ||
        (cfg_count > 0 && n_seg > INT64_MAX / cfg_count) ||
        (paired && cfg_count > 0 && n_seg * seg_len > INT64_MAX / cfg_count)) {
        if (paired)
            pvb_set_error("%s: invalid argument (n_seg=%lld seg_len=%lld cfg_count=%d; seg_len < 2^31, "
                          "cfg_count * n_seg * seg_len < 2^63)", fn, n_seg, seg_len, cfg_count);
        else
            pvb_set_error("%s: invalid argument (n_seg=%lld seg_len=%lld cfg_count=%d; seg_len < 2^31)", fn, n_seg,
                          seg_len, cfg_count);
        return PVB_ERR_INVALID;
    }
    return PVB_OK;
}

// The link points of the self forms: K per link with 1 <= K < 2^24, the inverse transforms and the allowed rows.
static int check_link_points(const char *fn, long long K, const float *inv_xforms, const uint8_t *allowed) {
    if (K < 1 || K >= (1ll << 24) || !inv_xforms || !allowed) {
        pvb_set_error("%s: invalid argument (K=%lld; 1 <= K < 2^24, inv_xforms and allowed not null)", fn, K);
        return PVB_ERR_INVALID;
    }
    return PVB_OK;
}

static int check_margin(const char *fn, float margin) {
    if (!(margin - margin == 0.f)) {                 // NaN or +-inf
        pvb_set_error("%s: the margin must be finite (margin=%g)", fn, (double)margin);
        return PVB_ERR_INVALID;
    }
    return PVB_OK;
}

// The forms without a generic route take robot_serial_kernel's sets only: <= 8 GRID links with the bounding-box rule,
// or primitives.  `instead` is the advice the refusal closes with.
static int check_fused_only(const char *fn, const pvb_sdf_desc *descs, int n_sdf, const char *instead) {
    if (n_sdf > kRsMaxS || !rs_links_ok(descs, n_sdf)) {
        pvb_set_error("%s: the fused query takes at most %d grid (bounding-box rule) or primitive sub-SDFs, no mesh or "
                      "LOOKUP_GT_SDF grid (n_sdf=%d); %s instead", fn, kRsMaxS, n_sdf, instead);
        return PVB_ERR_INVALID;
    }
    return PVB_OK;
}

// The rows of the self forms from allowed[i] (bit j allows the pair (i, j)): the diagonal cleared, and the sources
// with a non-empty row in ascending order (n_src of them).
static int scl_rows(const char *fn, const uint8_t *allowed, int n_sdf, SclRows &rows, int &n_src) {
    memset(&rows, 0, sizeof(rows));
    n_src = 0;
    for (int i = 0; i < n_sdf; ++i) {
        if (allowed[i] >> n_sdf) {
            pvb_set_error("%s: allowed row %d has bits beyond n_sdf=%d (0x%02x)", fn, i, n_sdf, allowed[i]);
            return PVB_ERR_INVALID;
        }
        rows.mask[i] = (unsigned char)(allowed[i] & ~(1u << i));
        if (rows.mask[i]) rows.src[n_src++] = (unsigned char)i;
    }
    return PVB_OK;
}

// The n minimum keys of a clearance form start all-ones: no point reached yet.
static int reset_keys(const char *fn, uint64_t *keys, size_t n, cudaStream_t stream) {
    if (!keys) {
        pvb_set_error("%s: invalid argument (keys is null)", fn);
        return PVB_ERR_INVALID;
    }
    if (cudaMemsetAsync(keys, 0xff, sizeof(uint64_t) * n, stream) != cudaSuccess) {
        pvb_set_error("%s: cudaMemsetAsync(keys) failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
        return PVB_ERR_CUDA;
    }
    return PVB_OK;
}

// Launch robot_clearance_kernel.  Chunk size from the sizes alone: the longest chunk (at least 64 points, or the whole
// segment) that still gives >= 4 waves of resident blocks over the tiles x segments x chunks, so that blocks of later
// waves start from the keys of earlier ones.
static int launch_robot_clearance(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                                  int cfg_count, const float *pts, long long n_seg, long long seg_len,
                                  unsigned long long *keys, bool ext, cudaStream_t stream) {
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const int gy = rs_tile_count(cfg_count);
    const long long want = 4ll * sm_count() * PVB_RS_MINB;          // blocks for 4 waves
    long long per_seg = (want + (long long)gy * n_seg - 1) / ((long long)gy * n_seg);
    if (per_seg > (seg_len + 63) / 64) per_seg = (seg_len + 63) / 64;
    if (per_seg < (seg_len + kRsMaxChunk - 1) / kRsMaxChunk) per_seg = (seg_len + kRsMaxChunk - 1) / kRsMaxChunk;
    if (per_seg < 1) per_seg = 1;
    const long long chunk = (seg_len + per_seg - 1) / per_seg;
    const long long chunks_per_seg = (seg_len + chunk - 1) / chunk;
    const long long n_work = n_seg * chunks_per_seg;
    const unsigned gx = (unsigned)(n_work < INT32_MAX ? n_work : INT32_MAX);
    dim3 grid(gx, (unsigned)gy);
    auto k = ext ? robot_clearance_kernel<true> : robot_clearance_kernel<false>;
    timing_mark(0, stream);
    k<<<grid, kRbCfg * kRsWarps, 0, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg,
                                              (int)seg_len, (int)chunk, (int)chunks_per_seg, keys);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query_clearance(robot)");
    return PVB_OK;
}

// The warp units of robot_paired_clearance_kernel and robot_self_clearance_kernel: `rows` rows of `len` points (a
// segment or a link's K points), each cut into chunks of whole warp steps.  The longest chunk (at least 64 points, at
// most kRsMaxChunk, or the whole row) that still gives >= 4 waves of resident units, so that the later chunks of a row
// start from the keys of its earlier ones.
struct WarpPlan {
    long long chunk, n_units;
    unsigned blocks;
};

static WarpPlan warp_plan(long long rows, long long len) {
    const long long want = 4ll * sm_count() * PVB_RS_MINB * kRsWarps;    // warp units for 4 waves
    long long per_row = (want + rows - 1) / rows;
    if (per_row > (len + 63) / 64) per_row = (len + 63) / 64;
    if (per_row < (len + kRsMaxChunk - 1) / kRsMaxChunk) per_row = (len + kRsMaxChunk - 1) / kRsMaxChunk;
    if (per_row < 1) per_row = 1;
    long long chunk = (len + per_row - 1) / per_row;
    chunk = (chunk + 31) / 32 * 32;                                      // whole steps of the warp
    if (chunk > len) chunk = len;
    const long long n_units = rows * ((len + chunk - 1) / chunk);
    const long long blocks = (n_units + kRsWarps - 1) / kRsWarps;
    return {chunk, n_units, (unsigned)(blocks < INT32_MAX ? blocks : INT32_MAX)};
}

// Launch robot_paired_clearance_kernel over the warp units of warp_plan.
static int launch_robot_paired_clearance(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg,
                                         int cfg_begin, int cfg_count, const float *pts, long long n_seg,
                                         long long seg_len, unsigned long long *keys, bool ext, cudaStream_t stream) {
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const WarpPlan p = warp_plan((long long)cfg_count * n_seg, seg_len);
    auto k = ext ? robot_paired_clearance_kernel<true> : robot_paired_clearance_kernel<false>;
    timing_mark(0, stream);
    k<<<p.blocks, kRbCfg * kRsWarps, 0, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg,
                                                  (int)seg_len, (int)p.chunk, p.n_units, keys);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query_paired_clearance(robot)");
    return PVB_OK;
}

// The keys of composed_clearance_kernel (unless `fused`: robot_clearance_kernel already left them), then
// clearance_finish_kernel.  kPaired: their paired forms, composed_paired_clearance_kernel (unless
// robot_paired_clearance_kernel left the keys) and paired_clearance_finish_kernel.
template <bool kMesh, bool kExt, int MAXS, bool kPaired = false>
static int launch_clearance(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                            int cfg_count, const float *pts, long long n_seg, long long seg_len, uint32_t mesh_mode,
                            unsigned long long *keys, bool fused, float *out_val, float *out_grad, int *out_point,
                            int *out_which, cudaStream_t stream) {
    const DescPack<MAXS> pack = desc_pack<MAXS>(descs, n_sdf);
    const CompConsts c = comp_consts(descs, n_sdf);
    if (!fused) {
        (kPaired ? composed_paired_clearance_kernel<kMesh, kExt, MAXS> : composed_clearance_kernel<kMesh, kExt, MAXS>)
            <<<grid_for((long long)cfg_count * n_seg * seg_len, kCompThreads, 8), kCompThreads, 0, stream>>>(
                pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len, mesh_mode, keys,
                c.nearest_first, c.margin_max);
        PVB_CHECK_LAUNCH("pvb_composed_query_clearance");
    }
    (kPaired ? paired_clearance_finish_kernel<kMesh, kExt, MAXS> : clearance_finish_kernel<kMesh, kExt, MAXS>)
        <<<grid_for((long long)cfg_count * n_seg, kCompThreads, 8), kCompThreads, 0, stream>>>(
            pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len, mesh_mode, keys, out_val, out_grad,
            out_point, out_which, c.nearest_first, c.margin_max);
    PVB_CHECK_LAUNCH("pvb_composed_query_clearance(finish)");
    return PVB_OK;
}

// pvb_composed_query_clearance, and pvb_composed_query_paired_clearance (kPaired: configuration c's points are its
// own n_seg * seg_len); they differ in the point count they bound and in their fused kernel.
template <bool kPaired>
static int clearance_query(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                           int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_seg,
                           int64_t seg_len, uint32_t mesh_mode, uint64_t *keys, float *out_val, float *out_grad,
                           int32_t *out_point, int32_t *out_which, void *stream) {
    const char *fn = kPaired ? "pvb_composed_query_paired_clearance" : "pvb_composed_query_clearance";
    if (int rc = check_segments(fn, n_seg, seg_len, cfg_count, kPaired)) return rc;
    const long long n_pts = n_seg * seg_len;                 // points per configuration
    bool any_ext;
    const int bad = composed_check_args(fn, descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, out_val,
                                        out_grad, any_ext);
    if (bad) return bad;
    if (n_seg == 0) return PVB_OK;
    if (cfg_count < 1) {
        if (n_pts == 0) return PVB_OK;
        pvb_set_error("%s: no minimum over an empty configuration slab (cfg_count=%d)", fn, cfg_count);
        return PVB_ERR_INVALID;
    }
    if (seg_len == 0) {
        pvb_set_error("%s: no minimum over an empty segment (seg_len=0, n_seg=%lld)", fn, (long long)n_seg);
        return PVB_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = reset_keys(fn, keys, (size_t)cfg_count * (size_t)n_seg, s)) return rc;
    unsigned long long *k = reinterpret_cast<unsigned long long *>(keys);
    // robot_serial_kernel's sets take the fused kernel: <= 8 GRID links with the bounding-box rule or primitives.  The
    // clearance kernel runs one grid row per configuration tile; the paired kernel's 1-D grid has no limit on cfg_count.
    const bool fused = !needs_mesh && n_sdf <= kRsMaxS && (kPaired || rs_tile_count(cfg_count) <= kRsMaxGridRows) &&
                       rs_links_ok(descs, n_sdf);
    if (fused) {
        const int rc = (kPaired ? launch_robot_paired_clearance : launch_robot_clearance)(
            descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len, k, any_ext, s);
        if (rc) return rc;
    }
    return comp_variant(needs_mesh, any_ext, n_sdf, [&](auto kMesh, auto kExt, auto kMaxS) {
        return launch_clearance<kMesh, kExt, kMaxS, kPaired>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts,
                                                             n_seg, seg_len, mesh_mode, k, fused, out_val, out_grad,
                                                             out_point, out_which, s);
    });
}

extern "C" int pvb_composed_query_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                            const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                            const float *pts, int64_t n_seg, int64_t seg_len, uint32_t mesh_mode,
                                            uint64_t *keys, float *out_val, float *out_grad, int32_t *out_point,
                                            int32_t *out_which, void *stream) {
    return clearance_query<false>(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                  mesh_mode, keys, out_val, out_grad, out_point, out_which, stream);
}

extern "C" int pvb_composed_query_paired_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                                   const float *xforms, int32_t n_cfg, int32_t cfg_begin,
                                                   int32_t cfg_count, const float *pts, int64_t n_seg, int64_t seg_len,
                                                   uint32_t mesh_mode, uint64_t *keys, float *out_val, float *out_grad,
                                                   int32_t *out_point, int32_t *out_which, void *stream) {
    return clearance_query<true>(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                 mesh_mode, keys, out_val, out_grad, out_point, out_which, stream);
}

// Launch robot_self_clearance_kernel (when some row is not empty) over the warp units of warp_plan, then
// self_clearance_finish_kernel.
static int launch_self_clearance(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, const float *inv_xforms,
                                 int n_cfg, int cfg_begin, int cfg_count, const float *link_pts, int K,
                                 const SclRows &rows, int n_src, unsigned long long *keys, float *out_val,
                                 float *out_grad, int *out_src, int *out_point, int *out_which, bool ext,
                                 cudaStream_t stream) {
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    if (n_src > 0) {
        const WarpPlan p = warp_plan((long long)cfg_count * n_src, K);
        auto k = ext ? robot_self_clearance_kernel<true> : robot_self_clearance_kernel<false>;
        timing_mark(0, stream);
        k<<<p.blocks, kRbCfg * kRsWarps, 0, stream>>>(pack, n_sdf, xforms, inv_xforms, n_cfg, cfg_begin, cfg_count,
                                                      link_pts, K, rows, n_src, (int)p.chunk, p.n_units, keys);
        timing_mark(1, stream);
        PVB_CHECK_LAUNCH("pvb_composed_query_self_clearance");
    }
    auto kf = ext ? self_clearance_finish_kernel<true> : self_clearance_finish_kernel<false>;
    kf<<<(unsigned)grid_for(cfg_count, kCompThreads, 8), kCompThreads, 0, stream>>>(
        pack, n_sdf, xforms, inv_xforms, n_cfg, cfg_begin, cfg_count, link_pts, K, rows, keys, out_val, out_grad,
        out_src, out_point, out_which);
    PVB_CHECK_LAUNCH("pvb_composed_query_self_clearance(finish)");
    return PVB_OK;
}

extern "C" int pvb_composed_query_self_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                                 const float *inv_xforms, int32_t n_cfg, int32_t cfg_begin,
                                                 int32_t cfg_count, const float *link_pts, int64_t K,
                                                 const uint8_t *allowed, uint64_t *keys, float *out_val,
                                                 float *out_grad, int32_t *out_src, int32_t *out_point,
                                                 int32_t *out_which, void *stream) {
    const char *fn = "pvb_composed_query_self_clearance";
    if (int rc = check_link_points(fn, K, inv_xforms, allowed)) return rc;
    bool any_ext;
    const int bad = composed_check_args(fn, descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, link_pts,
                                        (int64_t)n_sdf * K, out_val, out_grad, any_ext);
    if (bad) return bad;
    if (cfg_count < 1) {
        pvb_set_error("%s: no minimum over an empty configuration slab (cfg_count=%d)", fn, cfg_count);
        return PVB_ERR_INVALID;
    }
    if (int rc = check_fused_only(fn, descs, n_sdf, "compose the per-source paired clearance queries")) return rc;
    SclRows rows;
    int n_src;
    if (int rc = scl_rows(fn, allowed, n_sdf, rows, n_src)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = reset_keys(fn, keys, (size_t)cfg_count, s)) return rc;
    return launch_self_clearance(descs, n_sdf, xforms, inv_xforms, n_cfg, cfg_begin, cfg_count, link_pts, (int)K, rows,
                                 n_src, reinterpret_cast<unsigned long long *>(keys), out_val, out_grad, out_src,
                                 out_point, out_which, any_ext, s);
}

// Bytes of partial sums a collision-cost query needs: one fp32 row of 1 + 6 n_sdf per (configuration, segment, chunk);
// -1 for negative sizes or an overflow.
static long long collision_cost_bytes(int n_sdf, long long cfg_count, long long n_seg, long long seg_len) {
    if (n_sdf < 1 || cfg_count < 0 || n_seg < 0 || seg_len < 0) return -1;
    const long long row = 4ll * (1 + 6 * (long long)n_sdf);
    const long long cps = collision_cost_chunks(seg_len);
    long long n = cfg_count;
    for (const long long f : {n_seg, cps, row}) {
        if (f != 0 && n > INT64_MAX / f) return -1;
        n *= f;
    }
    return n;
}

extern "C" int64_t pvb_collision_cost_workspace(int32_t n_sdf, int32_t cfg_count, int64_t n_seg, int64_t seg_len) {
    return collision_cost_bytes(n_sdf, cfg_count, n_seg, seg_len);
}

// robot_collision_cost_kernel over every (tile, segment, chunk) unit, then collision_cost_finish_kernel.  kPaired:
// robot_paired_collision_cost_kernel over every (configuration, segment, chunk) warp unit instead.
template <bool kPaired>
static int launch_collision_cost(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                                 int cfg_count, const float *pts, long long n_seg, long long seg_len, float margin,
                                 float *partial, float *out_cost, float *out_twist, bool ext, cudaStream_t stream) {
    const char *fn = kPaired ? "pvb_composed_query_paired_collision_cost" : "pvb_composed_query_collision_cost";
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const int E = 1 + 6 * n_sdf;
    const long long chunk = collision_cost_chunk(seg_len), cps = collision_cost_chunks(seg_len);
    if (cps > 0 && kPaired) {
        auto k = ext ? robot_paired_collision_cost_kernel<true> : robot_paired_collision_cost_kernel<false>;
        const long long n_units = (long long)cfg_count * n_seg * cps;
        const long long blocks = (n_units + kRsWarps - 1) / kRsWarps;
        timing_mark(0, stream);
        k<<<(unsigned)(blocks < INT32_MAX ? blocks : INT32_MAX), kRbCfg * kRsWarps, 0, stream>>>(
            pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, (int)seg_len, (int)chunk, (int)cps, margin,
            n_units, partial);
        timing_mark(1, stream);
        PVB_CHECK_LAUNCH("pvb_composed_query_paired_collision_cost");
    } else if (cps > 0) {
        auto k = ext ? robot_collision_cost_kernel<true> : robot_collision_cost_kernel<false>;
        if (!ensure_smem(k, ext ? kSlotCollisionCostExt : kSlotCollisionCost, cc_smem_bytes(kRsMaxS))) {
            pvb_set_error("%s: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed", fn);
            return PVB_ERR_CUDA;
        }
        const long long n_units = (long long)((cfg_count + 31) >> 5) * n_seg * cps;
        const unsigned gx = (unsigned)(n_units < INT32_MAX ? n_units : INT32_MAX);
        timing_mark(0, stream);
        k<<<gx, kRbCfg * kCcWarps, cc_smem_bytes(n_sdf), stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts,
                                                                   n_seg, (int)seg_len, (int)chunk, (int)cps, margin,
                                                                   n_units, partial);
        timing_mark(1, stream);
        PVB_CHECK_LAUNCH("pvb_composed_query_collision_cost");
    }
    const long long rows = (long long)cfg_count * n_seg;
    collision_cost_finish_kernel<<<grid_for(rows * E, kCompThreads, 8), kCompThreads, 0, stream>>>(
        partial, rows, (int)cps, E, out_cost, out_twist);
    PVB_CHECK_LAUNCH(kPaired ? "pvb_composed_query_paired_collision_cost(finish)"
                             : "pvb_composed_query_collision_cost(finish)");
    return PVB_OK;
}

// pvb_composed_query_collision_cost, and pvb_composed_query_paired_collision_cost (kPaired: configuration c's points
// are its own n_seg * seg_len); they differ in the point count they bound and in their kernel, not in the workspace.
template <bool kPaired>
static int collision_cost_query(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms, int32_t n_cfg,
                                int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_seg, int64_t seg_len,
                                float margin, void *workspace, int64_t workspace_bytes, float *out_cost,
                                float *out_twist, void *stream) {
    const char *fn = kPaired ? "pvb_composed_query_paired_collision_cost" : "pvb_composed_query_collision_cost";
    if (int rc = check_segments(fn, n_seg, seg_len, cfg_count, kPaired)) return rc;
    if (int rc = check_margin(fn, margin)) return rc;
    const long long n_pts = n_seg * seg_len;                 // points per configuration
    bool any_ext;
    const int bad = composed_check_args(fn, descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts,
                                        kPaired ? (cfg_count > 0 ? cfg_count * n_pts : 0) : n_pts, out_cost,
                                        out_twist, any_ext);
    if (bad) return bad;
    if (n_seg == 0) return PVB_OK;
    if (cfg_count < 1) {
        if (n_pts == 0) return PVB_OK;
        pvb_set_error("%s: no configurations to sum for (cfg_count=%d) with points", fn, cfg_count);
        return PVB_ERR_INVALID;
    }
    if (!out_cost || !out_twist) {                   // empty segments still get their zeros
        pvb_set_error("%s: invalid argument (out_cost or out_twist is null)", fn);
        return PVB_ERR_INVALID;
    }
    if (int rc = check_fused_only(fn, descs, n_sdf, kPaired ? "compose it from pvb_composed_query_paired"
                                                             : "compose it from pvb_composed_query"))
        return rc;
    const long long need = collision_cost_bytes(n_sdf, cfg_count, n_seg, seg_len);
    if (need < 0 || (need > 0 && (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 3)))) {
        pvb_set_error("%s: the workspace must hold pvb_collision_cost_workspace() = %lld bytes, 4-byte aligned "
                      "(got %lld bytes)", fn, need, (long long)workspace_bytes);
        return PVB_ERR_INVALID;
    }
    return launch_collision_cost<kPaired>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len,
                                          margin, reinterpret_cast<float *>(workspace), out_cost, out_twist, any_ext,
                                          (cudaStream_t)stream);
}

extern "C" int pvb_composed_query_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                                 int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                                 const float *pts, int64_t n_seg, int64_t seg_len, float margin,
                                                 void *workspace, int64_t workspace_bytes, float *out_cost,
                                                 float *out_twist, void *stream) {
    return collision_cost_query<false>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len, margin,
                                       workspace, workspace_bytes, out_cost, out_twist, stream);
}

extern "C" int pvb_composed_query_paired_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf,
                                                        const float *xforms, int32_t n_cfg, int32_t cfg_begin,
                                                        int32_t cfg_count, const float *pts, int64_t n_seg,
                                                        int64_t seg_len, float margin, void *workspace,
                                                        int64_t workspace_bytes, float *out_cost, float *out_twist,
                                                        void *stream) {
    return collision_cost_query<true>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_seg, seg_len, margin,
                                      workspace, workspace_bytes, out_cost, out_twist, stream);
}

extern "C" int pvb_composed_query_self_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                                      const float *inv_xforms, int32_t n_cfg, int32_t cfg_begin,
                                                      int32_t cfg_count, const float *link_pts, int64_t K,
                                                      const uint8_t *allowed, float margin, float *out_cost,
                                                      float *out_twist, void *stream) {
    const char *fn = "pvb_composed_query_self_collision_cost";
    if (int rc = check_link_points(fn, K, inv_xforms, allowed)) return rc;
    if (int rc = check_margin(fn, margin)) return rc;
    bool any_ext;
    const int bad = composed_check_args(fn, descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, link_pts,
                                        (int64_t)n_sdf * K, out_cost, out_twist, any_ext);
    if (bad) return bad;
    if (cfg_count < 1) {
        pvb_set_error("%s: no cost over an empty configuration slab (cfg_count=%d)", fn, cfg_count);
        return PVB_ERR_INVALID;
    }
    if (int rc = check_fused_only(fn, descs, n_sdf, "compose the per-source paired queries")) return rc;
    SclRows rows;
    int n_src;
    if (int rc = scl_rows(fn, allowed, n_sdf, rows, n_src)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const RobotPack<kRsMaxS> pack = rs_pack(descs, n_sdf);
    const long long blocks = ((long long)cfg_count + kSccWarps - 1) / kSccWarps;
    auto k = any_ext ? robot_self_collision_cost_kernel<true> : robot_self_collision_cost_kernel<false>;
    timing_mark(0, s);
    k<<<(unsigned)blocks, kSccLanes * kSccWarps, 0, s>>>(pack, n_sdf, xforms, inv_xforms, n_cfg, cfg_begin, cfg_count,
                                                         link_pts, (int)K, rows, n_src, margin, out_cost, out_twist);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH("pvb_composed_query_self_collision_cost");
    return PVB_OK;
}

// The checks of both scene entry points, in order (`fn` names the entry point): K, inv_xforms and links
// (check_link_points), the scene as the composed entry points check their sub-SDFs (one configuration), the robot's
// sub-SDF count and slab, then no mesh and no LOOKUP_GT_SDF grid in the scene; the tested sources into `on`.
static int scene_check_args(const char *fn, const pvb_sdf_desc *scene, int32_t n_scene, const float *scene_xforms,
                            const float *inv_xforms, int32_t n_sdf, int32_t n_cfg, int32_t cfg_begin,
                            int32_t cfg_count, const float *link_pts, int64_t K, const uint8_t *links,
                            const float *out_a, const float *out_b, SceneLinks &on, bool &any_ext) {
    if (int rc = check_link_points(fn, K, inv_xforms, links)) return rc;
    if (int rc = composed_check_args(fn, scene, n_scene, scene_xforms, 1, 0, 1, link_pts,
                                     n_sdf > 0 ? (int64_t)n_sdf * K : 0, out_a, out_b, any_ext))
        return rc;
    if (n_sdf < 1 || n_sdf > kSceneMaxSources || n_cfg < 1 || cfg_begin < 0 || cfg_count < 1 ||
        cfg_begin > n_cfg - cfg_count) {
        pvb_set_error("%s: invalid argument (n_sdf=%d n_cfg=%d cfg=[%d,+%d); 1 <= n_sdf <= %d and a non-empty slab)",
                      fn, n_sdf, n_cfg, cfg_begin, cfg_count, kSceneMaxSources);
        return PVB_ERR_INVALID;
    }
    if (!rs_links_ok(scene, n_scene)) {
        pvb_set_error("%s: the fused scene query takes grid (bounding-box rule) or primitive scene sub-SDFs, no mesh or "
                      "LOOKUP_GT_SDF grid; query the scene at the posed link points instead", fn);
        return PVB_ERR_INVALID;
    }
    memset(&on, 0, sizeof(on));
    for (int i = 0; i < n_sdf; ++i) on.on[i] = links[i] ? 1 : 0;
    return PVB_OK;
}

extern "C" int pvb_composed_query_scene_clearance(const pvb_sdf_desc *scene, int32_t n_scene,
                                                  const float *scene_xforms, const float *inv_xforms, int32_t n_sdf,
                                                  int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                                  const float *link_pts, int64_t K, const uint8_t *links,
                                                  float *out_val, float *out_grad, int32_t *out_link,
                                                  int32_t *out_point, void *stream) {
    const char *fn = "pvb_composed_query_scene_clearance";
    SceneLinks on;
    bool any_ext;
    if (int rc = scene_check_args(fn, scene, n_scene, scene_xforms, inv_xforms, n_sdf, n_cfg, cfg_begin, cfg_count,
                                  link_pts, K, links, out_val, out_grad, on, any_ext))
        return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return comp_variant(false, any_ext, n_scene, [&](auto, auto kExt, auto kMaxS) {
        const DescPack<kMaxS> pack = desc_pack<kMaxS>(scene, n_scene);
        timing_mark(0, s);
        scene_clearance_kernel<kExt, kMaxS><<<(unsigned)cfg_count, kSceneLanes * kSceneWarps, 0, s>>>(
            pack, n_scene, scene_xforms, inv_xforms, n_sdf, n_cfg, cfg_begin, cfg_count, link_pts, (int)K, on, out_val,
            out_grad, out_link, out_point);
        timing_mark(1, s);
        PVB_CHECK_LAUNCH("pvb_composed_query_scene_clearance");
        return PVB_OK;
    });
}

extern "C" int pvb_composed_query_scene_collision_cost(const pvb_sdf_desc *scene, int32_t n_scene,
                                                       const float *scene_xforms, const float *inv_xforms,
                                                       int32_t n_sdf, int32_t n_cfg, int32_t cfg_begin,
                                                       int32_t cfg_count, const float *link_pts, int64_t K,
                                                       const uint8_t *links, float margin, float *out_cost,
                                                       float *out_twist, void *stream) {
    const char *fn = "pvb_composed_query_scene_collision_cost";
    if (int rc = check_margin(fn, margin)) return rc;
    SceneLinks on;
    bool any_ext;
    if (int rc = scene_check_args(fn, scene, n_scene, scene_xforms, inv_xforms, n_sdf, n_cfg, cfg_begin, cfg_count,
                                  link_pts, K, links, out_cost, out_twist, on, any_ext))
        return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return comp_variant(false, any_ext, n_scene, [&](auto, auto kExt, auto kMaxS) {
        const DescPack<kMaxS> pack = desc_pack<kMaxS>(scene, n_scene);
        timing_mark(0, s);
        scene_collision_cost_kernel<kExt, kMaxS><<<(unsigned)cfg_count, kSceneLanes * kSceneWarps, 0, s>>>(
            pack, n_scene, scene_xforms, inv_xforms, n_sdf, n_cfg, cfg_begin, cfg_count, link_pts, (int)K, on, margin,
            out_cost, out_twist);
        timing_mark(1, s);
        PVB_CHECK_LAUNCH("pvb_composed_query_scene_collision_cost");
        return PVB_OK;
    });
}

extern "C" int pvb_composed_query_multi(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                        const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                        const float *pts, int64_t n_pts, uint32_t mesh_mode,
                                        const pvb_out_target *targets, int32_t n_targets, int32_t *out_which,
                                        void *stream) {
    if (!targets || n_targets < 1 || n_targets > PVB_MAX_TARGETS) {
        pvb_set_error("pvb_composed_query_multi: n_targets must be 1..%d (got %d)", PVB_MAX_TARGETS, n_targets);
        return PVB_ERR_INVALID;
    }
    OutTargets tg{};
    tg.n = n_targets;
    for (int t = 0; t < n_targets; ++t) {
        if (!targets[t].val || !targets[t].grad) {
            pvb_set_error("pvb_composed_query_multi: target %d has a null pointer", t);
            return PVB_ERR_INVALID;
        }
        tg.val[t] = targets[t].val;
        tg.grad[t] = targets[t].grad;
    }
    return composed_dispatch(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, mesh_mode,
                             tg.val[0], tg.grad[0], out_which, &tg, stream);
}

extern "C" int pvb_composed_query_multicast(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                            const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                            const float *pts, int64_t n_pts, uint32_t mesh_mode, float *mc_val,
                                            float *mc_grad, void *stream) {
    if (!mc_val || !mc_grad || ((uintptr_t)mc_val % 16) || ((uintptr_t)mc_grad % 16)) {
        pvb_set_error("pvb_composed_query_multicast: multicast addresses must be non-null and 16-byte aligned");
        return PVB_ERR_INVALID;
    }
    OutTargets tg{};
    tg.n = 1;
    tg.mc = 1;
    tg.val[0] = mc_val;
    tg.grad[0] = mc_grad;
    return composed_dispatch(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, mesh_mode,
                             mc_val, mc_grad, nullptr, &tg, stream);
}

// ------------------------------------------------------------------------------------------------ peer buffers
#define PVB_CUDA_TRY(call, what)                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess) {                                                                     \
            pvb_set_error("%s: %s", what, cudaGetErrorString(e_));                                   \
            return PVB_ERR_CUDA;                                                                     \
        }                                                                                            \
    } while (0)

extern "C" int pvb_ipc_alloc(int64_t bytes, void **out_ptr) {
    if (bytes < 1 || !out_ptr) { pvb_set_error("pvb_ipc_alloc: invalid argument"); return PVB_ERR_INVALID; }
    PVB_CUDA_TRY(cudaMalloc(out_ptr, (size_t)bytes), "pvb_ipc_alloc(cudaMalloc)");
    return PVB_OK;
}

extern "C" int pvb_ipc_free(void *ptr) {
    if (!ptr) return PVB_OK;
    PVB_CUDA_TRY(cudaFree(ptr), "pvb_ipc_free(cudaFree)");
    return PVB_OK;
}

extern "C" int pvb_ipc_export(void *ptr, unsigned char *handle) {
    static_assert(sizeof(cudaIpcMemHandle_t) == PVB_IPC_HANDLE_BYTES, "IPC handle size");
    if (!ptr || !handle) { pvb_set_error("pvb_ipc_export: invalid argument"); return PVB_ERR_INVALID; }
    cudaIpcMemHandle_t h;
    PVB_CUDA_TRY(cudaIpcGetMemHandle(&h, ptr), "pvb_ipc_export(cudaIpcGetMemHandle)");
    memcpy(handle, &h, sizeof(h));
    return PVB_OK;
}

extern "C" int pvb_ipc_open(const unsigned char *handle, void **out_ptr) {
    if (!handle || !out_ptr) { pvb_set_error("pvb_ipc_open: invalid argument"); return PVB_ERR_INVALID; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    PVB_CUDA_TRY(cudaIpcOpenMemHandle(out_ptr, h, cudaIpcMemLazyEnablePeerAccess), "pvb_ipc_open(cudaIpcOpenMemHandle)");
    return PVB_OK;
}

extern "C" int pvb_ipc_close(void *ptr) {
    if (!ptr) return PVB_OK;
    PVB_CUDA_TRY(cudaIpcCloseMemHandle(ptr), "pvb_ipc_close(cudaIpcCloseMemHandle)");
    return PVB_OK;
}

static int fill_voxel_geom(VoxelGeom &g, int32_t d, const double *min64, const double *res64, const int32_t *dims,
                           int32_t fp32_mode, const char *who) {
    if (d < 1 || d > 3 || !min64 || !res64 || !dims) {
        pvb_set_error("%s: 1 <= d <= 3 coordinates per point and non-null geometry required (d=%d)", who, d);
        return PVB_ERR_INVALID;
    }
    long long cells = 1;
    for (int a = 0; a < 3; ++a) {
        g.min64[a] = a < d ? min64[a] : 0.0;
        g.res64[a] = a < d ? res64[a] : 1.0;
        g.min32[a] = (float)g.min64[a];
        g.res32[a] = (float)g.res64[a];
        g.dims[a] = a < d ? dims[a] : 1;
        if (g.dims[a] < 1) { pvb_set_error("%s: empty grid axis %d", who, a); return PVB_ERR_INVALID; }
        cells *= g.dims[a];
    }
    (void)cells;
    g.d = d;
    g.fp32_mode = fp32_mode ? 1 : 0;
    return PVB_OK;
}

extern "C" int pvb_voxel_index(int32_t d, const double *min64, const double *res64, const int32_t *dims,
                               int32_t fp32_mode, const float *pts, int64_t n, int64_t *out_index, void *stream) {
    VoxelGeom g;
    if (int rc = fill_voxel_geom(g, d, min64, res64, dims, fp32_mode, "pvb_voxel_index")) return rc;
    if (n < 0 || (n > 0 && (!pts || !out_index))) { pvb_set_error("pvb_voxel_index: null argument"); return PVB_ERR_INVALID; }
    if (n == 0) return PVB_OK;
    voxel_index_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(g, pts, n, (long long *)out_index);
    PVB_CHECK_LAUNCH("pvb_voxel_index");
    return PVB_OK;
}

extern "C" int pvb_voxel_scatter(int32_t d, const double *min64, const double *res64, const int32_t *dims,
                                 int32_t fp32_mode, const float *pts, int64_t n, int32_t elem_bytes, const void *values,
                                 double scalar, void *data, void *stream) {
    VoxelGeom g;
    if (int rc = fill_voxel_geom(g, d, min64, res64, dims, fp32_mode, "pvb_voxel_scatter")) return rc;
    if (n < 0 || (n > 0 && (!pts || !data)) || (elem_bytes != 4 && elem_bytes != 1)) {
        pvb_set_error("pvb_voxel_scatter: invalid argument (elem_bytes must be 4 = float32 or 1 = bool/uint8)");
        return PVB_ERR_INVALID;
    }
    if (n == 0) return PVB_OK;
    const int blocks = grid_for(n, 256, 8);
    if (elem_bytes == 4)
        voxel_scatter_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(g, pts, n, (const float *)values,
                                                                              (float)scalar, (float *)data);
    else
        voxel_scatter_kernel<unsigned char><<<blocks, 256, 0, (cudaStream_t)stream>>>(
            g, pts, n, (const unsigned char *)values, (unsigned char)(scalar != 0.0), (unsigned char *)data);
    PVB_CHECK_LAUNCH("pvb_voxel_scatter");
    return PVB_OK;
}

extern "C" int pvb_voxel_gather(int32_t d, const double *min64, const double *res64, const int32_t *dims,
                                int32_t fp32_mode, const float *pts, int64_t n, int32_t elem_bytes, const void *data,
                                double invalid, void *out, uint8_t *out_valid, void *stream) {
    VoxelGeom g;
    if (int rc = fill_voxel_geom(g, d, min64, res64, dims, fp32_mode, "pvb_voxel_gather")) return rc;
    if (n < 0 || (n > 0 && (!pts || !data || !out)) || (elem_bytes != 4 && elem_bytes != 1)) {
        pvb_set_error("pvb_voxel_gather: invalid argument (elem_bytes must be 4 = float32 or 1 = bool/uint8)");
        return PVB_ERR_INVALID;
    }
    if (n == 0) return PVB_OK;
    const int blocks = grid_for(n, 256, 8);
    if (elem_bytes == 4)
        voxel_gather_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(g, pts, n, (const float *)data,
                                                                             (float)invalid, (float *)out, out_valid);
    else
        voxel_gather_kernel<unsigned char><<<blocks, 256, 0, (cudaStream_t)stream>>>(
            g, pts, n, (const unsigned char *)data, (unsigned char)(invalid != 0.0), (unsigned char *)out, out_valid);
    PVB_CHECK_LAUNCH("pvb_voxel_gather");
    return PVB_OK;
}

extern "C" int64_t pvb_compact_workspace(int64_t n) {
    return ((n + kCompactBlock - 1) / kCompactBlock) * 4 + 16;
}

extern "C" int pvb_compact_nonempty(const void *data, int64_t n, int32_t elem_bytes, double empty, void *workspace,
                                    int64_t capacity, int64_t *out_index, int64_t *out_count, void *stream) {
    if (n < 0 || !out_count || (n > 0 && (!data || !workspace)) || (elem_bytes != 4 && elem_bytes != 1) ||
        capacity < 0 || (capacity > 0 && !out_index) || n >= (1ll << 32)) {
        pvb_set_error("pvb_compact_nonempty: invalid argument");
        return PVB_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) {
        if (cudaMemsetAsync(out_count, 0, 8, s) != cudaSuccess) { pvb_set_error("pvb_compact_nonempty: memset failed"); return PVB_ERR_CUDA; }
        return PVB_OK;
    }
    const long long n_blocks = (n + kCompactBlock - 1) / kCompactBlock;
    unsigned int *counts = reinterpret_cast<unsigned int *>(workspace);
    if (elem_bytes == 4)
        compact_count_kernel<float><<<(unsigned)n_blocks, 256, 0, s>>>((const float *)data, n, (float)empty, counts);
    else
        compact_count_kernel<unsigned char><<<(unsigned)n_blocks, 256, 0, s>>>((const unsigned char *)data, n,
                                                                             (unsigned char)(empty != 0.0), counts);
    compact_scan_kernel<<<1, 1024, 0, s>>>(counts, n_blocks, (long long *)out_count);
    if (capacity > 0) {
        if (elem_bytes == 4)
            compact_write_kernel<float><<<(unsigned)n_blocks, 256, 0, s>>>((const float *)data, n, (float)empty, counts,
                                                                          capacity, (long long *)out_index);
        else
            compact_write_kernel<unsigned char><<<(unsigned)n_blocks, 256, 0, s>>>(
                (const unsigned char *)data, n, (unsigned char)(empty != 0.0), counts, capacity, (long long *)out_index);
    }
    PVB_CHECK_LAUNCH("pvb_compact_nonempty");
    return PVB_OK;
}

// The checks both forward-kinematics entry points make on their links and joint columns.  distinct_slots: every
// output slot written once (pvb_fk_tree; pvb_fk_serial keeps its own rule).
static int fk_check_links(const char *who, const pvb_fk_frame *frames, int n_frames, const pvb_fk_link *links,
                          int n_links, int n_joints, bool distinct_slots) {
    int prev = -1;
    bool taken[PVB_FK_TREE_MAX_LINKS] = {};
    for (int s = 0; s < n_links; ++s) {
        const pvb_fk_link &lk = links[s];
        if (lk.frame < prev || lk.frame < 0 || lk.frame >= n_frames || lk.slot < 0 || lk.slot >= n_links ||
            (distinct_slots && taken[lk.slot])) {
            pvb_set_error(distinct_slots ? "%s: links must be sorted by frame, with frame in [0, n_frames) and distinct "
                                           "slots in [0, n_links)"
                                         : "%s: links must be sorted by frame, with frame in [0, n_frames) and slot in "
                                           "[0, n_links)", who);
            return PVB_ERR_INVALID;
        }
        if (distinct_slots) taken[lk.slot] = true;
        prev = lk.frame;
    }
    for (int f = 0; f < n_frames; ++f) {
        const pvb_fk_frame &fr = frames[f];
        if (fr.joint_type != PVB_FK_FIXED && (fr.q_index < 0 || fr.q_index >= n_joints)) {
            pvb_set_error("%s: frame %d reads joint value %d of %d", who, f, fr.q_index, n_joints);
            return PVB_ERR_INVALID;
        }
    }
    return PVB_OK;
}

extern "C" int pvb_fk_serial(const pvb_fk_frame *frames, int32_t n_frames, const pvb_fk_link *links, int32_t n_links,
                             const float *q, int32_t n_cfg, int32_t n_joints, float *out_xforms, void *stream) {
    if (!frames || !links || n_frames < 1 || n_frames > PVB_FK_MAX_FRAMES || n_links < 1 || n_links > PVB_FK_MAX_LINKS ||
        n_cfg < 0 || n_joints < 0 || (n_cfg > 0 && (!out_xforms || (n_joints > 0 && !q)))) {
        pvb_set_error("pvb_fk_serial: invalid argument (n_frames=%d n_links=%d n_cfg=%d n_joints=%d)", n_frames, n_links,
                      n_cfg, n_joints);
        return PVB_ERR_INVALID;
    }
    if ((uintptr_t)out_xforms % 16) {
        pvb_set_error("pvb_fk_serial: out_xforms must be 16-byte aligned");
        return PVB_ERR_INVALID;
    }
    FkSerialPlan plan;
    memset(&plan, 0, sizeof(plan));
    plan.n_frames = n_frames;
    plan.n_links = n_links;
    memcpy(plan.frame, frames, sizeof(pvb_fk_frame) * (size_t)n_frames);
    memcpy(plan.link, links, sizeof(pvb_fk_link) * (size_t)n_links);
    if (fk_check_links("pvb_fk_serial", plan.frame, n_frames, plan.link, n_links, n_joints, false) != PVB_OK)
        return PVB_ERR_INVALID;
    if (n_cfg == 0) return PVB_OK;
    fk_serial_kernel<<<(n_cfg + kFkThreads - 1) / kFkThreads, kFkThreads, 0, (cudaStream_t)stream>>>(plan, q, n_cfg,
                                                                                                     n_joints, out_xforms);
    PVB_CHECK_LAUNCH("pvb_fk_serial");
    return PVB_OK;
}

extern "C" int pvb_fk_tree(const pvb_fk_frame *frames, const int32_t *parents, int32_t n_frames,
                           const pvb_fk_link *links, int32_t n_links, const float *q, int32_t n_cfg, int32_t n_joints,
                           float *out_xforms, void *stream) {
    if (!frames || !parents || !links || n_frames < 1 || n_frames > PVB_FK_TREE_MAX_FRAMES || n_links < 1 ||
        n_links > PVB_FK_TREE_MAX_LINKS || n_cfg < 0 || n_joints < 0 ||
        (n_cfg > 0 && (!out_xforms || (n_joints > 0 && !q)))) {
        pvb_set_error("pvb_fk_tree: invalid argument (n_frames=%d n_links=%d n_cfg=%d n_joints=%d)", n_frames, n_links,
                      n_cfg, n_joints);
        return PVB_ERR_INVALID;
    }
    if ((uintptr_t)out_xforms % 16) {
        pvb_set_error("pvb_fk_tree: out_xforms must be 16-byte aligned");
        return PVB_ERR_INVALID;
    }
    FkTreePlanMax plan;
    memset(&plan, 0, sizeof(plan));
    plan.n_frames = n_frames;
    plan.n_links = n_links;
    memcpy(plan.frame, frames, sizeof(pvb_fk_frame) * (size_t)n_frames);
    memcpy(plan.link, links, sizeof(pvb_fk_link) * (size_t)n_links);
    const int bad = fk_tree_slots(parents, n_frames, plan.load, plan.save, &plan.n_saves);
    if (bad >= 0) {
        pvb_set_error("pvb_fk_tree: frame %d has parent %d: parents must be a depth-first pre-order (parents[0] = -1, "
                      "and parents[f] is f - 1 or an ancestor of f - 1)", bad, parents[bad]);
        return PVB_ERR_INVALID;
    }
    if (fk_check_links("pvb_fk_tree", plan.frame, n_frames, plan.link, n_links, n_joints, true) != PVB_OK)
        return PVB_ERR_INVALID;
    if (n_cfg == 0) return PVB_OK;
    const size_t smem = sizeof(float) * 12 * kFkThreads * (size_t)plan.n_saves;
    if (smem > 48 * 1024)
        PVB_CUDA_TRY(cudaFuncSetAttribute(fk_tree_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     "pvb_fk_tree");
    fk_tree_kernel<<<(n_cfg + kFkThreads - 1) / kFkThreads, kFkThreads, smem, (cudaStream_t)stream>>>(plan, q, n_cfg,
                                                                                                      n_joints, out_xforms);
    PVB_CHECK_LAUNCH("pvb_fk_tree");
    return PVB_OK;
}

extern "C" int pvb_memcpy_async(void *dst, const void *src, int64_t bytes, void *stream) {
    if (bytes < 0 || (bytes > 0 && (!dst || !src))) { pvb_set_error("pvb_memcpy_async: invalid argument"); return PVB_ERR_INVALID; }
    if (bytes == 0) return PVB_OK;
    PVB_CUDA_TRY(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, (cudaStream_t)stream), "pvb_memcpy_async");
    return PVB_OK;
}

extern "C" int64_t pvb_chamfer_workspace(int64_t n_pts) {
    return (int64_t)grid_for(n_pts < 1 ? 1 : n_pts, kChamThreads, 4);
}

extern "C" int pvb_chamfer(const pvb_sdf_desc *obj, const float *world_to_object, int32_t n_tf, const float *pts,
                           int64_t n_pts, float scale, float *workspace, float *out, void *sort_workspace,
                           int64_t sort_workspace_bytes, void *stream) {
    if (!obj || !world_to_object || n_tf < 0 || n_pts < 1 || !pts || !workspace || !out) {
        pvb_set_error("pvb_chamfer: invalid argument");
        return PVB_ERR_INVALID;
    }
    if (obj->kind < PVB_KIND_GRID || obj->kind > PVB_KIND_CYLINDER) {
        pvb_set_error("pvb_chamfer: unknown kind %d", obj->kind);
        return PVB_ERR_INVALID;
    }
    if (obj->kind == PVB_KIND_MESH)
        if (int rc = check_mesh(obj, "pvb_chamfer")) return rc;
    if (obj->kind == PVB_KIND_GRID && (obj->flags & PVB_GRID_TRILINEAR)) {
        // the chamfer kernel evaluates grids with the nearest-voxel rule only; refuse rather than answer differently
        pvb_set_error("pvb_chamfer: PVB_GRID_TRILINEAR descriptors are not supported");
        return PVB_ERR_INVALID;
    }
    if (n_tf == 0) return PVB_OK;
    if (n_tf > 65535) {
        pvb_set_error("pvb_chamfer: at most 65535 transforms per call (got %d)", n_tf);
        return PVB_ERR_INVALID;
    }
    const int n_blk = (int)pvb_chamfer_workspace(n_pts);
    const int n_stage = obj->kind == PVB_KIND_MESH ? stage_nodes_for(obj->n_nodes) : 0;
    if (!ensure_smem(chamfer_partial_kernel, kSlotChamfer, kStageNodesMax * 128)) {
        pvb_set_error("pvb_chamfer: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
        return PVB_ERR_CUDA;
    }
    int rc = PVB_OK;
    // the cloud is binned in the object frame of the FIRST transform; the others are rigid too, so locality carries over
    SortedQueries sq{nullptr, nullptr, nullptr};
    if (obj->kind == PVB_KIND_MESH)
        sq = sort_queries(obj, pts, n_pts, world_to_object, sort_workspace,
                          (size_t)(sort_workspace_bytes < 0 ? 0 : sort_workspace_bytes), (cudaStream_t)stream, &rc);
    if (rc != PVB_OK) return rc;
    timing_mark(0, (cudaStream_t)stream);
    if (!sq.sorted) {
        chamfer_partial_kernel<<<dim3((unsigned)n_blk, (unsigned)n_tf), kChamThreads, (size_t)n_stage * 128,
                                 (cudaStream_t)stream>>>(*obj, world_to_object, pts, n_pts, nullptr, scale, n_stage,
                                                         workspace, nullptr);
        PVB_CHECK_LAUNCH("pvb_chamfer(partial)");
    } else {
        // binned: scaled distances of kChamSdPass transforms at a time in the result staging (16 B per point), then
        // the unbinned kernel's fixed-order sum over them
        float *sd = reinterpret_cast<float *>(sq.stage);
        for (int b0 = 0; b0 < n_tf; b0 += kChamSdPass) {
            const dim3 grid((unsigned)n_blk, (unsigned)(n_tf - b0 < kChamSdPass ? n_tf - b0 : kChamSdPass));
            chamfer_partial_kernel<<<grid, kChamThreads, (size_t)n_stage * 128, (cudaStream_t)stream>>>(
                *obj, world_to_object + (size_t)b0 * 16, pts, n_pts, sq.sorted, scale, n_stage, nullptr, sd);
            PVB_CHECK_LAUNCH("pvb_chamfer(partial)");
            chamfer_sum_kernel<<<grid, kChamThreads, 0, (cudaStream_t)stream>>>(sd, sq.inv, n_pts,
                                                                               workspace + (size_t)b0 * n_blk);
            PVB_CHECK_LAUNCH("pvb_chamfer(sum)");
        }
    }
    timing_mark(1, (cudaStream_t)stream);
    chamfer_finish_kernel<<<n_tf, 32, 0, (cudaStream_t)stream>>>(workspace, n_blk, n_pts, out);
    PVB_CHECK_LAUNCH("pvb_chamfer(finish)");
    return PVB_OK;
}

extern "C" int pvb_mesh_sample(const double *verts64, const int32_t *faces, int64_t n_faces, const int64_t *cum_counts,
                               int64_t n, uint64_t seed, double *out_pts, int32_t *out_face, void *stream) {
    if (!verts64 || !faces || !cum_counts || n_faces < 1 || n < 0 || (n > 0 && !out_pts)) {
        pvb_set_error("pvb_mesh_sample: invalid argument");
        return PVB_ERR_INVALID;
    }
    if (n == 0) return PVB_OK;
    mesh_sample_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(
        verts64, faces, n_faces, (const long long *)cum_counts, n, seed, out_pts, out_face);
    PVB_CHECK_LAUNCH("pvb_mesh_sample");
    return PVB_OK;
}

extern "C" int pvb_transform_points_paired(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts,
                                           float *out, void *stream) {
    if (!xforms || n_tf < 0 || n_pts < 0 || (n_tf > 0 && n_pts > 0 && (!pts || !out)) ||
        (n_tf > 0 && n_pts > INT64_MAX / 3 / n_tf)) {
        pvb_set_error("pvb_transform_points_paired: invalid argument");
        return PVB_ERR_INVALID;
    }
    if (n_tf == 0 || n_pts == 0) return PVB_OK;
    const long long n = (long long)n_tf * n_pts;
    transform_points_paired_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(xforms, pts, n_pts, n, out);
    PVB_CHECK_LAUNCH("pvb_transform_points_paired");
    return PVB_OK;
}

extern "C" int pvb_transform_points(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts, float *out,
                                    void *stream) {
    if (!xforms || n_tf < 0 || n_pts < 0 || (n_tf > 0 && n_pts > 0 && (!pts || !out)) ||
        (n_tf > 0 && n_pts > INT64_MAX / 3 / n_tf)) {
        pvb_set_error("pvb_transform_points: invalid argument");
        return PVB_ERR_INVALID;
    }
    if (n_tf == 0 || n_pts == 0) return PVB_OK;
    const long long n = (long long)n_tf * n_pts;
    transform_points_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(xforms, pts, n_pts, n, out);
    PVB_CHECK_LAUNCH("pvb_transform_points");
    return PVB_OK;
}

// ---------------------------------------------------------------- occupancy distance transform (OccupancySDF)
// Two transforms run side by side, blockIdx.y (or the word set) picking the state: 0 takes the occupied voxels as
// sites, 1 the free ones.  Each pass writes its EdtPairs for state t at [t * n_vox, (t + 1) * n_vox).
constexpr int kEdtWarps = 8;            // edt_z_kernel: one line per warp
constexpr int kEdtLineThreads = 128;    // edt_envelope_kernel: one line per thread

// Pass 1, along the contiguous z axis: a warp reads a line with coalesced byte loads, packs its occupancy into bit
// words with ballots (shared memory), then every lane looks up the nearest site of each state for its positions.
__global__ void __launch_bounds__(32 * kEdtWarps) edt_z_kernel(const unsigned char *__restrict__ occ, int nz,
                                                               long long n_lines, long long n_vox,
                                                               EdtPair *__restrict__ out) {
    __shared__ uint32_t words[kEdtWarps][2][kEdtMaxDim / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n_words = (nz + 31) >> 5;
    for (long long line = (long long)blockIdx.x * kEdtWarps + w; line < n_lines; line += (long long)gridDim.x * kEdtWarps) {
        const long long base = line * nz;
        for (int j = 0; j < n_words; ++j) {
            const int p = 32 * j + lane;
            const bool in = p < nz;
            const uint32_t mo = __ballot_sync(0xffffffffu, in && occ[base + p] != 0);
            const uint32_t mv = __ballot_sync(0xffffffffu, in);
            if (lane == 0) { words[w][0][j] = mo; words[w][1][j] = mv & ~mo; }
        }
        __syncwarp();
        for (int p = lane; p < nz; p += 32) {
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int r = edt_line_nearest(words[w][t], n_words, p);
                out[t * n_vox + base + p] = r < 0 ? EdtPair{-1, -1} : EdtPair{(p - r) * (p - r), (int)(base + r)};
            }
        }
        __syncwarp();
    }
}

// Passes 2 and 3: one thread per line of n voxels spaced `stride` apart (y: stride nz; x: stride ny nz), threads laid
// along the contiguous z coordinate so that every step's warp accesses are coalesced; the envelope stack of line t
// is stk[k * n_lines + t], coalesced the same way.
__global__ void __launch_bounds__(kEdtLineThreads) edt_envelope_kernel(const EdtPair *__restrict__ in,
                                                                       EdtPair *__restrict__ out,
                                                                       EdtPair *__restrict__ stk, int n,
                                                                       long long stride, long long n_lines,
                                                                       long long n_vox) {
    const long long t = (long long)blockIdx.x * kEdtLineThreads + threadIdx.x;
    if (t >= n_lines) return;
    const long long base = (t / stride) * (stride * n) + t % stride, off = (long long)blockIdx.y * n_vox;
    edt_envelope(in + off + base, out + off + base, stride, n, stk + off + t, n_lines);
}

// The outputs of voxel c from the transform of the other state: squared distance, site and table record.
__global__ void edt_record_kernel(const unsigned char *__restrict__ occ, const EdtPair *__restrict__ edt, int ny,
                                  int nz, long long n_vox, float r32, int32_t *__restrict__ out_sqdist,
                                  int32_t *__restrict__ out_site, float4 *__restrict__ out_table) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_vox; c += stride) {
        const bool o = occ[c] != 0;
        const EdtPair e = edt[(o ? n_vox : 0) + c];
        if (out_sqdist) out_sqdist[c] = e.d;
        if (out_site) out_site[c] = e.s;
        if (out_table) {
            const int ci = (int)c, cz = ci % nz, cy = (ci / nz) % ny, cx = ci / nz / ny;
            const int s = e.s < 0 ? 0 : e.s, sz = s % nz, sy = (s / nz) % ny, sx = s / nz / ny;
            out_table[c] = edt_record(e.d, o, cx, cy, cz, sx, sy, sz, r32);
        }
    }
}

static int edt_check_dims(const char *fn, const int32_t *dims) {
    if (!dims) { pvb_set_error("%s: invalid argument (dims is null)", fn); return PVB_ERR_INVALID; }
    for (int k = 0; k < 3; ++k) {
        if (dims[k] < 2 || dims[k] > kEdtMaxDim) {
            pvb_set_error("%s: every axis must hold 2..%d voxels (dims=[%d, %d, %d])", fn, kEdtMaxDim, dims[0],
                          dims[1], dims[2]);
            return PVB_ERR_INVALID;
        }
    }
    return PVB_OK;
}

extern "C" int64_t pvb_occupancy_sdf_workspace(const int32_t *dims) {
    if (edt_check_dims("pvb_occupancy_sdf_workspace", dims)) return -1;
    // two transforms x (pass buffer A, pass buffer B, envelope stacks), one EdtPair per voxel each
    return (int64_t)6 * (int64_t)sizeof(EdtPair) * dims[0] * dims[1] * dims[2];
}

extern "C" int pvb_occupancy_sdf(const uint8_t *occ, const int32_t *dims, float resolution, void *workspace,
                                 int64_t workspace_bytes, int32_t *out_sqdist, int32_t *out_site, float *out_table,
                                 void *stream) {
    const char *fn = "pvb_occupancy_sdf";
    if (int rc = edt_check_dims(fn, dims)) return rc;
    if (!(resolution > 0.f) || !isfinite(resolution)) {
        pvb_set_error("%s: the resolution must be finite and positive (resolution=%g)", fn, (double)resolution);
        return PVB_ERR_INVALID;
    }
    const int64_t need = pvb_occupancy_sdf_workspace(dims);
    if (!workspace || workspace_bytes < need || (uintptr_t)workspace % alignof(EdtPair)) {
        pvb_set_error("%s: the workspace must hold pvb_occupancy_sdf_workspace() = %lld bytes, 8-byte aligned "
                      "(got %lld bytes at %p)", fn, (long long)need, (long long)workspace_bytes, workspace);
        return PVB_ERR_INVALID;
    }
    if (!occ) { pvb_set_error("%s: invalid argument (occ is null)", fn); return PVB_ERR_INVALID; }
    if (!out_sqdist && !out_site && !out_table) {
        pvb_set_error("%s: invalid argument (out_sqdist, out_site and out_table are all null)", fn);
        return PVB_ERR_INVALID;
    }
    if ((uintptr_t)out_table % 16) {
        pvb_set_error("%s: out_table must be 16-byte aligned", fn);
        return PVB_ERR_INVALID;
    }
    const int nx = dims[0], ny = dims[1], nz = dims[2];
    const long long n_vox = (long long)nx * ny * nz;
    EdtPair *a = static_cast<EdtPair *>(workspace), *b = a + 2 * n_vox, *stk = b + 2 * n_vox;
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    const long long z_lines = (long long)nx * ny;
    edt_z_kernel<<<grid_for((z_lines + kEdtWarps - 1) / kEdtWarps, 1, 8), 32 * kEdtWarps, 0, s>>>(occ, nz, z_lines,
                                                                                                  n_vox, a);
    const long long y_lines = n_vox / ny, x_lines = n_vox / nx;
    edt_envelope_kernel<<<dim3((unsigned)((y_lines + kEdtLineThreads - 1) / kEdtLineThreads), 2), kEdtLineThreads, 0,
                          s>>>(a, b, stk, ny, nz, y_lines, n_vox);
    edt_envelope_kernel<<<dim3((unsigned)((x_lines + kEdtLineThreads - 1) / kEdtLineThreads), 2), kEdtLineThreads, 0,
                          s>>>(b, a, stk, nx, (long long)ny * nz, x_lines, n_vox);
    edt_record_kernel<<<grid_for(n_vox, 256, 8), 256, 0, s>>>(occ, a, ny, nz, n_vox, resolution, out_sqdist,
                                                              out_site, reinterpret_cast<float4 *>(out_table));
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}

// ---------------------------------------------------------------- depth images (depth_to_points, depth_occupancy)
// The view parameters travel as one __grid_constant__ parameter: per view {fx, fy, cx, cy} and the three rows of a
// rigid transform (camera -> world for the points, world -> camera for the carve).
struct DepthViews {
    float4 cam[kDepthMaxViews];
    float4 rows[kDepthMaxViews][3];
};
constexpr int kDepthMaxSide = 32768;
constexpr int kDepthThreads = 256;

// One thread per pixel, pixels in row-major order (the depth image's own layout).
__global__ void __launch_bounds__(kDepthThreads) depth_points_kernel(const float *__restrict__ depth, int H, int W,
                                                                    long long n_px,
                                                                    const __grid_constant__ DepthViews views,
                                                                    float max_depth, float *__restrict__ out) {
    const long long stride = (long long)gridDim.x * blockDim.x, hw = (long long)H * W;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_px; t += stride) {
        const int v = (int)(t / hw), pix = (int)(t - v * hw), i = pix / W, j = pix - i * W;
        const float d = depth[t];
        f3 p = mk3(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
        if (depth_valid(d, max_depth))
            p = depth_point(i, j, d, views.cam[v], views.rows[v][0], views.rows[v][1], views.rows[v][2]);
        out[3 * t] = p.x; out[3 * t + 1] = p.y; out[3 * t + 2] = p.z;
    }
}

// One thread per voxel, z fastest, so that neighbouring threads gather neighbouring pixels.  The view parameters are
// staged in shared memory once per block.  A voxel stops at its first free view: the result is an OR over the views.
__global__ void __launch_bounds__(kDepthThreads) depth_carve_kernel(const float *__restrict__ depth, int n_views,
                                                                   int H, int W,
                                                                   const __grid_constant__ DepthViews views,
                                                                   float max_depth, float margin, float lo_x,
                                                                   float lo_y, float lo_z, float r, int ny, int nz,
                                                                   long long n_vox, uint8_t *__restrict__ out) {
    __shared__ float4 s_cam[kDepthMaxViews], s_rows[kDepthMaxViews][3];
    for (int k = threadIdx.x; k < n_views; k += blockDim.x) {
        s_cam[k] = views.cam[k];
        s_rows[k][0] = views.rows[k][0]; s_rows[k][1] = views.rows[k][1]; s_rows[k][2] = views.rows[k][2];
    }
    __syncthreads();
    const float lo[3] = {lo_x, lo_y, lo_z};
    const long long stride = (long long)gridDim.x * blockDim.x, hw = (long long)H * W;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_vox; c += stride) {
        const int ci = (int)c, iz = ci % nz, iy = (ci / nz) % ny, ix = ci / nz / ny;
        const f3 x = depth_voxel_centre(lo, r, ix, iy, iz);
        uint8_t state = 2;
        for (int v = 0; v < n_views; ++v) {
            if (depth_says_free(depth + v * hw, H, W, s_cam[v], s_rows[v][0], s_rows[v][1], s_rows[v][2], x,
                                max_depth, margin)) {
                state = 0;
                break;
            }
        }
        out[c] = state;
    }
}

// The checks both entry points share; fills `views` from the HOST intrinsics and rows.
static int depth_check_views(const char *fn, const float *depth, int32_t V, int32_t H, int32_t W,
                             const float *intrinsics, const float *rows, float max_depth, DepthViews &views) {
    if (V < 1 || V > kDepthMaxViews || H < 1 || H > kDepthMaxSide || W < 1 || W > kDepthMaxSide) {
        pvb_set_error("%s: V must be 1..%d and H, W 1..%d (V=%d, H=%d, W=%d)", fn, kDepthMaxViews, kDepthMaxSide, V,
                      H, W);
        return PVB_ERR_INVALID;
    }
    if (!depth || !intrinsics || !rows) {
        pvb_set_error("%s: invalid argument (depth, intrinsics or the transforms are null)", fn);
        return PVB_ERR_INVALID;
    }
    if (!(max_depth > 0.f)) {
        pvb_set_error("%s: max_depth must be positive (max_depth=%g)", fn, (double)max_depth);
        return PVB_ERR_INVALID;
    }
    for (int v = 0; v < V; ++v) {
        const float *k = intrinsics + 4 * v;
        if (!(k[0] > 0.f && k[1] > 0.f) || !isfinite(k[0]) || !isfinite(k[1]) || !isfinite(k[2]) || !isfinite(k[3])) {
            pvb_set_error("%s: view %d: the focal lengths must be finite and positive and the principal point finite "
                          "(fx=%g, fy=%g, cx=%g, cy=%g)", fn, v, (double)k[0], (double)k[1], (double)k[2],
                          (double)k[3]);
            return PVB_ERR_INVALID;
        }
        for (int e = 0; e < 12; ++e) {
            if (!isfinite(rows[12 * v + e])) {
                pvb_set_error("%s: view %d: the transform is not finite", fn, v);
                return PVB_ERR_INVALID;
            }
        }
        views.cam[v] = make_float4(k[0], k[1], k[2], k[3]);
        for (int q = 0; q < 3; ++q) {
            const float *m = rows + 12 * v + 4 * q;
            views.rows[v][q] = make_float4(m[0], m[1], m[2], m[3]);
        }
    }
    return PVB_OK;
}

extern "C" int pvb_depth_points(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                                const float *cam_to_world, float max_depth, float *out_points, void *stream) {
    const char *fn = "pvb_depth_points";
    DepthViews views = {};
    if (int rc = depth_check_views(fn, depth, V, H, W, intrinsics, cam_to_world, max_depth, views)) return rc;
    if (!out_points) { pvb_set_error("%s: invalid argument (out_points is null)", fn); return PVB_ERR_INVALID; }
    const long long n_px = (long long)V * H * W;
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    depth_points_kernel<<<grid_for(n_px, kDepthThreads, 8), kDepthThreads, 0, s>>>(depth, H, W, n_px, views,
                                                                                   max_depth, out_points);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}

extern "C" int pvb_depth_carve(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                               const float *world_to_cam, float max_depth, float free_margin, const float *lo,
                               float resolution, const int32_t *dims, uint8_t *out_state, void *stream) {
    const char *fn = "pvb_depth_carve";
    DepthViews views = {};
    if (int rc = depth_check_views(fn, depth, V, H, W, intrinsics, world_to_cam, max_depth, views)) return rc;
    if (int rc = edt_check_dims(fn, dims)) return rc;
    if (!(resolution > 0.f) || !isfinite(resolution)) {
        pvb_set_error("%s: the resolution must be finite and positive (resolution=%g)", fn, (double)resolution);
        return PVB_ERR_INVALID;
    }
    if (!(free_margin >= 0.f) || !isfinite(free_margin)) {
        pvb_set_error("%s: free_margin must be finite and non-negative (free_margin=%g)", fn, (double)free_margin);
        return PVB_ERR_INVALID;
    }
    if (!lo || !out_state) { pvb_set_error("%s: invalid argument (lo or out_state is null)", fn); return PVB_ERR_INVALID; }
    if (!isfinite(lo[0]) || !isfinite(lo[1]) || !isfinite(lo[2])) {
        pvb_set_error("%s: the lattice origin lo must be finite", fn);
        return PVB_ERR_INVALID;
    }
    const long long n_vox = (long long)dims[0] * dims[1] * dims[2];
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    depth_carve_kernel<<<grid_for(n_vox, kDepthThreads, 8), kDepthThreads, 0, s>>>(
        depth, V, H, W, views, max_depth, free_margin, lo[0], lo[1], lo[2], resolution, dims[1], dims[2], n_vox,
        out_state);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}

// ---------------------------------------------------------------- occupancy maps (OccupancyMap.integrate)
// depth_carve_kernel's layout: one thread per voxel, z fastest, the views staged in shared memory once per block.  A
// voxel a valid pixel's point fell into (its hit byte, set by pvb_voxel_scatter) is a hit and skips the views; any
// other voxel runs the views up to the first that says free.  The update is applied in place, and the hit byte is
// cleared, so the scratch grid is zero again for the next call without a memset.
__global__ void __launch_bounds__(kDepthThreads) depth_integrate_kernel(const float *__restrict__ depth, int n_views,
                                                                       int H, int W,
                                                                       const __grid_constant__ DepthViews views,
                                                                       float max_depth, float margin, float lo_x,
                                                                       float lo_y, float lo_z, float r, int ny, int nz,
                                                                       long long n_vox, OccupancyParams params,
                                                                       uint8_t *__restrict__ hits,
                                                                       int16_t *__restrict__ log_odds) {
    __shared__ float4 s_cam[kDepthMaxViews], s_rows[kDepthMaxViews][3];
    for (int k = threadIdx.x; k < n_views; k += blockDim.x) {
        s_cam[k] = views.cam[k];
        s_rows[k][0] = views.rows[k][0]; s_rows[k][1] = views.rows[k][1]; s_rows[k][2] = views.rows[k][2];
    }
    __syncthreads();
    const float lo[3] = {lo_x, lo_y, lo_z};
    const long long stride = (long long)gridDim.x * blockDim.x, hw = (long long)H * W;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_vox; c += stride) {
        const bool hit = hits[c] != 0;
        bool free = false;
        if (!hit) {
            const int ci = (int)c, iz = ci % nz, iy = (ci / nz) % ny, ix = ci / nz / ny;
            const f3 x = depth_voxel_centre(lo, r, ix, iy, iz);
            for (int v = 0; v < n_views && !free; ++v)
                free = depth_says_free(depth + v * hw, H, W, s_cam[v], s_rows[v][0], s_rows[v][1], s_rows[v][2], x,
                                       max_depth, margin);
        }
        if (hit || free) log_odds[c] = (int16_t)occupancy_update(log_odds[c], hit, free, params);
        if (hit) hits[c] = 0;
    }
}

extern "C" int pvb_depth_integrate(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                                   const float *world_to_cam, float max_depth, float free_margin, const float *lo,
                                   float resolution, const int32_t *dims, uint8_t *hits, int16_t *log_odds,
                                   const int32_t *params, void *stream) {
    const char *fn = "pvb_depth_integrate";
    DepthViews views = {};
    if (int rc = depth_check_views(fn, depth, V, H, W, intrinsics, world_to_cam, max_depth, views)) return rc;
    if (int rc = edt_check_dims(fn, dims)) return rc;
    if (!(resolution > 0.f) || !isfinite(resolution)) {
        pvb_set_error("%s: the resolution must be finite and positive (resolution=%g)", fn, (double)resolution);
        return PVB_ERR_INVALID;
    }
    if (!(free_margin >= 0.f) || !isfinite(free_margin)) {
        pvb_set_error("%s: free_margin must be finite and non-negative (free_margin=%g)", fn, (double)free_margin);
        return PVB_ERR_INVALID;
    }
    if (!lo || !hits || !log_odds || !params) {
        pvb_set_error("%s: invalid argument (lo, hits, log_odds or params is null)", fn);
        return PVB_ERR_INVALID;
    }
    if (!isfinite(lo[0]) || !isfinite(lo[1]) || !isfinite(lo[2])) {
        pvb_set_error("%s: the lattice origin lo must be finite", fn);
        return PVB_ERR_INVALID;
    }
    const OccupancyParams p = {params[0], params[1], params[2], params[3]};
    if (!(-32767 <= p.clamp_lo && p.clamp_lo <= p.miss && p.miss < 0 && 0 < p.hit && p.hit <= p.clamp_hi &&
          p.clamp_hi <= 32767)) {
        pvb_set_error("%s: the parameters must satisfy -32767 <= clamp_lo <= miss < 0 < hit <= clamp_hi <= 32767 "
                      "(hit=%d, miss=%d, clamp_lo=%d, clamp_hi=%d)", fn, p.hit, p.miss, p.clamp_lo, p.clamp_hi);
        return PVB_ERR_INVALID;
    }
    const long long n_vox = (long long)dims[0] * dims[1] * dims[2];
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    depth_integrate_kernel<<<grid_for(n_vox, kDepthThreads, 8), kDepthThreads, 0, s>>>(
        depth, V, H, W, views, max_depth, free_margin, lo[0], lo[1], lo[2], resolution, dims[1], dims[2], n_vox, p,
        hits, log_odds);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}

// ---------------------------------------------------------------- ray-cast point clouds (OccupancyMap.integrate_points)
constexpr int kRayThreads = 256;

// One thread per ray on a grid-stride loop: ray_valid, then out_points, then ray_walk writes 2 on every voxel of the
// free segment.  Every write stores the same value, so the marks depend on neither the ray order nor the thread order.
__global__ void __launch_bounds__(kRayThreads) ray_carve_kernel(const float *__restrict__ points, long long n_rays,
                                                                long long per_origin,
                                                                const float *__restrict__ origins, float max_range,
                                                                float margin, float lo_x, float lo_y, float lo_z,
                                                                float r, int nx, int ny, int nz,
                                                                uint8_t *__restrict__ marks, float *__restrict__ out) {
    const float lo[3] = {lo_x, lo_y, lo_z};
    const int n[3] = {nx, ny, nz};
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_rays; t += stride) {
        const float *q = origins + 3 * (t / per_origin);
        const f3 o = mk3(__ldg(q), __ldg(q + 1), __ldg(q + 2));
        const f3 p = mk3(points[3 * t], points[3 * t + 1], points[3 * t + 2]);
        f3 d;
        float len;
        const bool valid = ray_valid(o, p, max_range, d, len);
        const float nan = __int_as_float(0x7fc00000);
        out[3 * t] = valid ? p.x : nan; out[3 * t + 1] = valid ? p.y : nan; out[3 * t + 2] = valid ? p.z : nan;
        if (valid)
            ray_walk(o, d, len, margin, lo, r, n, [&](int ix, int iy, int iz) {
                marks[((long long)ix * ny + iy) * nz + iz] = 2;
            });
    }
}

// One thread per voxel: mark 1 is a hit, 2 a free observation, 0 nothing (occupancy_update); every mark is cleared.
__global__ void __launch_bounds__(256) occupancy_apply_kernel(uint8_t *__restrict__ marks,
                                                              int16_t *__restrict__ log_odds, long long n_vox,
                                                              OccupancyParams params) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_vox; c += stride) {
        const uint8_t m = marks[c];
        if (m == 0) continue;
        log_odds[c] = (int16_t)occupancy_update(log_odds[c], m == 1, m == 2, params);
        marks[c] = 0;
    }
}

extern "C" int pvb_ray_carve(const float *points, int64_t n_rays, int64_t rays_per_origin, const float *origins,
                             float max_range, float free_margin, const float *lo, float resolution,
                             const int32_t *dims, uint8_t *marks, float *out_points, void *stream) {
    const char *fn = "pvb_ray_carve";
    if (!points || !origins || !lo || !marks || !out_points) {
        pvb_set_error("%s: invalid argument (points, origins, lo, marks or out_points is null)", fn);
        return PVB_ERR_INVALID;
    }
    if (n_rays < 1 || n_rays >= ((int64_t)1 << 31) || rays_per_origin < 1 || n_rays % rays_per_origin) {
        pvb_set_error("%s: n_rays must be 1..2^31 - 1 and a multiple of rays_per_origin >= 1 (n_rays=%lld, "
                      "rays_per_origin=%lld)", fn, (long long)n_rays, (long long)rays_per_origin);
        return PVB_ERR_INVALID;
    }
    if (!(max_range > 0.f)) {
        pvb_set_error("%s: max_range must be positive (max_range=%g)", fn, (double)max_range);
        return PVB_ERR_INVALID;
    }
    if (int rc = edt_check_dims(fn, dims)) return rc;
    if (!(resolution > 0.f) || !isfinite(resolution)) {
        pvb_set_error("%s: the resolution must be finite and positive (resolution=%g)", fn, (double)resolution);
        return PVB_ERR_INVALID;
    }
    if (!(free_margin >= 0.f) || !isfinite(free_margin)) {
        pvb_set_error("%s: free_margin must be finite and non-negative (free_margin=%g)", fn, (double)free_margin);
        return PVB_ERR_INVALID;
    }
    if (!isfinite(lo[0]) || !isfinite(lo[1]) || !isfinite(lo[2])) {
        pvb_set_error("%s: the lattice origin lo must be finite", fn);
        return PVB_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    ray_carve_kernel<<<grid_for(n_rays, kRayThreads, 8), kRayThreads, 0, s>>>(
        points, n_rays, rays_per_origin, origins, max_range, free_margin, lo[0], lo[1], lo[2], resolution, dims[0],
        dims[1], dims[2], marks, out_points);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}

extern "C" int pvb_occupancy_apply(uint8_t *marks, int16_t *log_odds, const int32_t *dims, const int32_t *params,
                                   void *stream) {
    const char *fn = "pvb_occupancy_apply";
    if (int rc = edt_check_dims(fn, dims)) return rc;
    if (!marks || !log_odds || !params) {
        pvb_set_error("%s: invalid argument (marks, log_odds or params is null)", fn);
        return PVB_ERR_INVALID;
    }
    const OccupancyParams p = {params[0], params[1], params[2], params[3]};
    if (!(-32767 <= p.clamp_lo && p.clamp_lo <= p.miss && p.miss < 0 && 0 < p.hit && p.hit <= p.clamp_hi &&
          p.clamp_hi <= 32767)) {
        pvb_set_error("%s: the parameters must satisfy -32767 <= clamp_lo <= miss < 0 < hit <= clamp_hi <= 32767 "
                      "(hit=%d, miss=%d, clamp_lo=%d, clamp_hi=%d)", fn, p.hit, p.miss, p.clamp_lo, p.clamp_hi);
        return PVB_ERR_INVALID;
    }
    const long long n_vox = (long long)dims[0] * dims[1] * dims[2];
    cudaStream_t s = (cudaStream_t)stream;
    timing_mark(0, s);
    occupancy_apply_kernel<<<grid_for(n_vox, 256, 8), 256, 0, s>>>(marks, log_odds, n_vox, p);
    timing_mark(1, s);
    PVB_CHECK_LAUNCH(fn);
    return PVB_OK;
}
