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
       kSlotCount };
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
// EXTENSION, opt-in (CachedSDF(interpolation="trilinear")): the reference looks up the NEAREST voxel and a stored
// gradient table (sdf.py:537-550), which is what every other kernel in this file reproduces.  This one
// interpolates the value table trilinearly and returns the analytic gradient of the interpolant (per-cell finite
// differences of the corner values) -- smoother for optimisation, not comparable to the reference within 1e-5
// (the difference is O(resolution)); it is validated against its own CPU restatement (oracle/port.py).
__global__ void __launch_bounds__(256)
grid_trilinear_kernel(const pvb_sdf_desc g, const float *__restrict__ pts, long long n, float *__restrict__ out_val,
                      float *__restrict__ out_grad) {
    const float4 *tab = reinterpret_cast<const float4 *>(g.table);
    const long long stride = (long long)gridDim.x * blockDim.x;
    const int n0 = g.dims[0], n1 = g.dims[1], n2 = g.dims[2];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const f3 p = load_point(pts, i);
        const bool inb = (p.x >= g.valid_lo[0]) & (p.x <= g.valid_hi[0]) & (p.y >= g.valid_lo[1]) &
                         (p.y <= g.valid_hi[1]) & (p.z >= g.valid_lo[2]) & (p.z <= g.valid_hi[2]);
        SdfOut o;
        if (inb) {
            const float u[3] = {(p.x - g.min32[0]) * g.inv_res32[0], (p.y - g.min32[1]) * g.inv_res32[1],
                                (p.z - g.min32[2]) * g.inv_res32[2]};
            const int nn[3] = {n0, n1, n2};
            int c0[3];
            float f[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                c0[a] = min(max((int)floorf(u[a]), 0), max(nn[a] - 2, 0));
                f[a] = nn[a] > 1 ? fminf(fmaxf(u[a] - (float)c0[a], 0.f), 1.f) : 0.f;
            }
            const int s0 = n1 * n2, s1 = n2;
            const int base = c0[0] * s0 + c0[1] * s1 + c0[2];
            const int dx = n0 > 1 ? s0 : 0, dy = n1 > 1 ? s1 : 0, dz = n2 > 1 ? 1 : 0;
            const float v000 = __ldg(tab + base).x, v001 = __ldg(tab + base + dz).x;
            const float v010 = __ldg(tab + base + dy).x, v011 = __ldg(tab + base + dy + dz).x;
            const float v100 = __ldg(tab + base + dx).x, v101 = __ldg(tab + base + dx + dz).x;
            const float v110 = __ldg(tab + base + dx + dy).x, v111 = __ldg(tab + base + dx + dy + dz).x;
            const float fx = f[0], fy = f[1], fz = f[2];
            const float c00 = v000 + fz * (v001 - v000), c01 = v010 + fz * (v011 - v010);
            const float c10 = v100 + fz * (v101 - v100), c11 = v110 + fz * (v111 - v110);
            const float c0_ = c00 + fy * (c01 - c00), c1_ = c10 + fy * (c11 - c10);
            o.val = c0_ + fx * (c1_ - c0_);
            // d/dx: difference of the two y-z interpolated faces over the cell size, and likewise for y, z
            const float gx = (c1_ - c0_) * g.inv_res32[0];
            const float e0 = c01 - c00, e1 = c11 - c10;
            const float gy = (e0 + fx * (e1 - e0)) * g.inv_res32[1];
            const float z00 = v001 - v000, z01 = v011 - v010, z10 = v101 - v100, z11 = v111 - v110;
            const float z0 = z00 + fy * (z01 - z00), z1 = z10 + fy * (z11 - z10);
            const float gz = (z0 + fx * (z1 - z0)) * g.inv_res32[2];
            o.grad = mk3(n0 > 1 ? gx : 0.f, n1 > 1 ? gy : 0.f, n2 > 1 ? gz : 0.f);
        } else {
            float dist, ex, ey, ez, r;        // out of range: the reference's AABB rule, unchanged
            aabb_rule(g, p, dist, ex, ey, ez, r);
            o.val = dist;
            o.grad = mk3(ex * r, ey * r, ez * r);
        }
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

template <bool kMesh, int PTS, int MAXS, bool kMulti>
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
                    const float4 *row = reinterpret_cast<const float4 *>(xforms + ((size_t)s * n_cfg + cfg) * 16);
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
                        const bool bounded = d.kind == PVB_KIND_GRID ? (d.flags & PVB_GRID_PRUNE_OK) != 0
                                             : (d.kind == PVB_KIND_MESH && (d.flags & PVB_MESH_CLOSED) && (mesh_mode & PVB_MESH_SIGNED));
                        key[s] = bounded ? composed_aabb_lb2(d, composed_xform(r0, r1, r2, p[0])) : -1.f;
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
                        composed_consider<kMesh>(d, st, s, composed_xform(r0, r1, r2, p[0]), mesh_mode, idx, best[0], bg[0], bs[0]);
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
                    composed_consider<kMesh>(d, st, s, composed_xform(r0, r1, r2, p[k]), mesh_mode, idx, best[k], bg[k],
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

template <bool kMulti>
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
        const bool ok = d.kind == PVB_KIND_GRID && (d.flags & PVB_GRID_PRUNE_OK) && dev < 1e-5f;
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
                composed_consider<false>(d, st, s, composed_xform(r0, r1, r2, p[k]), 0u, 0ull, best[k], bg[k], bs[k]);
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

// Everything that is not "in range, fp32 index estimate certain" -- the exact index of a point inside a cell
// boundary's uncertainty band, or the point-to-AABB rule of an out-of-range point -- out of line and through a
// pointer to the descriptor in parameter space: rare, and 32 inlined copies of it (4 points x 8 unrolled links) were
// two thirds of the kernel's code.
__device__ __noinline__ float4 robot_lookup_slow(const pvb_sdf_desc *dp, float qx, float qy, float qz) {
    const pvb_sdf_desc &d = *dp;
    NodeStage st; st.smem = nullptr; st.n = 0;
    const SdfOut o = grid_eval<false, true>(d, st, mk3(qx, qy, qz), 0u, 0ull, nullptr);
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

// In-range + certain: the record of the nearest voxel, same arithmetic as grid_eval (pvb_device.cuh).
__device__ __forceinline__ float4 robot_lookup(const pvb_sdf_desc &g, f3 p) {
    const float kMagic = 12582912.f;   // 1.5 * 2^23
    const float qx = (p.x - g.min32[0]) * g.inv_res32[0];
    const float qy = (p.y - g.min32[1]) * g.inv_res32[1];
    const float qz = (p.z - g.min32[2]) * g.inv_res32[2];
    const float mx = __fadd_rn(qx, kMagic), my = __fadd_rn(qy, kMagic), mz = __fadd_rn(qz, kMagic);
    const int kx = __float_as_int(mx) - 0x4B400000, ky = __float_as_int(my) - 0x4B400000,
              kz = __float_as_int(mz) - 0x4B400000;
    const bool certain = (fabsf(qx - __fsub_rn(mx, kMagic)) <= g.idx_certain[0]) &
                         (fabsf(qy - __fsub_rn(my, kMagic)) <= g.idx_certain[1]) &
                         (fabsf(qz - __fsub_rn(mz, kMagic)) <= g.idx_certain[2]);
    const bool inb = (p.x >= g.valid_lo[0]) & (p.x <= g.valid_hi[0]) & (p.y >= g.valid_lo[1]) &
                     (p.y <= g.valid_hi[1]) & (p.z >= g.valid_lo[2]) & (p.z <= g.valid_hi[2]);
    if (inb & certain)      // the index is exact and inside the table: no clamp needed
        return __ldg(reinterpret_cast<const float4 *>(g.table) + ((kx * g.dims[1] + ky) * g.dims[2] + kz));
    return robot_lookup_slow(&g, p.x, p.y, p.z);
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
// wavefronts (~166 per point: 32 sphere reads, ~54 transform rows, ~66 table gathers of 32 distinct sectors, 12 staging)
// and issue slots.
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

struct __align__(16) RsSmem {
    float4 xf[kRbCfg][3 * kRsMaxS + 1];
    float4 sph[kRbCfg][kRsMaxS + 1];
    // per-warp staging, LC rows x (8 * 32/LC values + 1) resp. (24 * 32/LC gradient floats + 1): at most 32 x 9 / 32 x 25
    float sv[kRsWarps][kRbCfg][kRsValStride];
    float sg[kRsWarps][kRbCfg][kRsGradStride];
};

// sqrt(0.9998) * 0.999999: 0.9998 on the squared distance absorbs the 1e-5 non-rigidity tolerated below, 0.999999 the
// approximate reciprocal square root (2 ulp) and the roundings of the three fused multiply-adds
constexpr float kRsBoundScale = 0.99989899f;

__device__ __forceinline__ float rsqrt_approx(float x) {      // one MUFU.RSQ, no denormal fix-up (callers keep x >= 1e-20)
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// (configuration tiles and the flush index arithmetic: rs_tile / rs_flush_piece in pvb_device.cuh, checked on the CPU tier)
template <int kDest>
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
    // ---- bounding spheres (object frame) of every (configuration, link) of the tile ----
    for (int item = threadIdx.x; item < LC * kRsMaxS; item += blockDim.x) {
        const int ci = item & (LC - 1), si = item >> lc_log2;
        // slots beyond n_sdf: radius -inf, so that their bound is +inf -- never the nearest, never visited
        float4 sp = make_float4(0.f, 0.f, 0.f, -PVB_INF);
        if (si < n_sdf) {
            const pvb_sdf_desc &d = pk.d[si];
            const float4 r0 = sm.xf[ci][3 * si], r1 = sm.xf[ci][3 * si + 1], r2 = sm.xf[ci][3 * si + 2];
            // sphere around the link AABB, centre carried to the object frame: c_obj = R^T (c_link - t)
            const f3 cen = mk3(0.5f * (d.bb_min[0] + d.bb_max[0]), 0.5f * (d.bb_min[1] + d.bb_max[1]),
                               0.5f * (d.bb_min[2] + d.bb_max[2]));
            const f3 hl = mk3(0.5f * (d.bb_max[0] - d.bb_min[0]), 0.5f * (d.bb_max[1] - d.bb_min[1]),
                              0.5f * (d.bb_max[2] - d.bb_min[2]));
            const f3 u = mk3(cen.x - r0.w, cen.y - r1.w, cen.z - r2.w);
            const f3 co = mk3(r0.x * u.x + r1.x * u.y + r2.x * u.z, r0.y * u.x + r1.y * u.y + r2.y * u.z,
                              r0.z * u.x + r1.z * u.y + r2.z * u.z);
            const float rad = sqrtf(hl.x * hl.x + hl.y * hl.y + hl.z * hl.z) * 1.0001f + 1e-6f;
            // the bound needs an isometry: |R R^T - I| must vanish, otherwise this (cfg, link) is never rejected by it
            const float e00 = r0.x * r0.x + r0.y * r0.y + r0.z * r0.z - 1.f, e11 = r1.x * r1.x + r1.y * r1.y + r1.z * r1.z - 1.f,
                        e22 = r2.x * r2.x + r2.y * r2.y + r2.z * r2.z - 1.f;
            const float e01 = r0.x * r1.x + r0.y * r1.y + r0.z * r1.z, e02 = r0.x * r2.x + r0.y * r2.y + r0.z * r2.z,
                        e12 = r1.x * r2.x + r1.y * r2.y + r1.z * r2.z;
            const float dev = fmaxf(fmaxf(fmaxf(fabsf(e00), fabsf(e11)), fmaxf(fabsf(e22), fabsf(e01))),
                                    fmaxf(fabsf(e02), fabsf(e12)));
            const bool ok = (d.flags & PVB_GRID_PRUNE_OK) && dev < 1e-5f;
            sp = make_float4(co.x, co.y, co.z, ok ? rad + d.prune_margin : PVB_INF);
        }
        sm.sph[ci][si] = sp;
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
    // ~7 in a register the compiler cannot fold (n_sdf <= 8): (bits & ~7) | si is then ONE LOP3 with the immediate si
    const int low3_off = ~7 | (n_sdf >> 30);
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
            // ---- lower bounds of every link's value from its bounding sphere: value_s >= |p - c_s| - radius_s.
            // 0.9998 absorbs the 1e-5 non-rigidity tolerated above, 0.999999 the approximate reciprocal square root
            // (2 ulp); + 1e-20 keeps its argument a normal number (and raises the bound by < 1e-10, inside the 1e-5
            // slack of the radius).  radius = inf (bound not valid) gives -inf: never rejected.
            float lb[kRsMaxS], key[kRsMaxS];
#pragma unroll
            for (int si = 0; si < kRsMaxS; ++si) {
                const float4 sp = sm.sph[cl][si];
                const float dx = p.x - sp.x, dy = p.y - sp.y, dz = p.z - sp.z;
                const float d2 = fmaf(dz, dz, fmaf(dy, dy, fmaf(dx, dx, 1e-20f)));
                lb[si] = fmaf(d2 * rsqrt_approx(d2), kRsBoundScale, -sp.w);
                key[si] = rs_bound_key(lb[si], low3_off, si);       // link index in the 3 low mantissa bits
            }
            // one visiting order per point group: its first lane's nearest sphere (neighbouring configurations agree;
            // rs_nearest in pvb_device.cuh: any link is a valid first visit, the order never changes a result)
            const int pred = __shfl_sync(0xffffffffu, rs_nearest(key, n_sdf), sub << lc_log2);
            float best = PVB_INF;
            f3 bg = mk3(0.f, 0.f, 0.f);
            int bs = -1;
            // one link: transform, AABB bound against the running minimum, nearest-voxel lookup, running argmin
            auto visit = [&](const pvb_sdf_desc &d, const int si) {
                const float4 r0 = sm.xf[cl][3 * si], r1 = sm.xf[cl][3 * si + 1], r2 = sm.xf[cl][3 * si + 2];
                const f3 q = composed_xform(r0, r1, r2, p);
                if ((d.flags & PVB_GRID_PRUNE_OK) && bs >= 0) {
                    const float thr = best + d.prune_margin;
                    if (thr < 0.f || composed_aabb_lb2(d, q) > thr * thr) return;
                }
                const float4 o = robot_lookup(d, q);
                if (bs < 0 || o.x < best || (o.x == best && si < bs)) {
                    best = o.x; bg = mk3(o.y, o.z, o.w); bs = si;
                }
            };
            // (lanes past the last point work on p = 0 and are not stored: no `on` in the conditions below)
            visit(pk.d[pred], pred);
#pragma unroll
            for (int si = 0; si < kRsMaxS; ++si) {
                // reject when the sphere bound already exceeds the running minimum (exact: lb <= value); best is finite
                // after the first visit, so the +inf bound of a slot beyond n_sdf never passes
                if (si != pred && !(lb[si] > best)) visit(pk.d[si], si);
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
// RobotSDF.set_joint_configuration (model_to_sdf.py:82-115): for every joint configuration a and every mesh link s,
// the object->mesh-frame transform (FK_s(q_a) @ visual_offset_s)^-1 = offset_s^-1 @ FK_s(q_a)^-1, written link-major
// (row s * A + a) as the 4x4 row-major matrices the composed kernels read.  One thread per configuration walks the
// serial chain in registers: T <- T @ joint_origin @ motion(q_j) (revolute: Rodrigues rotation about the axis,
// prismatic: translation along it, fixed: identity), the same fp32 products the eager path took as dozens of small
// launches (this kernel: one launch for every configuration).
struct FkPlan {
    pvb_fk_frame frame[PVB_FK_MAX_FRAMES];
    pvb_fk_link link[PVB_FK_MAX_LINKS];
    int n_frames, n_links;
};

struct Rt34 { float m[12]; };       // rows of [R | t]

__device__ __forceinline__ Rt34 rt_mul(const Rt34 &a, const float *b) {       // a @ b, both [R | t] with last row 0 0 0 1
    Rt34 o;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float v = a.m[4 * r] * b[c] + a.m[4 * r + 1] * b[4 + c] + a.m[4 * r + 2] * b[8 + c];
            if (c == 3) v += a.m[4 * r + 3];
            o.m[4 * r + c] = v;
        }
    }
    return o;
}

__global__ void fk_serial_kernel(const __grid_constant__ FkPlan plan, const float *__restrict__ q, int n_cfg,
                                 int n_joints, float *__restrict__ out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_cfg) return;
    Rt34 cur;
#pragma unroll
    for (int e = 0; e < 12; ++e) cur.m[e] = (e % 5 == 0) ? 1.f : 0.f;
    int next_link = 0;
    for (int f = 0; f < plan.n_frames; ++f) {
        const pvb_fk_frame &fr = plan.frame[f];
        cur = rt_mul(cur, fr.origin);
        if (fr.joint_type != PVB_FK_FIXED) {
            const float th = __ldg(q + (size_t)a * n_joints + fr.q_index);
            float mot[12];
            const float x = fr.axis[0], y = fr.axis[1], z = fr.axis[2];
            if (fr.joint_type == PVB_FK_REVOLUTE) {
                const float c = cosf(th), s = sinf(th), t = 1.f - c;
                mot[0] = c + x * x * t;     mot[1] = x * y * t - z * s; mot[2] = x * z * t + y * s;  mot[3] = 0.f;
                mot[4] = y * x * t + z * s; mot[5] = c + y * y * t;     mot[6] = y * z * t - x * s;  mot[7] = 0.f;
                mot[8] = z * x * t - y * s; mot[9] = z * y * t + x * s; mot[10] = c + z * z * t;     mot[11] = 0.f;
            } else {
                mot[0] = 1.f; mot[1] = 0.f; mot[2] = 0.f; mot[3] = x * th;
                mot[4] = 0.f; mot[5] = 1.f; mot[6] = 0.f; mot[7] = y * th;
                mot[8] = 0.f; mot[9] = 0.f; mot[10] = 1.f; mot[11] = z * th;
            }
            cur = rt_mul(cur, mot);
        }
        // mesh links attached to this frame (sorted by frame on the host)
        while (next_link < plan.n_links && plan.link[next_link].frame == f) {
            const pvb_fk_link &lk = plan.link[next_link];
            // rigid inverse of the link pose: [R^T | -R^T t]
            float inv[12];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                inv[4 * r] = cur.m[r]; inv[4 * r + 1] = cur.m[4 + r]; inv[4 * r + 2] = cur.m[8 + r];
                inv[4 * r + 3] = -(cur.m[r] * cur.m[3] + cur.m[4 + r] * cur.m[7] + cur.m[8 + r] * cur.m[11]);
            }
            Rt34 off;
#pragma unroll
            for (int e = 0; e < 12; ++e) off.m[e] = lk.mesh_from_link[e];
            const Rt34 m = rt_mul(off, inv);
            float4 *dst = reinterpret_cast<float4 *>(out + ((size_t)lk.slot * n_cfg + a) * 16);
            dst[0] = make_float4(m.m[0], m.m[1], m.m[2], m.m[3]);
            dst[1] = make_float4(m.m[4], m.m[5], m.m[6], m.m[7]);
            dst[2] = make_float4(m.m[8], m.m[9], m.m[10], m.m[11]);
            dst[3] = make_float4(0.f, 0.f, 0.f, 1.f);
            ++next_link;
        }
    }
}

// =================================================================== chamfer
// grid = (tiles, n_tf).  Each block: transform its points with W_b, unsigned
// distance (no sign pass: the value is squared, chamfer.py:92), block-reduce
// (scale*d)^2 into one partial; a second tiny kernel sums the partials in a
// fixed order (deterministic) and divides by N.
constexpr int kChamThreads = 256;

__global__ void __launch_bounds__(kChamThreads)
chamfer_partial_kernel(const pvb_sdf_desc obj, const float *__restrict__ w2o, const float *__restrict__ pts,
                       long long n_pts, const float4 *__restrict__ sorted, float scale, int n_stage_max,
                       float *__restrict__ partial) {
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
            d = sphere_eval(obj.radius, q).val;
        }
        const float sd = scale * d;
        acc = fmaf(sd, sd, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kChamThreads / 32; ++w) s += s_red[w];
        partial[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
    }
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
__global__ void transform_points_kernel(const float *__restrict__ xforms, int n_tf, const float *__restrict__ pts,
                                        long long n_pts, float *__restrict__ out) {
    const int b = blockIdx.y;
    const float *xf = xforms + (size_t)b * 16;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pts; i += stride) {
        const f3 p = load_point(pts, i);
        float *o = out + ((size_t)b * n_pts + i) * 3;
        o[0] = fmaf(xf[0], p.x, fmaf(xf[1], p.y, fmaf(xf[2], p.z, xf[3])));
        o[1] = fmaf(xf[4], p.x, fmaf(xf[5], p.y, fmaf(xf[6], p.z, xf[7])));
        o[2] = fmaf(xf[8], p.x, fmaf(xf[9], p.y, fmaf(xf[10], p.z, xf[11])));
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

template <bool kMesh, int PTS, int MAXS>
static int launch_composed(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                           int cfg_count, const float *pts, long long first_pt, long long n_pts, uint32_t mesh_mode,
                           float *out_val, float *out_grad, int *out_which, const OutTargets *tg, cudaStream_t stream) {
    const long long n_items = (n_pts - first_pt) / PTS;
    if (n_items <= 0) return PVB_OK;
    DescPack<MAXS> pack;
    memcpy(pack.d, descs, sizeof(pvb_sdf_desc) * (size_t)n_sdf);
    fill_order(pack, n_sdf);
    const int gx = grid_for(n_items, kCompThreads, 8);
    int gy = cfg_count < 65535 ? cfg_count : 65535;
    const long long cap = (long long)sm_count() * 64;     // bound the block count for huge configuration batches
    if ((long long)gx * gy > cap) { gy = (int)(cap / gx); if (gy < 1) gy = 1; }
    dim3 grid((unsigned)gx, (unsigned)gy);
    // mesh sub-SDFs: nearest-bound-first evaluation (PVB_COMP_NEAREST_FIRST=0 restores the fixed bit-reversed order)
    static const int nearest_first = [] { const char *e = getenv("PVB_COMP_NEAREST_FIRST"); return e ? atoi(e) : 1; }();
    float margin_max = 0.f;
    for (int i = 0; i < n_sdf; ++i) margin_max = descs[i].prune_margin > margin_max ? descs[i].prune_margin : margin_max;
    timing_mark(0, stream);
    if (tg)
        composed_query_kernel<kMesh, PTS, MAXS, true><<<grid, kCompThreads, 0, stream>>>(
            pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, first_pt, n_pts, mesh_mode, nullptr, nullptr,
            out_which, *tg, nearest_first, margin_max);
    else
        composed_query_kernel<kMesh, PTS, MAXS, false><<<grid, kCompThreads, 0, stream>>>(
            pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, first_pt, n_pts, mesh_mode, out_val, out_grad,
            out_which, OutTargets{}, nearest_first, margin_max);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query");
    return PVB_OK;
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
    auto k0 = robot_query_kernel<MAXS, kUnroll, 0>;
    auto k1 = robot_query_kernel<MAXS, kUnroll, 1>;
    auto k2 = robot_query_kernel<MAXS, kUnroll, 2>;
    const int smem = (int)sizeof(RobotSmem<MAXS>);
    const int slot0 = kUnroll ? kSlotRobot : kSlotRobotWide;
    if (!ensure_smem(k0, slot0, smem) || !ensure_smem(k1, slot0 + 1, smem) || !ensure_smem(k2, slot0 + 2, smem)) {
        pvb_set_error("pvb_composed_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
        return PVB_ERR_CUDA;
    }
    const int gy = (cfg_count + kRbCfg - 1) / kRbCfg;
    const long long n_tiles = (n_pts + kRbTilePts - 1) / kRbTilePts;
    static const int waves = [] { const char *e = getenv("PVB_ROBOT_WAVES"); return e ? atoi(e) : 4; }();
    long long gx = ((long long)sm_count() * (kUnroll ? 4 : 3) * waves + gy - 1) / gy;
    if (gx > n_tiles) gx = n_tiles;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, (unsigned)gy);
    const OutTargets none{};
    timing_mark(0, stream);
    if (kind == 0)
        k0<<<grid, kRbCfg * kRbWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, out_val, out_grad, out_which, none);
    else if (kind == 1)
        k1<<<grid, kRbCfg * kRbWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, nullptr, nullptr, out_which, *tg);
    else
        k2<<<grid, kRbCfg * kRbWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, nullptr, nullptr, out_which, *tg);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query(robot)");
    return PVB_OK;
}

// Launch robot_serial_kernel (<= 8 GRID sub-SDFs with the bounding-box rule).
static int launch_robot_serial(const pvb_sdf_desc *descs, int n_sdf, const float *xforms, int n_cfg, int cfg_begin,
                               int cfg_count, const float *pts, long long n_pts, int vec, float *out_val,
                               float *out_grad, int *out_which, const OutTargets *tg, cudaStream_t stream) {
    RobotPack<kRsMaxS> pack;
    memset(&pack, 0, sizeof(pack));
    for (int si = 0; si < n_sdf; ++si) { pack.d[si] = descs[si]; pack.orig[si] = si; }
    const int kind = !tg ? 0 : (tg->mc ? 2 : 1);
    auto k0 = robot_serial_kernel<0>;
    auto k1 = robot_serial_kernel<1>;
    auto k2 = robot_serial_kernel<2>;
    const int smem = (int)sizeof(RsSmem);
    if (!ensure_smem(k0, kSlotSerial, smem) || !ensure_smem(k1, kSlotSerial + 1, smem) ||
        !ensure_smem(k2, kSlotSerial + 2, smem)) {
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
    static const int waves = [] { const char *e = getenv("PVB_ROBOT_WAVES"); return e ? atoi(e) : 4; }();
    long long gx = ((long long)sm_count() * PVB_RS_MINB * waves + gy - 1) / gy;
    const long long gx_max = (n_chunks + kRsWarps - 1) / kRsWarps;
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    const long long spw = chunk_log2;
    dim3 grid((unsigned)gx, (unsigned)gy);
    const OutTargets none{};
    timing_mark(0, stream);
    if (kind == 0)
        k0<<<grid, kRbCfg * kRsWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, (int)spw, out_val, out_grad, out_which, none);
    else if (kind == 1)
        k1<<<grid, kRbCfg * kRsWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, (int)spw, nullptr, nullptr, out_which, *tg);
    else
        k2<<<grid, kRbCfg * kRsWarps, smem, stream>>>(pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, (int)n_pts,
                                                      vec, (int)spw, nullptr, nullptr, out_which, *tg);
    timing_mark(1, stream);
    PVB_CHECK_LAUNCH("pvb_composed_query(robot-serial)");
    return PVB_OK;
}

// tg == nullptr: one destination (out_val / out_grad); otherwise the kMulti instantiations store to every target
static int composed_dispatch(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                             int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_pts,
                             uint32_t mesh_mode, float *out_val, float *out_grad, int32_t *out_which,
                             const OutTargets *tg, void *stream) {
    if (!descs || !xforms || n_sdf < 1 || n_cfg < 1 || cfg_begin < 0 || cfg_count < 0 ||
        cfg_begin + cfg_count > n_cfg || n_pts < 0 || (n_pts > 0 && cfg_count > 0 && (!pts || !out_val || !out_grad))) {
        pvb_set_error("pvb_composed_query: invalid argument (n_sdf=%d n_cfg=%d cfg=[%d,+%d) n_pts=%lld)", n_sdf, n_cfg,
                      cfg_begin, cfg_count, (long long)n_pts);
        return PVB_ERR_INVALID;
    }
    if (n_sdf > 128) {
        pvb_set_error("pvb_composed_query: at most 128 sub-SDFs per call (got %d)", n_sdf);
        return PVB_ERR_INVALID;
    }
    if (n_pts == 0 || cfg_count == 0) return PVB_OK;
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
    if (tg && tg->mc) {
        // multicast destinations exist only in robot_query_kernel: refuse anything that would fall through
        bool grids = !needs_mesh && n_sdf <= 16;
        for (int i = 0; i < n_sdf && grids; ++i)
            grids = descs[i].kind == PVB_KIND_GRID && !(descs[i].flags & (PVB_GRID_OOB_GT | PVB_GRID_TRILINEAR));
        if (!grids || n_pts >= (1ll << 31)) {
            pvb_set_error("pvb_composed_query_multicast: needs <= 16 GRID sub-SDFs with the bounding-box rule");
            return PVB_ERR_INVALID;
        }
    }
    const bool vec = !needs_mesh && aligned16(pts) && out_aligned && aligned16(out_which) && (n_pts % 4 == 0);
    const long long n_vec = vec ? n_pts : 0;
    int rc = PVB_OK;
    static const int cfg_major = [] { const char *e = getenv("PVB_COMP_CFGMAJOR"); return e ? atoi(e) : 1; }();
    // lanes = configurations: only worthwhile when the 32-wide configuration tiles are well filled (25 configurations
    // per rank on 8 GPUs would idle 22 % of the lanes, and point-major is faster there)
    const int cm_tiles = (cfg_count + kCmCfg - 1) / kCmCfg;
    // ... except with several destinations: the configuration-major epilogue owns whole rows and stores them as full
    // sectors, which is what the NVLink-bound re-assembly needs; idle lanes cost less than partial-sector packets
    const bool cm_filled = (cfg_count >= 16 && (double)cfg_count >= 0.85 * (double)(cm_tiles * kCmCfg)) ||
                           (tg && tg->vec && cfg_count >= 8);
    static const int robot_kernel = [] { const char *e = getenv("PVB_ROBOT_KERNEL"); return e ? atoi(e) : 2; }();
    static const double robot_fill = [] { const char *e = getenv("PVB_ROBOT_MIN_FILL"); return e ? atof(e) : 0.85; }();
    bool all_grid = !needs_mesh && n_sdf <= 16 && n_pts < (1ll << 31);
    for (int i = 0; i < n_sdf && all_grid; ++i)
        all_grid = descs[i].kind == PVB_KIND_GRID && !(descs[i].flags & (PVB_GRID_OOB_GT | PVB_GRID_TRILINEAR));
    const bool rb_filled = (cfg_count >= 16 && (double)cfg_count >= robot_fill * (double)(cm_tiles * kCmCfg)) ||
                           (tg && tg->vec && cfg_count >= 8) || (tg && tg->mc);
    // the point-serial kernel has no fill problem (remainder configurations run in lane-split tiles): any batch of
    // PVB_ROBOT_MIN_CFG or more configurations takes it
    static const int serial_min_cfg = [] { const char *e = getenv("PVB_ROBOT_MIN_CFG"); return e ? atoi(e) : 8; }();
    const bool serial_ok = robot_kernel >= 2 && n_sdf <= kRsMaxS && cfg_count >= serial_min_cfg &&
                           cfg_count <= 65535 * kRbCfg;          // one grid row per 32-configuration tile
    if (robot_kernel && cfg_major && all_grid && (rb_filled || serial_ok)) {
        const int vec_rows = (tg ? tg->vec : (out_aligned && (n_pts % 4 == 0))) && aligned16(pts);
        // PVB_ROBOT_KERNEL: 2 (default) = point-serial nearest-sphere-first kernel for <= 8 links, 1 = the
        // 4-points-per-thread kernel, 0 = round 1's configuration-major kernel
        if (serial_ok)
            return launch_robot_serial(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                       (tg ? tg->vec : (out_aligned && (n_pts % 4 == 0))), out_val, out_grad, out_which,
                                       tg, s);
        return n_sdf <= 8 ? launch_robot<8, true>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, vec_rows,
                                                  out_val, out_grad, out_which, tg, s)
                          : launch_robot<16, false>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts,
                                                    vec_rows, out_val, out_grad, out_which, tg, s);
    }
    if (cfg_major && !needs_mesh && n_sdf <= kCmMaxS && cm_filled) {
        if (!ensure_smem(composed_cfgmajor_kernel<false>, kSlotCfgMajor, (int)sizeof(CmSmem)) ||
            !ensure_smem(composed_cfgmajor_kernel<true>, kSlotCfgMajorMulti, (int)sizeof(CmSmem))) {
            pvb_set_error("pvb_composed_query: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
            return PVB_ERR_CUDA;
        }
        DescPack<kCmMaxS> pack;
        memcpy(pack.d, descs, sizeof(pvb_sdf_desc) * (size_t)n_sdf);
        fill_order(pack, n_sdf);
        const int gy = (cfg_count + kCmCfg - 1) / kCmCfg;
        const long long n_tiles = (n_pts + kCmTilePts - 1) / kCmTilePts;
        long long gx = ((long long)sm_count() * 3 * 4 + gy - 1) / gy;     // ~4 waves of resident CTAs
        if (gx > n_tiles) gx = n_tiles;
        if (gx < 1) gx = 1;
        dim3 grid((unsigned)gx, (unsigned)gy);
        timing_mark(0, s);
        if (tg)
            composed_cfgmajor_kernel<true><<<grid, kCmCfg * kCmWarps, sizeof(CmSmem), s>>>(
                pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, nullptr, nullptr, out_which, *tg);
        else
            composed_cfgmajor_kernel<false><<<grid, kCmCfg * kCmWarps, sizeof(CmSmem), s>>>(
                pack, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, out_val, out_grad, out_which,
                OutTargets{});
        timing_mark(1, s);
        PVB_CHECK_LAUNCH("pvb_composed_query(cfg-major)");
        return PVB_OK;
    }
#define PVB_COMP(MESH, PTS, FIRST, N)                                                                              \
    (n_sdf <= 16 ? launch_composed<MESH, PTS, 16>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, FIRST, N,  \
                                                  mesh_mode, out_val, out_grad, out_which, tg, s)                  \
                 : launch_composed<MESH, PTS, 128>(descs, n_sdf, xforms, n_cfg, cfg_begin, cfg_count, pts, FIRST, N, \
                                                   mesh_mode, out_val, out_grad, out_which, tg, s))
    if (n_vec > 0) {
        rc = PVB_COMP(false, PVB_COMP_PTS, 0, n_pts);
    } else if (needs_mesh) {
        rc = PVB_COMP(true, 1, 0, n_pts);
    } else {
        rc = PVB_COMP(false, 1, 0, n_pts);
    }
#undef PVB_COMP
    return rc;
}

extern "C" int pvb_composed_query(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                                  int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                  const float *pts, int64_t n_pts, uint32_t mesh_mode, float *out_val, float *out_grad,
                                  int32_t *out_which, void *stream) {
    return composed_dispatch(descs, n_sdf, needs_mesh, xforms, n_cfg, cfg_begin, cfg_count, pts, n_pts, mesh_mode,
                             out_val, out_grad, out_which, nullptr, stream);
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
    FkPlan plan;
    memset(&plan, 0, sizeof(plan));
    plan.n_frames = n_frames;
    plan.n_links = n_links;
    memcpy(plan.frame, frames, sizeof(pvb_fk_frame) * (size_t)n_frames);
    memcpy(plan.link, links, sizeof(pvb_fk_link) * (size_t)n_links);
    int prev = -1;
    for (int s = 0; s < n_links; ++s) {
        const pvb_fk_link &lk = plan.link[s];
        if (lk.frame < prev || lk.frame < 0 || lk.frame >= n_frames || lk.slot < 0 || lk.slot >= n_links) {
            pvb_set_error("pvb_fk_serial: links must be sorted by frame, with frame in [0, n_frames) and slot in [0, n_links)");
            return PVB_ERR_INVALID;
        }
        prev = lk.frame;
    }
    for (int f = 0; f < n_frames; ++f) {
        const pvb_fk_frame &fr = plan.frame[f];
        if (fr.joint_type != PVB_FK_FIXED && (fr.q_index < 0 || fr.q_index >= n_joints)) {
            pvb_set_error("pvb_fk_serial: frame %d reads joint value %d of %d", f, fr.q_index, n_joints);
            return PVB_ERR_INVALID;
        }
    }
    if (n_cfg == 0) return PVB_OK;
    fk_serial_kernel<<<(n_cfg + 63) / 64, 64, 0, (cudaStream_t)stream>>>(plan, q, n_cfg, n_joints, out_xforms);
    PVB_CHECK_LAUNCH("pvb_fk_serial");
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
    if (obj->kind == PVB_KIND_MESH)
        if (int rc = check_mesh(obj, "pvb_chamfer")) return rc;
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
    dim3 grid((unsigned)n_blk, (unsigned)n_tf);
    timing_mark(0, (cudaStream_t)stream);
    chamfer_partial_kernel<<<grid, kChamThreads, (size_t)n_stage * 128, (cudaStream_t)stream>>>(
        *obj, world_to_object, pts, n_pts, sq.sorted, scale, n_stage, workspace);
    timing_mark(1, (cudaStream_t)stream);
    PVB_CHECK_LAUNCH("pvb_chamfer(partial)");
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

extern "C" int pvb_transform_points(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts, float *out,
                                    void *stream) {
    if (!xforms || n_tf < 0 || n_pts < 0 || (n_tf > 0 && n_pts > 0 && (!pts || !out)) || n_tf > 65535) {
        pvb_set_error("pvb_transform_points: invalid argument");
        return PVB_ERR_INVALID;
    }
    if (n_tf == 0 || n_pts == 0) return PVB_OK;
    dim3 grid((unsigned)grid_for(n_pts, 256, 8), (unsigned)n_tf);
    transform_points_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(xforms, n_tf, pts, n_pts, out);
    PVB_CHECK_LAUNCH("pvb_transform_points");
    return PVB_OK;
}
