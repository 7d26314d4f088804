// pvb_device.cuh -- device-side building blocks shared by the sm_90a kernels.
//
//   grid_eval      CachedSDF.__call__ for one point          (reference sdf.py:535-571)
//   bvh_closest    closest point on the mesh                 (Embree rtcPointQuery role, sdf.py:134)
//   bvh_parity     ray/triangle crossing parity              (count_intersections role, sdf.py:152-154)
//   mesh_eval      ObjectFactory._do_object_frame_closest_point epilogue (sdf.py:139-164)
//   composed_point ComposedSDF.__call__ for one (configuration, point) pair (sdf.py:392-433)
#pragma once
#include "../../include/pvb.h"
#include <cuda_runtime.h>
#include <stdint.h>

namespace pvb {

constexpr int kStack = 64;            // traversal stack entries per thread; the builder bounds the depth at 20

// Traversal statistics hook: expands to nothing in the CUDA build; the host build of this header (tests/hostsim)
// defines it to count node visits and triangle tests per query (SURVEY 8d-iii, scripts/traversal_stats.py).
#ifndef PVB_STAT
#define PVB_STAT(counter)
#endif
#define PVB_INF (__builtin_huge_valf())

struct f3 { float x, y, z; };
__device__ __forceinline__ f3 mk3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ f3 operator*(f3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot(f3 a, f3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ float sel(f3 v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : v.z); }

// The top of the BVH staged in shared memory (first `n` nodes of the BFS layout).
struct NodeStage {
    const float4 *smem;   // 8 float4 per node
    int n;
};

__device__ __forceinline__ const float4 *node_ptr(const float4 *gnodes, const NodeStage &st, int idx) {
    return idx < st.n ? st.smem + 8 * idx : gnodes + 8 * (size_t)idx;
}

// ----------------------------------------------------------------------------
// Closest point on triangle (Ericson, RTCD 5.1.5), fp32.
// (Round 2 tried deriving d3..d6 from d1, d2 and the Gram terms ab.ab, ab.ac, ac.ac -- 4 subtractions instead of 6
// subtractions + 12 multiply-adds in the tree walk's hottest function.  Rejected on the CPU tier before it
// reached a GPU: on sliver triangles the cancellation costs accuracy, tests/test_hostsim.py's degenerate-soup fuzz read
// 2.2e-6 relative distance error against the 2e-6 bound the direct dot products meet.)
__device__ __forceinline__ f3 closest_on_triangle(f3 p, f3 a, f3 b, f3 c) {
    const f3 ab = b - a, ac = c - a, ap = p - a;
    const float d1 = dot(ab, ap), d2 = dot(ac, ap);
    if (d1 <= 0.f && d2 <= 0.f) return a;
    const f3 bp = p - b;
    const float d3 = dot(ab, bp), d4 = dot(ac, bp);
    if (d3 >= 0.f && d4 <= d3) return b;
    const float vc = d1 * d4 - d3 * d2;
    if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
        const float v = __fdiv_rn(d1, d1 - d3);
        return a + ab * v;
    }
    const f3 cp = p - c;
    const float d5 = dot(ab, cp), d6 = dot(ac, cp);
    if (d6 >= 0.f && d5 <= d6) return c;
    const float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
        const float w = __fdiv_rn(d2, d2 - d6);
        return a + ac * w;
    }
    const float va = d3 * d6 - d5 * d4;
    if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) {
        const float w = __fdiv_rn(d4 - d3, (d4 - d3) + (d5 - d6));
        return b + (c - b) * w;
    }
    const float denom = __fdiv_rn(1.f, va + vb + vc);
    const float v = vb * denom, w = vc * denom;
    return a + ab * v + ac * w;
}

struct Closest {
    f3 q;        // closest point
    float d2;    // squared distance
    int face;    // original face index, -1 if nothing within the initial radius
};

__device__ __forceinline__ float box_d2(float lx, float ly, float lz, float hx, float hy, float hz, f3 p) {
    const float dx = fmaxf(fmaxf(lx - p.x, p.x - hx), 0.f);
    const float dy = fmaxf(fmaxf(ly - p.y, p.y - hy), 0.f);
    const float dz = fmaxf(fmaxf(lz - p.z, p.z - hz), 0.f);
    return fmaf(dx, dx, fmaf(dy, dy, dz * dz));
}

// Nearest-first BVH4 descent.  `init_d2` is an initial search radius (squared);
// candidates farther than that are never reported (face stays -1).
// (Rejected alternatives: leaves as stack entries popped in distance order -- the extra local-memory stack traffic
// costs more than the better lane occupancy of the triangle code buys; runs of consecutive queries seeded with the
// previous closest point; a phase-aligned "while-while" walk (Aila & Laine: advance to a leaf first, then test
// triangles together) -- no gain, the cost is in the triangle tests themselves.)
__device__ __forceinline__ Closest bvh_closest(const float4 *__restrict__ gnodes, const NodeStage &st,
                                               const float4 *__restrict__ tris, f3 p, float init_d2) {
    Closest best;
    best.q = mk3(0.f, 0.f, 0.f);
    best.d2 = init_d2;
    best.face = -1;
    int stack_n[kStack];
    float stack_d[kStack];
    int sp = 0;
    stack_n[sp] = 0; stack_d[sp] = 0.f; ++sp;
    // box distances are lower bounds only up to fp32 rounding of either side; keep a margin
    constexpr float kSlack = 0.99999f;
    while (sp > 0) {
        --sp;
        const int ni = stack_n[sp];
        if (stack_d[sp] * kSlack > best.d2) continue;
        PVB_STAT(closest_nodes)
        const float4 *n = node_ptr(gnodes, st, ni);
        const float4 lox = n[0], loy = n[1], loz = n[2], hix = n[3], hiy = n[4], hiz = n[5];
        const int4 ch = *reinterpret_cast<const int4 *>(n + 6);
        float d[4];
        int c[4];
        d[0] = box_d2(lox.x, loy.x, loz.x, hix.x, hiy.x, hiz.x, p); c[0] = ch.x;
        d[1] = box_d2(lox.y, loy.y, loz.y, hix.y, hiy.y, hiz.y, p); c[1] = ch.y;
        d[2] = box_d2(lox.z, loy.z, loz.z, hix.z, hiy.z, hiz.z, p); c[2] = ch.z;
        d[3] = box_d2(lox.w, loy.w, loz.w, hix.w, hiy.w, hiz.w, p); c[3] = ch.w;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (c[k] == INT32_MIN) d[k] = PVB_INF;
        // sort the four children by distance (5-comparator network), nearest first
#define PVB_CSWAP(i, j)                                                          \
    if (d[j] < d[i]) { const float td = d[i]; d[i] = d[j]; d[j] = td;            \
                       const int tc = c[i]; c[i] = c[j]; c[j] = tc; }
        PVB_CSWAP(0, 1) PVB_CSWAP(2, 3) PVB_CSWAP(0, 2) PVB_CSWAP(1, 3) PVB_CSWAP(1, 2)
#undef PVB_CSWAP
        // leaves first (nearest first) so that the bound tightens before pushing
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (c[k] < 0 && c[k] != INT32_MIN && d[k] * kSlack <= best.d2) {
                const unsigned code = (unsigned)~c[k];
                const int first = (int)(code >> 2), cnt = (int)(code & 3u) + 1;
                for (int t = first; t < first + cnt; ++t) {
                    PVB_STAT(closest_tris)
                    const float4 v0 = __ldg(tris + 3 * (size_t)t);
                    const float4 v1 = __ldg(tris + 3 * (size_t)t + 1);
                    const float4 v2 = __ldg(tris + 3 * (size_t)t + 2);
                    const f3 q = closest_on_triangle(p, mk3(v0.x, v0.y, v0.z), mk3(v1.x, v1.y, v1.z),
                                                     mk3(v2.x, v2.y, v2.z));
                    const f3 g = q - p;
                    const float dd = dot(g, g);
                    const int face = __float_as_int(v0.w);
                    // ties -> lowest original face index (the oracle's brute-force rule)
                    if (dd < best.d2 || (dd == best.d2 && (best.face < 0 || face < best.face))) {
                        best.d2 = dd; best.q = q; best.face = face;
                    }
                }
            }
        }
        // inner children, farthest pushed first
#pragma unroll
        for (int k = 3; k >= 0; --k) {
            if (c[k] >= 0 && d[k] * kSlack <= best.d2 && sp < kStack) {
                stack_n[sp] = c[k]; stack_d[sp] = d[k]; ++sp;
            }
        }
    }
    return best;
}

// ----------------------------------------------------------------------------
// Crossing parity of the ray o + t*dir, t in [0, inf), with the triangle soup.
// Watertight ray/triangle test (Woop, Benthin, Wald 2013): shared edges and
// vertices are counted consistently, so the parity of a closed mesh is exact.
__device__ __forceinline__ int bvh_parity(const float4 *__restrict__ gnodes, const NodeStage &st,
                                          const float4 *__restrict__ tris, f3 o, f3 dir) {
    // shear setup
    const float ax = fabsf(dir.x), ay = fabsf(dir.y), az = fabsf(dir.z);
    int kz = (ax > ay) ? (ax > az ? 0 : 2) : (ay > az ? 1 : 2);
    int kx = kz + 1; if (kx == 3) kx = 0;
    int ky = kx + 1; if (ky == 3) ky = 0;
    if (sel(dir, kz) < 0.f) { const int t = kx; kx = ky; ky = t; }
    const float dz = sel(dir, kz);
    const float Sx = __fdiv_rn(sel(dir, kx), dz), Sy = __fdiv_rn(sel(dir, ky), dz), Sz = __fdiv_rn(1.f, dz);
    // slab setup (guard exact zeros; the box test only has to be conservative)
    const float tiny = 1e-30f;
    const f3 inv = mk3(__fdiv_rn(1.f, fabsf(dir.x) < tiny ? copysignf(tiny, dir.x) : dir.x),
                       __fdiv_rn(1.f, fabsf(dir.y) < tiny ? copysignf(tiny, dir.y) : dir.y),
                       __fdiv_rn(1.f, fabsf(dir.z) < tiny ? copysignf(tiny, dir.z) : dir.z));
    int hits = 0;
    int stack_n[kStack];
    int sp = 0;
    stack_n[sp++] = 0;
    while (sp > 0) {
        const int ni = stack_n[--sp];
        PVB_STAT(parity_nodes)
        const float4 *n = node_ptr(gnodes, st, ni);
        const float4 lox = n[0], loy = n[1], loz = n[2], hix = n[3], hiy = n[4], hiz = n[5];
        const int4 ch = *reinterpret_cast<const int4 *>(n + 6);
        const float lx[4] = {lox.x, lox.y, lox.z, lox.w}, ly[4] = {loy.x, loy.y, loy.z, loy.w},
                    lz[4] = {loz.x, loz.y, loz.z, loz.w};
        const float hx[4] = {hix.x, hix.y, hix.z, hix.w}, hy[4] = {hiy.x, hiy.y, hiy.z, hiy.w},
                    hz[4] = {hiz.x, hiz.y, hiz.z, hiz.w};
        const int c[4] = {ch.x, ch.y, ch.z, ch.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (c[k] == INT32_MIN) continue;
            const float t0x = (lx[k] - o.x) * inv.x, t1x = (hx[k] - o.x) * inv.x;
            const float t0y = (ly[k] - o.y) * inv.y, t1y = (hy[k] - o.y) * inv.y;
            const float t0z = (lz[k] - o.z) * inv.z, t1z = (hz[k] - o.z) * inv.z;
            float tmin = fmaxf(fmaxf(fminf(t0x, t1x), fminf(t0y, t1y)), fminf(t0z, t1z));
            float tmax = fminf(fminf(fmaxf(t0x, t1x), fmaxf(t0y, t1y)), fmaxf(t0z, t1z));
            // conservative padding of the interval (Ize 2013)
            tmin = tmin - fabsf(tmin) * 4e-7f;
            tmax = tmax + fabsf(tmax) * 4e-7f;
            if (!(fmaxf(tmin, 0.f) <= tmax)) continue;
            if (c[k] >= 0) {
                if (sp < kStack) stack_n[sp++] = c[k];
                continue;
            }
            const unsigned code = (unsigned)~c[k];
            const int first = (int)(code >> 2), cnt = (int)(code & 3u) + 1;
            for (int t = first; t < first + cnt; ++t) {
                PVB_STAT(parity_tris)
                const float4 v0 = __ldg(tris + 3 * (size_t)t);
                const float4 v1 = __ldg(tris + 3 * (size_t)t + 1);
                const float4 v2 = __ldg(tris + 3 * (size_t)t + 2);
                const f3 A = mk3(v0.x, v0.y, v0.z) - o, B = mk3(v1.x, v1.y, v1.z) - o,
                         C = mk3(v2.x, v2.y, v2.z) - o;
                const float Akz = sel(A, kz), Bkz = sel(B, kz), Ckz = sel(C, kz);
                // sheared coordinates: a function of the vertex alone, so shared
                // vertices get bit-identical values in every triangle
                const float Ax = fmaf(-Sx, Akz, sel(A, kx)), Ay = fmaf(-Sy, Akz, sel(A, ky));
                const float Bx = fmaf(-Sx, Bkz, sel(B, kx)), By = fmaf(-Sy, Bkz, sel(B, ky));
                const float Cx = fmaf(-Sx, Ckz, sel(C, kx)), Cy = fmaf(-Sy, Ckz, sel(C, ky));
                // edge functions without contraction: exact antisymmetry across a shared edge
                float U = __fsub_rn(__fmul_rn(Cx, By), __fmul_rn(Cy, Bx));
                float V = __fsub_rn(__fmul_rn(Ax, Cy), __fmul_rn(Ay, Cx));
                float W = __fsub_rn(__fmul_rn(Bx, Ay), __fmul_rn(By, Ax));
                if (U == 0.f || V == 0.f || W == 0.f) {
                    U = (float)((double)Cx * (double)By - (double)Cy * (double)Bx);
                    V = (float)((double)Ax * (double)Cy - (double)Ay * (double)Cx);
                    W = (float)((double)Bx * (double)Ay - (double)By * (double)Ax);
                }
                if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) continue;
                const float det = U + V + W;
                if (det == 0.f) continue;
                const float Az = Sz * Akz, Bz = Sz * Bkz, Cz = Sz * Ckz;
                const float T = fmaf(U, Az, fmaf(V, Bz, W * Cz));
                // t = T / det >= 0
                if ((det > 0.f) ? (T >= 0.f) : (T <= 0.f)) ++hits;
            }
        }
    }
    return hits & 1;
}

// ----------------------------------------------------------------------------
// Crossing parity along +x for CLOSED meshes (every directed edge matched by its reverse, checked on the host).
// The parity of a closed surface does not depend on the ray direction, so the reference's diagonal ray
// (sdf.py:147-153) can be replaced by the axis through the query point: the box test becomes an exact 2-D
// containment (no slabs, no divisions), the triangle test loses the shear, and far fewer nodes are visited.
// Exactness: same translated-vertex edge functions as above (shared edges antisymmetric by construction); an edge
// function that is exactly zero is resolved by symbolic perturbation of the origin by (eps, eps^2) in (y, z) --
// sign of dU/dy, then dU/dz, both exact coordinate comparisons -- so that a ray through an edge or a vertex is
// counted by exactly one of the adjacent triangles and tangential contacts cancel.
__device__ __forceinline__ float edge_sign_x(float By, float Bz, float Cy, float Cz, float vBy, float vBz, float vCy,
                                             float vCz) {
    // U = Cy' * Bz' - Cz' * By' with primes = translated by the origin; exact sign
    float U = __fsub_rn(__fmul_rn(Cy, Bz), __fmul_rn(Cz, By));
    if (U == 0.f) {
        const double Ud = (double)Cy * (double)Bz - (double)Cz * (double)By;
        if (Ud != 0.0) U = Ud > 0.0 ? 1.f : -1.f;
        else {
            // dU/dPy = Cz - Bz, dU/dPz = By - Cy (untranslated vertex coordinates: exact comparisons)
            if (vCz != vBz) U = vCz > vBz ? 1.f : -1.f;
            else U = vBy > vCy ? 1.f : (vBy < vCy ? -1.f : 0.f);
        }
    }
    return U;
}

__device__ __forceinline__ int bvh_parity_x(const float4 *__restrict__ gnodes, const NodeStage &st,
                                            const float4 *__restrict__ tris, f3 o) {
    int hits = 0;
    int stack_n[kStack];
    int sp = 0;
    stack_n[sp++] = 0;
    while (sp > 0) {
        const int ni = stack_n[--sp];
        PVB_STAT(parity_nodes)
        const float4 *n = node_ptr(gnodes, st, ni);
        const float4 loy = n[1], loz = n[2], hix = n[3], hiy = n[4], hiz = n[5];
        const int4 ch = *reinterpret_cast<const int4 *>(n + 6);
        const float ly[4] = {loy.x, loy.y, loy.z, loy.w}, lz[4] = {loz.x, loz.y, loz.z, loz.w};
        const float hx[4] = {hix.x, hix.y, hix.z, hix.w}, hy[4] = {hiy.x, hiy.y, hiy.z, hiy.w},
                    hz[4] = {hiz.x, hiz.y, hiz.z, hiz.w};
        const int c[4] = {ch.x, ch.y, ch.z, ch.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            // exact: a triangle crossed at t >= 0 has the crossing point inside its box
            const bool in = (c[k] != INT32_MIN) & (o.y >= ly[k]) & (o.y <= hy[k]) & (o.z >= lz[k]) & (o.z <= hz[k]) &
                            (hx[k] >= o.x);
            if (!in) continue;
            if (c[k] >= 0) {
                if (sp < kStack) stack_n[sp++] = c[k];
                continue;
            }
            const unsigned code = (unsigned)~c[k];
            const int first = (int)(code >> 2), cnt = (int)(code & 3u) + 1;
            for (int t = first; t < first + cnt; ++t) {
                PVB_STAT(parity_tris)
                const float4 v0 = __ldg(tris + 3 * (size_t)t);
                const float4 v1 = __ldg(tris + 3 * (size_t)t + 1);
                const float4 v2 = __ldg(tris + 3 * (size_t)t + 2);
                const float Ay = v0.y - o.y, Az = v0.z - o.z, By = v1.y - o.y, Bz = v1.z - o.z, Cy = v2.y - o.y,
                            Cz = v2.z - o.z;
                const float U = edge_sign_x(By, Bz, Cy, Cz, v1.y, v1.z, v2.y, v2.z);
                const float V = edge_sign_x(Cy, Cz, Ay, Az, v2.y, v2.z, v0.y, v0.z);
                const float W = edge_sign_x(Ay, Az, By, Bz, v0.y, v0.z, v1.y, v1.z);
                if ((U < 0.f || V < 0.f || W < 0.f) && (U > 0.f || V > 0.f || W > 0.f)) continue;
                if (U == 0.f && V == 0.f && W == 0.f) continue;       // degenerate in projection (edge-on triangle)
                // x of the crossing relative to the origin, in exact-sign arithmetic where it matters
                const double Ud = (double)__fsub_rn(__fmul_rn(Cy, Bz), __fmul_rn(Cz, By));
                const double Vd = (double)__fsub_rn(__fmul_rn(Ay, Cz), __fmul_rn(Az, Cy));
                const double Wd = (double)__fsub_rn(__fmul_rn(By, Az), __fmul_rn(Bz, Ay));
                const double det = Ud + Vd + Wd;
                const double T = Ud * (double)(v0.x - o.x) + Vd * (double)(v1.x - o.x) + Wd * (double)(v2.x - o.x);
                if (det == 0.0) {
                    // barycentric weights vanished in fp32 although the signs are decided: fall back to the plane
                    // through the three translated vertices evaluated in fp64
                    const double ux = (double)v1.x - v0.x, uy = (double)v1.y - v0.y, uz = (double)v1.z - v0.z;
                    const double wx = (double)v2.x - v0.x, wy = (double)v2.y - v0.y, wz = (double)v2.z - v0.z;
                    const double nx = uy * wz - uz * wy, ny = uz * wx - ux * wz, nz = ux * wy - uy * wx;
                    if (nx == 0.0) continue;
                    const double tx = (nx * ((double)v0.x - o.x) + ny * ((double)v0.y - o.y) + nz * ((double)v0.z - o.z)) / nx;
                    if (tx >= 0.0) ++hits;
                    continue;
                }
                if ((det > 0.0) ? (T >= 0.0) : (T <= 0.0)) ++hits;
            }
        }
    }
    return hits & 1;
}

// ----------------------------------------------------------------------------
// EXTENSION, opt-in (ObjectFactory.sign_mode = "winding"): generalized winding number of the triangle soup at q,
// w(q) = (1 / 4 pi) * sum of signed solid angles.  The reference decides inside/outside by crossing parity
// (sdf.py:146-157), which is what the default path reproduces; parity is meaningless on open or self-intersecting
// surfaces, the winding number degrades gracefully there.  Hierarchical evaluation (Barill, Dickson, Schmidt, Levin,
// Jacobson 2018, first-order term): a subtree whose bounding sphere (centre = area-weighted centroid p~, radius r)
// is farther than beta * r is replaced by the dipole (p~ - q) . N / |p~ - q|^3 with N the sum of its area vectors;
// near subtrees are opened, leaves use the exact Van Oosterom-Strackee solid angle.
__device__ __forceinline__ float bvh_winding(const float4 *__restrict__ gnodes, const float4 *__restrict__ wn,
                                             const NodeStage &st, const float4 *__restrict__ tris, f3 q) {
    constexpr float kBeta2 = 4.f;          // beta = 2
    float w = 0.f;
    int stack_n[kStack];
    int sp = 0;
    stack_n[sp++] = 0;
    while (sp > 0) {
        const int ni = stack_n[--sp];
        const int4 ch = *reinterpret_cast<const int4 *>(node_ptr(gnodes, st, ni) + 6);
        const int c[4] = {ch.x, ch.y, ch.z, ch.w};
        const float4 *wv = wn + 8 * (size_t)ni;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (c[k] == INT32_MIN) continue;
            const float4 pr = __ldg(wv + k), nn = __ldg(wv + 4 + k);
            const f3 dlt = mk3(pr.x - q.x, pr.y - q.y, pr.z - q.z);
            const float d2 = dot(dlt, dlt);
            if (d2 > kBeta2 * pr.w * pr.w) {                 // far: dipole
                w += dot(dlt, mk3(nn.x, nn.y, nn.z)) * rsqrtf(d2) / d2;
                continue;
            }
            if (c[k] >= 0) {
                if (sp < kStack) stack_n[sp++] = c[k];
                continue;
            }
            const unsigned code = (unsigned)~c[k];
            const int first = (int)(code >> 2), cnt = (int)(code & 3u) + 1;
            for (int t = first; t < first + cnt; ++t) {
                const float4 v0 = __ldg(tris + 3 * (size_t)t), v1 = __ldg(tris + 3 * (size_t)t + 1),
                             v2 = __ldg(tris + 3 * (size_t)t + 2);
                const f3 A = mk3(v0.x - q.x, v0.y - q.y, v0.z - q.z), B = mk3(v1.x - q.x, v1.y - q.y, v1.z - q.z),
                         C = mk3(v2.x - q.x, v2.y - q.y, v2.z - q.z);
                const float la = sqrtf(dot(A, A)), lb = sqrtf(dot(B, B)), lc = sqrtf(dot(C, C));
                const float num = A.x * (B.y * C.z - B.z * C.y) - A.y * (B.x * C.z - B.z * C.x) +
                                  A.z * (B.x * C.y - B.y * C.x);
                const float den = la * lb * lc + dot(A, B) * lc + dot(B, C) * la + dot(C, A) * lb;
                w += 2.f * atan2f(num, den);                 // solid angle of the triangle seen from q
            }
        }
    }
    return w * 0.07957747154594767f;                          // 1 / (4 pi)
}

// ----------------------------------------------------------------------------
// Deterministic stand-in for the reference's unseeded ray jitter (sdf.py:149):
// three ~N(0,1) numbers per point from an integer hash (sum of four 16-bit
// uniforms), every step exact in fp32 so that a host mirror reproduces it.
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
__device__ __forceinline__ float hash_normal(uint32_t seed, uint64_t idx, uint32_t comp) {
    const uint32_t h0 = mix32(seed ^ mix32((uint32_t)idx * 3u + comp + 0x9e3779b9u) ^ mix32((uint32_t)(idx >> 32) + 0x85ebca6bu));
    const uint32_t h1 = mix32(h0 + 0x6a09e667u);
    const float s = (float)((h0 & 0xffffu) + (h0 >> 16) + (h1 & 0xffffu) + (h1 >> 16));
    return (s - 131070.0f) * 2.6428816e-05f;   // 1 / sqrt(4 * (65536^2 - 1) / 12)
}

struct SdfOut { float val; f3 grad; };

// MeshSDF value + gradient for one point (sdf.py:139-164).
//   mode: PVB_MESH_* flags.  `idx` seeds the ray jitter.
//   init_d2: squared search radius (PVB_INF for an unconditional query); when nothing lies within it, *face_out
//   is -1 and the returned value is meaningless.  known_outside: the caller has proven the point outside the
//   surface (outside the AABB of a closed mesh), so the parity walk is skipped.
__device__ __forceinline__ SdfOut mesh_eval(const pvb_sdf_desc &m, const NodeStage &st, f3 p, uint32_t mode,
                                            uint64_t idx, f3 *closest_out, int *face_out, float init_d2 = PVB_INF,
                                            bool known_outside = false) {
    const float4 *nodes = reinterpret_cast<const float4 *>(m.nodes);
    const float4 *tris = reinterpret_cast<const float4 *>(m.tris);
    const Closest c = bvh_closest(nodes, st, tris, p, init_d2);
    if (c.face < 0) {
        if (face_out) *face_out = -1;
        SdfOut none; none.val = PVB_INF; none.grad = mk3(0.f, 0.f, 0.f);
        return none;
    }
    f3 g = c.q - p;                                            // sdf.py:139
    float dist = sqrtf(fmaf(g.x, g.x, fmaf(g.y, g.y, g.z * g.z)));   // sdf.py:141
    if (dist > 0.f) {                                          // sdf.py:143-144
        g.x = __fdiv_rn(g.x, dist); g.y = __fdiv_rn(g.y, dist); g.z = __fdiv_rn(g.z, dist);
    }
    bool inside = false;
    if ((mode & PVB_MESH_SIGNED) && !known_outside) {          // sdf.py:146-154
        const f3 dir = mk3(fmaf(1e-4f, hash_normal(m.ray_seed, idx, 0), m.ray_far[0]),
                           fmaf(1e-4f, hash_normal(m.ray_seed, idx, 1), m.ray_far[1]),
                           fmaf(1e-4f, hash_normal(m.ray_seed, idx, 2), m.ray_far[2]));
        // closed mesh: any direction gives the same parity -> exact axis-aligned walk; otherwise the reference's
        // own direction rule, because on an open surface the answer depends on it
        inside = (m.flags & PVB_MESH_CLOSED) ? bvh_parity_x(nodes, st, tris, p) != 0
                                             : bvh_parity(nodes, st, tris, p, dir) != 0;
    }
    if (inside) dist = -dist;                                  // sdf.py:155
    else { g.x = -g.x; g.y = -g.y; g.z = -g.z; }               // sdf.py:157
    if ((mode & PVB_MESH_SURFACE_NORMAL) && fabsf(dist) < 1e-3f && c.face >= 0) {   // sdf.py:162-164
        const float *fn = m.face_normals + 3 * (size_t)c.face;
        g = mk3(__ldg(fn), __ldg(fn + 1), __ldg(fn + 2));
    }
    if (closest_out) *closest_out = c.q;
    if (face_out) *face_out = c.face;
    SdfOut o; o.val = dist; o.grad = g;
    return o;
}

// ----------------------------------------------------------------------------
// CachedSDF: nearest-voxel index (TorchMultidimView.ensure_index_key semantics).
//
// The reference formula, exactly: round((p - min) / res), in fp64 when the range came from numpy (torch.tensor of
// numpy scalars is float64) and in fp32 for Python-float ranges.  Out of line: it runs for ~0.03 % of the points
// and must not cost the streaming path registers or instruction slots.
__device__ __noinline__ int grid_axis_index_exact(float pv, double min64, double res64, float min32, float res32,
                                                  bool fp32_mode, int n) {
    float kf;
    if (fp32_mode) kf = rintf(__fdiv_rn(pv - min32, res32));
    else kf = (float)rint(__ddiv_rn((double)pv - min64, res64));
    return min(max((int)kf, 0), n - 1);
}

// The evaluator is written branch-free on purpose: the first version of this kernel spent a large share of its issue
// slots on BRA/BSSY/BSYNC and saturated the XU pipe (FRND/F2I/MUFU).
//   * rint / float->int by the 1.5*2^23 magic add (FADD on the FMA pipe, no XU op); valid for |q| < 2^22, and
//     anything larger is out of range anyway
//   * the fp32 estimate q = (p - min32) * inv_res32 is accepted when |q - rint(q)| <= idx_certain (it then provably
//     rounds like the exact formula); otherwise ONE rare branch re-evaluates the three axes exactly
//   * in-range gather is a predicated load; the point-to-AABB rule (sdf.py:555-571) is evaluated for every point
//     with selects, its 1/dist by MUFU.RSQ + one Newton step (<= 1 ulp from the reference's sqrt + divide)
// Returns the ravelled key through key_out (-1 when the point fails all(min <= p <= max)).
// Point-to-AABB rule for out-of-range points (sdf.py:555-571), branch-free: delta = signed per-axis overshoot,
// dist = |delta|, r = 1/dist by MUFU.RSQ + one Newton step (<= 1 ulp from the reference's sqrt + divide).
__device__ __forceinline__ void aabb_rule(const pvb_sdf_desc &g, f3 p, float &dist, float &dx, float &dy, float &dz,
                                          float &r) {
    const float bx = g.bb_min[0] - p.x, by = g.bb_min[1] - p.y, bz = g.bb_min[2] - p.z;
    const float ax = p.x - g.bb_max[0], ay = p.y - g.bb_max[1], az = p.z - g.bb_max[2];
    const float tx = fmaxf(bx, 0.f) + fmaxf(ax, 0.f), ty = fmaxf(by, 0.f) + fmaxf(ay, 0.f),
                tz = fmaxf(bz, 0.f) + fmaxf(az, 0.f);
    dx = bx > 0.f ? -tx : tx; dy = by > 0.f ? -ty : ty; dz = bz > 0.f ? -tz : tz;
    const float d2 = dx * dx + dy * dy + dz * dz;
    r = rsqrtf(d2);                                         // MUFU.RSQ; +inf at d2 == 0
    r = r * fmaf(-0.5f * d2 * r, r, 1.5f);                  // one Newton step: 1/sqrt(d2) to ~1 ulp
    dist = d2 > 0.f ? d2 * r : 0.f;                         // the reference yields 0 and NaN gradients here (0/0)
}

// kBranchOOB: skip the AABB rule with a branch when the point is in range (composed kernels, where out-of-range
// points are rare and warps mostly agree) instead of evaluating it for every point with selects (streaming kernel,
// 42 % out of range at C2: both sides would run anyway).
template <bool kMesh, bool kBranchOOB = false>
__device__ __forceinline__ SdfOut grid_eval(const pvb_sdf_desc &g, const NodeStage &st, f3 p, uint32_t mesh_mode,
                                            uint64_t idx, long long *key_out) {
    const float kMagic = 12582912.f;   // 1.5 * 2^23
    const float qx = (p.x - g.min32[0]) * g.inv_res32[0];
    const float qy = (p.y - g.min32[1]) * g.inv_res32[1];
    const float qz = (p.z - g.min32[2]) * g.inv_res32[2];
    const float mx = __fadd_rn(qx, kMagic), my = __fadd_rn(qy, kMagic), mz = __fadd_rn(qz, kMagic);
    int kx = __float_as_int(mx) - 0x4B400000, ky = __float_as_int(my) - 0x4B400000,
        kz = __float_as_int(mz) - 0x4B400000;
    const bool certain = (fabsf(qx - __fsub_rn(mx, kMagic)) <= g.idx_certain[0]) &
                         (fabsf(qy - __fsub_rn(my, kMagic)) <= g.idx_certain[1]) &
                         (fabsf(qz - __fsub_rn(mz, kMagic)) <= g.idx_certain[2]);
    const bool inb = (p.x >= g.valid_lo[0]) & (p.x <= g.valid_hi[0]) & (p.y >= g.valid_lo[1]) &
                     (p.y <= g.valid_hi[1]) & (p.z >= g.valid_lo[2]) & (p.z <= g.valid_hi[2]);
    if (inb & !certain) {   // rare: within the uncertainty band of a cell boundary
        const bool f32 = (g.flags & PVB_GRID_INDEX_FP32) != 0;
        kx = grid_axis_index_exact(p.x, g.min64[0], g.res64[0], g.min32[0], g.res32[0], f32, g.dims[0]);
        ky = grid_axis_index_exact(p.y, g.min64[1], g.res64[1], g.min32[1], g.res32[1], f32, g.dims[1]);
        kz = grid_axis_index_exact(p.z, g.min64[2], g.res64[2], g.min32[2], g.res32[2], f32, g.dims[2]);
    }
    int key = (kx * g.dims[1] + ky) * g.dims[2] + kz;
    key = max(min(key, g.dims[0] * g.dims[1] * g.dims[2] - 1), 0);   // memory safety only (exact when inb)
    if (key_out) *key_out = inb ? (long long)key : -1ll;
    float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
    if (inb) e = __ldg(reinterpret_cast<const float4 *>(g.table) + key);
    if constexpr (kMesh) {
        if (!inb && (g.flags & PVB_GRID_OOB_GT))
            return mesh_eval(g, st, p, mesh_mode, idx, nullptr, nullptr);   // sdf.py:553-554
    }
    if constexpr (kBranchOOB) {
        if (inb) {
            SdfOut o; o.val = e.x; o.grad = mk3(e.y, e.z, e.w);
            return o;
        }
    }
    // point-to-AABB rule (sdf.py:555-571), branch-free
    float dist, dx, dy, dz, r;
    aabb_rule(g, p, dist, dx, dy, dz, r);
    SdfOut o;
    o.val = inb ? e.x : dist;
    o.grad = mk3(inb ? e.y : dx * r, inb ? e.z : dy * r, inb ? e.w : dz * r);
    return o;
}

// ----------------------------------------------------------------------------
// EXTENSION, opt-in (CachedSDF(interpolation="trilinear"), PVB_GRID_TRILINEAR): the reference looks up the NEAREST
// voxel and a stored gradient table (sdf.py:537-550).  This interpolates the value table trilinearly and returns the
// analytic gradient of the interpolant (per-cell finite differences of the corner values) -- smoother for
// optimisation, not comparable to the reference within 1e-5 (the difference is O(resolution)); it is validated
// against its own CPU restatement (oracle/port.py).  One arithmetic for every kernel that honours the flag
// (grid_trilinear_kernel, the composed kernels, robot_serial_kernel), so their results agree bit for bit.
__device__ __forceinline__ bool grid_in_range(const pvb_sdf_desc &g, f3 p) {
    return (p.x >= g.valid_lo[0]) & (p.x <= g.valid_hi[0]) & (p.y >= g.valid_lo[1]) & (p.y <= g.valid_hi[1]) &
           (p.z >= g.valid_lo[2]) & (p.z <= g.valid_hi[2]);
}

// In range only (grid_in_range(g, p)): the interpolant and its gradient.
__device__ __forceinline__ SdfOut grid_trilinear_interp(const pvb_sdf_desc &g, f3 p) {
    const float4 *tab = reinterpret_cast<const float4 *>(g.table);
    const int n0 = g.dims[0], n1 = g.dims[1], n2 = g.dims[2];
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
    SdfOut o;
    o.val = c0_ + fx * (c1_ - c0_);
    // d/dx: difference of the two y-z interpolated faces over the cell size, and likewise for y, z
    const float gx = (c1_ - c0_) * g.inv_res32[0];
    const float e0 = c01 - c00, e1 = c11 - c10;
    const float gy = (e0 + fx * (e1 - e0)) * g.inv_res32[1];
    const float z00 = v001 - v000, z01 = v011 - v010, z10 = v101 - v100, z11 = v111 - v110;
    const float z0 = z00 + fy * (z01 - z00), z1 = z10 + fy * (z11 - z10);
    const float gz = (z0 + fx * (z1 - z0)) * g.inv_res32[2];
    o.grad = mk3(n0 > 1 ? gx : 0.f, n1 > 1 ? gy : 0.f, n2 > 1 ? gz : 0.f);
    return o;
}

// Any point: the interpolant in range, the reference's point-to-AABB rule (sdf.py:555-571) out of range.
__device__ __forceinline__ SdfOut grid_trilinear_eval(const pvb_sdf_desc &g, f3 p) {
    if (grid_in_range(g, p)) return grid_trilinear_interp(g, p);
    float dist, ex, ey, ez, r;
    aabb_rule(g, p, dist, ex, ey, ez, r);
    SdfOut o;
    o.val = dist;
    o.grad = mk3(ex * r, ey * r, ez * r);
    return o;
}

__device__ __forceinline__ SdfOut sphere_eval(float radius, f3 p) {   // sdf.py:291-295
    const float r = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
    const float den = r + 1e-12f;
    SdfOut o;
    o.val = r - radius;
    o.grad = mk3(__fdiv_rn(p.x, den), __fdiv_rn(p.y, den), __fdiv_rn(p.z, den));
    return o;
}

// ----------------------------------------------------------------------------
// EXTENSION (not reference behaviour; the reference skips non-mesh URDF visuals): analytic URDF primitives, centred at
// the origin, exact Euclidean SDF.  Every operation is an explicit fmaf / _rn intrinsic or cannot be contracted, so
// the host build (-ffp-contract=off) gives the same bits as the device.
//
// BOX (PVB_KIND_BOX): half extents h = bb_max (bb_min = -h), e = |q| - h per axis.
//   outside (|max(e, 0)| > 0): value |max(e, 0)|, gradient the unit vector from the closest box point to q,
//     (sign(q_k) max(e_k, 0)) / value;
//   inside or on the surface: value max_k e_k, gradient s e_k for that axis -- the FIRST axis on ties -- with
//     s = q_k >= 0 ? +1 : -1 (-0 counts as +).
__device__ __forceinline__ SdfOut box_eval(const pvb_sdf_desc &d, f3 q) {
    const float ex = __fsub_rn(fabsf(q.x), d.bb_max[0]), ey = __fsub_rn(fabsf(q.y), d.bb_max[1]),
                ez = __fsub_rn(fabsf(q.z), d.bb_max[2]);
    const float wx = fmaxf(ex, 0.f), wy = fmaxf(ey, 0.f), wz = fmaxf(ez, 0.f);
    const float w2 = fmaf(wx, wx, fmaf(wy, wy, __fmul_rn(wz, wz)));
    SdfOut o;
    if (w2 > 0.f) {
        const float dist = sqrtf(w2);
        o.val = dist;
        o.grad = mk3(copysignf(__fdiv_rn(wx, dist), q.x), copysignf(__fdiv_rn(wy, dist), q.y),
                     copysignf(__fdiv_rn(wz, dist), q.z));
        return o;
    }
    // (also when max(e, 0) is nonzero but its square underflows: value max_k e_k, a few 1e-20 at most)
    int k = 0;
    float m = ex;
    if (ey > m) { m = ey; k = 1; }
    if (ez > m) { m = ez; k = 2; }
    o.val = m;
    o.grad = mk3(k == 0 ? (q.x >= 0.f ? 1.f : -1.f) : 0.f, k == 1 ? (q.y >= 0.f ? 1.f : -1.f) : 0.f,
                 k == 2 ? (q.z >= 0.f ? 1.f : -1.f) : 0.f);
    return o;
}

// CYLINDER (PVB_KIND_CYLINDER): axis along local z, radius r = radius, half length h = bb_max[2].  rho = |(x, y)|,
// radial unit u = (x, y) / rho, or (1, 0) when rho = 0; d = (rho - r, |z| - h); sz = z >= 0 ? +1 : -1.
//   outside (|max(d, 0)| > 0): w = max(d, 0), value |w|, gradient (w_0 u, w_1 sz) / |w|;
//   inside or on the surface: value max(d), gradient (u, 0) when d_0 >= d_1 (radial wins ties), else (0, 0, sz).
__device__ __forceinline__ SdfOut cylinder_eval(const pvb_sdf_desc &d, f3 q) {
    const float rho = sqrtf(fmaf(q.x, q.x, __fmul_rn(q.y, q.y)));
    const float ux = rho > 0.f ? __fdiv_rn(q.x, rho) : 1.f, uy = rho > 0.f ? __fdiv_rn(q.y, rho) : 0.f;
    const float sz = q.z >= 0.f ? 1.f : -1.f;
    const float dr = __fsub_rn(rho, d.radius), dz = __fsub_rn(fabsf(q.z), d.bb_max[2]);
    const float wr = fmaxf(dr, 0.f), wz = fmaxf(dz, 0.f);
    const float w2 = fmaf(wr, wr, __fmul_rn(wz, wz));
    SdfOut o;
    if (w2 > 0.f) {
        const float dist = sqrtf(w2);
        const float a = __fdiv_rn(wr, dist);
        o.val = dist;
        o.grad = mk3(__fmul_rn(a, ux), __fmul_rn(a, uy), __fmul_rn(__fdiv_rn(wz, dist), sz));
        return o;
    }
    const bool radial = dr >= dz;
    o.val = radial ? dr : dz;
    o.grad = radial ? mk3(ux, uy, 0.f) : mk3(0.f, 0.f, sz);
    return o;
}

// SPHERE / BOX / CYLINDER descriptor at q (in its own frame).  Any other kind is evaluated as a sphere: the entry
// points refuse kinds outside PVB_KIND_GRID .. PVB_KIND_CYLINDER, and GRID / MESH never reach this function.
__device__ __forceinline__ SdfOut primitive_eval(const pvb_sdf_desc &d, f3 q) {
    if (d.kind == PVB_KIND_BOX) return box_eval(d, q);
    if (d.kind == PVB_KIND_CYLINDER) return cylinder_eval(d, q);
    return sphere_eval(d.radius, q);
}


// ----------------------------------------------------------------------------
// Composition primitives shared by the point-major and the configuration-major kernels (ComposedSDF.__call__,
// sdf.py:392-433): the rigid transform into a sub-frame, the exact rejection bound, one "consider this sub-SDF"
// step of the running argmin, and the gradient rotation back to the object frame.

// The transforms of every query take the layout [S][n_cfg][4][4], row-major: the rows [R | t] of sub-SDF s in
// configuration cfg are the first three float4 of its matrix.
__host__ __device__ inline const float4 *xf_rows(const float *m, int n_cfg, int s, size_t cfg) {
    return reinterpret_cast<const float4 *>(m + ((size_t)s * n_cfg + cfg) * 16);
}
__host__ __device__ inline float4 *xf_rows(float *m, int n_cfg, int s, size_t cfg) {
    return reinterpret_cast<float4 *>(m + ((size_t)s * n_cfg + cfg) * 16);
}

// Transform3d.transform_points: R p + t (sdf.py:399); rows r0..r2 of the 4x4 object->sub-frame matrix
__device__ __forceinline__ f3 composed_xform(const float4 &r0, const float4 &r1, const float4 &r2, f3 v) {
    return mk3(fmaf(r0.x, v.x, fmaf(r0.y, v.y, fmaf(r0.z, v.z, r0.w))),
               fmaf(r1.x, v.x, fmaf(r1.y, v.y, fmaf(r1.z, v.z, r1.w))),
               fmaf(r2.x, v.x, fmaf(r2.y, v.y, fmaf(r2.z, v.z, r2.w))));
}

// squared distance from q to the sub-SDF's box (0 inside)
__device__ __forceinline__ float composed_aabb_lb2(const pvb_sdf_desc &d, f3 q) {
    const float ex = fmaxf(fmaxf(d.bb_min[0] - q.x, q.x - d.bb_max[0]), 0.f);
    const float ey = fmaxf(fmaxf(d.bb_min[1] - q.y, q.y - d.bb_max[1]), 0.f);
    const float ez = fmaxf(fmaxf(d.bb_min[2] - q.z, q.z - d.bb_max[2]), 0.f);
    return ex * ex + ey * ey + ez * ez;
}

// link_frame_to_obj_frame[i].transform_normals(g) = g @ inv(inv(M)[:3,:3]) = g @ M[:3,:3]
// (sdf.py:380-383, 409): the double inversion cancels, no inverse is needed.
__device__ __forceinline__ f3 composed_rotate_back(const float4 &r0, const float4 &r1, const float4 &r2, f3 g) {
    return mk3(fmaf(g.x, r0.x, fmaf(g.y, r1.x, g.z * r2.x)), fmaf(g.x, r0.y, fmaf(g.y, r1.y, g.z * r2.y)),
               fmaf(g.x, r0.z, fmaf(g.y, r1.z, g.z * r2.z)));
}

// Sub-SDF `s` (descriptor d, query q already in its frame) as a candidate for the running minimum
// (best, bg, bs) of one point; bs < 0 = nothing evaluated yet.  Skipped without touching its table / tree when
// provably not the argmin: value >= dist(q, box) - prune_margin (measured on the table for grids, fp32 slack for
// closed meshes).  torch.argmin semantics (sdf.py:421): smallest value, first index on ties -- whatever the
// visiting order.  kExt: the extension kinds are present -- GRID descriptors with PVB_GRID_TRILINEAR are evaluated
// through grid_trilinear_eval, SPHERE / BOX / CYLINDER through primitive_eval and pruned by the grid rule (their
// PVB_GRID_PRUNE_OK means the same bound holds).  A template flag, so that the nearest-voxel instantiations carry no
// code for the opt-in modes.
template <bool kMesh, bool kExt = false>
__device__ __forceinline__ void composed_consider(const pvb_sdf_desc &d, const NodeStage &st, int s, f3 q,
                                                  uint32_t mesh_mode, uint64_t idx, float &best, f3 &bg, int &bs) {
    SdfOut o;
    if (d.kind == PVB_KIND_GRID || (kExt && d.kind != PVB_KIND_MESH)) {
        if ((d.flags & PVB_GRID_PRUNE_OK) && bs >= 0) {
            const float thr = best + d.prune_margin;
            if (thr < 0.f || composed_aabb_lb2(d, q) > thr * thr) return;
        }
        // (the bound holds for the interpolant too: it is a convex combination of 8 corner values, and the weighted
        // mean distance of q to those corners is at most half a cell diagonal -- tests/test_trilinear_composed_cpu.py)
        if (kExt && d.kind != PVB_KIND_GRID) o = primitive_eval(d, q);
        else if (kExt && (d.flags & PVB_GRID_TRILINEAR)) o = grid_trilinear_eval(d, q);
        else o = grid_eval<kMesh, true>(d, st, q, mesh_mode, idx, nullptr);
    } else if (kMesh && d.kind == PVB_KIND_MESH) {
        // closed mesh, query outside its AABB: the value is +distance >= dist(q, AABB), so (a) skip it when that
        // bound already exceeds the running min, (b) otherwise search only within the running min and (c) skip
        // the parity walk -- all exact
        float init_d2 = PVB_INF;
        bool outside_box = false;
        if ((d.flags & PVB_MESH_CLOSED) && (mesh_mode & PVB_MESH_SIGNED)) {
            const float lb2 = composed_aabb_lb2(d, q);
            outside_box = lb2 > 0.f;
            if (outside_box && bs >= 0) {
                const float thr = best + d.prune_margin;
                if (thr < 0.f || lb2 > thr * thr) return;
                if (best > 0.f) init_d2 = thr * thr;
            }
        }
        int face;
        o = mesh_eval(d, st, q, mesh_mode, idx, nullptr, &face, init_d2, outside_box);
        if (face < 0) return;          // nothing within the running min: cannot be the argmin
    } else {
        o = sphere_eval(d.radius, q);
    }
    if (bs < 0 || o.val < best || (o.val == best && s < bs)) {
        best = o.val; bg = o.grad; bs = s;
    }
}

// One (configuration, point) pair of the composition: every sub-SDF through composed_consider, then the winning
// gradient rotated back to the object frame.  The per-pair work of composed_paired_kernel: the same sequence as the
// one-point path of composed_query_kernel (visiting order, nearest-bound-first for meshes, jitter index, rotation
// back), so that a paired query equals the per-configuration query on the same points bit for bit.
// (composed_query_kernel keeps its own copy of the loop: routed through this function, its mesh instantiations
// compiled to different SASS with more spills.)
//   descs / order: the sub-SDFs and the fixed visiting order (DescPack::order, bit-reversed)
//   load_xf(s, r0, r1, r2): rows 0..2 of sub-SDF s's object->sub-frame matrix for this configuration
//   pair: cfg * n_pts + i with the ABSOLUTE configuration index; the mesh ray jitter of sub-SDF s is seeded by
//   pair * n_sdf + s, so results do not depend on how the configurations are split over launches or GPUs
//   nearest_first / margin_max: see below (kMesh only)
struct ComposedOut { float val; f3 grad; int which; };

template <bool kMesh, bool kExt, class LoadXf>
__device__ __forceinline__ ComposedOut composed_point(const pvb_sdf_desc *descs, const unsigned char *order, int n_sdf,
                                                      const LoadXf &load_xf, const NodeStage &st, f3 p,
                                                      uint32_t mesh_mode, uint64_t pair, int nearest_first,
                                                      float margin_max) {
    float best = PVB_INF;
    f3 bg = mk3(0.f, 0.f, 0.f);
    int bs = -1;
    // Every sub-SDF in visiting order, skipped when provably not the argmin (composed_consider).  (Evaluating the
    // sub-SDF with the smallest AABB lower bound first -- an extra pass over all of them without table access -- saves
    // lookups but adds issue slots to a kernel that is issue-bound.)
    // ... except when sub-SDFs are MESHES (kMesh): an evaluation is a tree walk of thousands of instructions, so one
    // cheap pass computes every sub-SDF's AABB lower bound and the thread then evaluates them NEAREST BOUND FIRST,
    // stopping as soon as the smallest remaining bound exceeds the running minimum.  A fixed order evaluates every
    // sub-SDF that is a running record when its turn comes (~H_16 = 3.4 of 16 at C3, plus those inside the slack);
    // nearest-first evaluates the winner and its near ties.  Exact for the same reason as the fixed order: bounds are
    // conservative and the argmin keeps torch's first-index rule explicitly.
    bool ordered = false;
    if constexpr (kMesh) {
        if (n_sdf <= 32 && nearest_first) {
            ordered = true;
            float key[32];                           // squared lower bound; -1 = no valid bound (evaluate)
            unsigned todo = n_sdf >= 32 ? 0xffffffffu : ((1u << n_sdf) - 1u);
            for (int s = 0; s < n_sdf; ++s) {
                const pvb_sdf_desc &d = descs[s];
                float4 r0, r1, r2;
                load_xf(s, r0, r1, r2);
                const bool bounded = (d.kind == PVB_KIND_GRID || (kExt && d.kind != PVB_KIND_MESH))
                                         ? (d.flags & PVB_GRID_PRUNE_OK) != 0
                                         : (d.kind == PVB_KIND_MESH && (d.flags & PVB_MESH_CLOSED) && (mesh_mode & PVB_MESH_SIGNED));
                const float lb2 = bounded ? composed_aabb_lb2(d, composed_xform(r0, r1, r2, p)) : -1.f;
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
                const pvb_sdf_desc &d = descs[s];
                if (bs >= 0 && kmin >= 0.f) {
                    // every remaining bound is at least kmin: when even the most generous margin cannot bring it under
                    // the running minimum, nothing left can win (margins are per sub-SDF: test this one exactly, and
                    // stop the loop only on the margin-free comparison)
                    const float thr = best + d.prune_margin;
                    if (thr < 0.f || kmin > thr * thr) {
                        if (best + margin_max < 0.f || kmin > (best + margin_max) * (best + margin_max)) break;
                        continue;
                    }
                }
                float4 r0, r1, r2;
                load_xf(s, r0, r1, r2);
                composed_consider<kMesh, kExt>(d, st, s, composed_xform(r0, r1, r2, p), mesh_mode,
                                               pair * (uint64_t)n_sdf + (uint64_t)s, best, bg, bs);
            }
        }
    }
    for (int si = 0; si < (ordered ? 0 : n_sdf); ++si) {
        const int s = order[si];
        float4 r0, r1, r2;
        load_xf(s, r0, r1, r2);
        composed_consider<kMesh, kExt>(descs[s], st, s, composed_xform(r0, r1, r2, p), mesh_mode,
                                       pair * (uint64_t)n_sdf + (uint64_t)s, best, bg, bs);
    }
    float4 r0, r1, r2;
    load_xf(max(bs, 0), r0, r1, r2);
    ComposedOut o;
    o.val = best; o.grad = composed_rotate_back(r0, r1, r2, bg); o.which = bs;
    return o;
}

// Paired queries (composed_paired_kernel): flat pair index t in [0, cfg_count * n_pts) -> (configuration c relative
// to cfg_begin, point i).  64-bit throughout: cfg_count * n_pts may exceed 2^31 where n_pts alone does not.
__device__ __forceinline__ void paired_index(long long t, long long n_pts, long long &c, long long &i) {
    c = t / n_pts;
    i = t - c * n_pts;
}

// ----------------------------------------------------------------------------
// Index arithmetic of robot_serial_kernel (pvb_kernels.cu), kept here so that the CPU tier can check it exhaustively
// (tests/test_hostsim.py): which configurations a tile holds, and which 16-byte piece of a staging tile a thread flushes.

// Configuration tiles.  The first cfg_count / 32 tiles hold 32 configurations each (lanes = configurations, one point
// per warp step).  The remainder R = cfg_count % 32 is split by its binary digits into FULL tiles of 16 / 8 / 4 / 2 / 1
// configurations, in which the 32 lanes are 32 / LC point groups x LC configurations: no lane ever idles because the
// configuration count is not a multiple of 32 (200 = 6 x 32 + 8 would run a seventh tile at 8 of 32 lanes; the
// 25-configuration slab of an 8-GPU split at 25 of 32).
__device__ __forceinline__ void rs_tile(int cfg_count, int t, int &c0, int &lc_log2) {
    const int n_full = cfg_count >> 5;
    if (t < n_full) { c0 = t << 5; lc_log2 = 5; return; }
    int rem = cfg_count & 31, idx = t - n_full;
    c0 = n_full << 5;
    lc_log2 = 0;
    for (int b = 4; b >= 0; --b) {
        if (rem & (1 << b)) {
            if (idx == 0) { lc_log2 = b; return; }
            --idx;
            c0 += 1 << b;
        }
    }
}

// Launch limits of the robot-family kernels, shared by the host's route choice and the CPU tier.
// Grid rows: robot_serial_kernel and robot_clearance_kernel run one grid row per rs_tile tile, robot_query_kernel and
// composed_cfgmajor_kernel one per 32 configurations, and gridDim.y is at most 65535.
constexpr int kRsMaxGridRows = 65535;
__host__ __device__ inline int rs_tile_count(int cfg_count) {
    const int r = cfg_count & 31;
    return (cfg_count >> 5) + (r & 1) + ((r >> 1) & 1) + ((r >> 2) & 1) + ((r >> 3) & 1) + ((r >> 4) & 1);
}
// Points: robot_serial_kernel and robot_query_kernel index the points with int.  A step's end reaches
// n_pts + kRsIntPtsSpan - 1, the span being the points a block flushes at once in robot_serial_kernel's
// multi-destination form (8 warps x 32 point groups x 8 points; robot_query_kernel's 32-point tile is less), so a batch
// takes them only while that end stays below 2^31.
constexpr long long kRsIntPtsSpan = 2048;
__host__ __device__ inline bool rs_int_pts_ok(long long n_pts) { return n_pts <= 0x7fffffffll - (kRsIntPtsSpan - 1); }

// A staging tile holds LC = 32 >> sub_log2 configuration rows of row_pts = (1 << (w_log2 + chunk_log2 + sub_log2)) points:
// row_pts values and 3 row_pts gradient floats per row.  It leaves as LC * row_pts pieces of 16 bytes -- the first
// LC * row_pts / 4 are values, the rest gradients -- numbered so that consecutive pieces are consecutive in a row.
// Piece c -> (values or gradients, row, index of the piece inside the row's values / gradients).
__device__ __forceinline__ void rs_flush_piece(int c, int chunk_log2, int sub_log2, int w_log2, bool &is_val, int &row,
                                               int &part) {
    const int vper_log2 = w_log2 + chunk_log2 - 2 + sub_log2;    // value pieces per row = row_pts / 4 (a power of two)
    const int n_val = 32 << (w_log2 + chunk_log2 - 2);           // value pieces of the tile = LC * row_pts / 4
    is_val = c < n_val;
    const int g = is_val ? c : c - n_val;
    const int q = g >> vper_log2;                                // values: the row; gradients (3 x as many per row): 3 row + k
    // q / 3 without a division: q < 3 * 32, and (q * 43691) >> 17 == q / 3 for every q < 98304
    row = is_val ? q : (q * 43691) >> 17;
    part = is_val ? g & ((1 << vper_log2) - 1) : g - ((3 * row) << vper_log2);
}

// The first visit of a point goes to the link whose bounding sphere gives the smallest lower bound.  Instead of a
// compare + two selects per link, every bound becomes a key that carries its link index in the 3 low mantissa bits --
// (bits & ~7) | si, ONE LOP3 in the device build with ~7 in a register the compiler cannot fold -- and the smallest key
// of 8 (5 FMNMX) names the link.  A bound of -inf (not valid: never rejected) or +inf (slot beyond n_sdf) turns into a
// NaN pattern for si > 0, which fminf drops; the result is clamped to a real link.  Any link is a valid first visit --
// the visiting order never changes a result -- so the 7-ulp blur of the keys is harmless (tests/test_hostsim.py).
__device__ __forceinline__ int rs_and_or(int a, int b, int c) {
#ifdef __CUDA_ARCH__
    int r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
#else
    return (a & b) | c;
#endif
}

__device__ __forceinline__ float rs_bound_key(float lb, int low3_off, int si) {
    return __int_as_float(rs_and_or(__float_as_int(lb), low3_off, si));
}

// low3_off of the kernels: ~7 in a register the compiler cannot fold (n_sdf <= 8, so n_sdf >> 30 is 0)
__device__ __forceinline__ int rs_low3_off(int n_sdf) { return ~7 | (n_sdf >> 30); }

__device__ __forceinline__ float rs_min(float a, float b) {
#ifdef __CUDA_ARCH__
    return fminf(a, b);             // FMNMX: a NaN operand loses, signalling or not
#else
    return a != a ? b : (b != b ? a : (a < b ? a : b));     // (glibc's fminf turns a signalling NaN into a quiet one)
#endif
}

__device__ __forceinline__ int rs_nearest(const float (&key)[8], int n_sdf) {
    const float kmin = rs_min(rs_min(rs_min(key[0], key[1]), rs_min(key[2], key[3])),
                              rs_min(rs_min(key[4], key[5]), rs_min(key[6], key[7])));
    const int si = __float_as_int(kmin) & 7;
    return si < n_sdf - 1 ? si : n_sdf - 1;
}

// The bounding-sphere bound of robot_serial_kernel: value_s(p) >= |p - c_s| - r_s - prune_margin_s, c_s the centre of
// link s's AABB carried to the object frame, r_s its half-diagonal.  Split by what it varies with: the radius term is
// per link (host, constant bank), the centre per (configuration, link) (shared memory), the bound per point.
// sph_rad: r (+1e-4 relative, +1e-6: the fp32 roundings of the radius and the centre) + prune_margin; +inf without
// PVB_GRID_PRUNE_OK, so that the bound is -inf and never rejects.  visit_margin: the margin of the exact AABB test at
// the head of a visit, +inf without PVB_GRID_PRUNE_OK (best + inf never rejects either).
__host__ __device__ inline void rs_link_consts(const pvb_sdf_desc &d, float &sph_rad, float &visit_margin) {
    const float hx = 0.5f * (d.bb_max[0] - d.bb_min[0]), hy = 0.5f * (d.bb_max[1] - d.bb_min[1]),
                hz = 0.5f * (d.bb_max[2] - d.bb_min[2]);
    const float rad = sqrtf(hx * hx + hy * hy + hz * hz) * 1.0001f + 1e-6f;
    const bool ok = (d.flags & PVB_GRID_PRUNE_OK) != 0;
    sph_rad = ok ? rad + d.prune_margin : PVB_INF;
    visit_margin = ok ? d.prune_margin : PVB_INF;
}

// c_obj = R^T (c_link - t) from the rows r0..r2 of the object->link transform.  The bound needs an isometry: when
// |R R^T - I| exceeds 1e-5 the centre is NaN, which makes the bound NaN -- `lb > best` never rejects it and the
// nearest-link key (rs_bound_key / rs_nearest) ignores it.
__device__ __forceinline__ f3 rs_sphere_centre(const pvb_sdf_desc &d, float4 r0, float4 r1, float4 r2) {
    const f3 cen = mk3(0.5f * (d.bb_min[0] + d.bb_max[0]), 0.5f * (d.bb_min[1] + d.bb_max[1]),
                       0.5f * (d.bb_min[2] + d.bb_max[2]));
    const f3 u = mk3(cen.x - r0.w, cen.y - r1.w, cen.z - r2.w);
    const f3 co = mk3(r0.x * u.x + r1.x * u.y + r2.x * u.z, r0.y * u.x + r1.y * u.y + r2.y * u.z,
                      r0.z * u.x + r1.z * u.y + r2.z * u.z);
    const float e00 = r0.x * r0.x + r0.y * r0.y + r0.z * r0.z - 1.f, e11 = r1.x * r1.x + r1.y * r1.y + r1.z * r1.z - 1.f,
                e22 = r2.x * r2.x + r2.y * r2.y + r2.z * r2.z - 1.f;
    const float e01 = r0.x * r1.x + r0.y * r1.y + r0.z * r1.z, e02 = r0.x * r2.x + r0.y * r2.y + r0.z * r2.z,
                e12 = r1.x * r2.x + r1.y * r2.y + r1.z * r2.z;
    const float dev = fmaxf(fmaxf(fmaxf(fabsf(e00), fabsf(e11)), fmaxf(fabsf(e22), fabsf(e01))),
                            fmaxf(fabsf(e02), fabsf(e12)));
    return dev < 1e-5f ? co : mk3(__int_as_float(0x7fffffff), 0.f, 0.f);
}

// Slot si of a configuration's staged row of sphere centres ({x, y, z} of the 8 links back to back: 6 float4), from
// the link descriptors descs and its staged transform rows xf (link si at xf[3 si .. 3 si + 2]), both read only for
// si < n_sdf.  Slots beyond n_sdf get centre 0: with the radius -inf that rs_pack gives them, their bound is +inf --
// never the nearest, never visited.
__device__ __forceinline__ void rs_centre_slot(const pvb_sdf_desc *descs, int si, int n_sdf, const float4 *xf,
                                               float4 *sph) {
    const f3 co =
        si < n_sdf ? rs_sphere_centre(descs[si], xf[3 * si], xf[3 * si + 1], xf[3 * si + 2]) : mk3(0.f, 0.f, 0.f);
    float *c = reinterpret_cast<float *>(sph) + 3 * si;
    c[0] = co.x; c[1] = co.y; c[2] = co.z;
}

__device__ __forceinline__ float rsqrt_approx(float x) {      // one MUFU.RSQ, no denormal fix-up (callers keep x >= 1e-20)
#ifdef __CUDA_ARCH__
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return 1.0f / sqrtf(x);
#endif
}

// sqrt(0.9998) * 0.999999: 0.9998 on the squared distance absorbs the 1e-5 non-rigidity tolerated above, 0.999999 the
// approximate reciprocal square root (2 ulp) and the roundings of the three fused multiply-adds
constexpr float kRsBoundScale = 0.99989899f;

// lb <= value_s(p) for the centre c and the link's sph_rad.  + 1e-20 keeps the argument of the reciprocal square root
// a normal number (and raises the bound by < 1e-10, inside the 1e-6 slack of the radius).  Slots beyond n_sdf: c = 0
// and sph_rad = -inf give +inf.
__device__ __forceinline__ float rs_sphere_lb(f3 p, float cx, float cy, float cz, float sph_rad) {
    const float dx = p.x - cx, dy = p.y - cy, dz = p.z - cz;
    const float d2 = fmaf(dz, dz, fmaf(dy, dy, fmaf(dx, dx, 1e-20f)));
    return fmaf(d2 * rsqrt_approx(d2), kRsBoundScale, -sph_rad);
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

// In-range + certain: the record of the nearest voxel, same arithmetic as grid_eval.
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

// PVB_GRID_TRILINEAR link: the interpolant of grid_trilinear_eval in range; out of range the
// point-to-AABB rule, which is the same for both modes, out of line as above.
__device__ __forceinline__ float4 robot_lookup_trilinear(const pvb_sdf_desc &g, f3 p) {
    if (grid_in_range(g, p)) {
        const SdfOut o = grid_trilinear_interp(g, p);
        return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
    }
    return robot_lookup_slow(&g, p.x, p.y, p.z);
}

// SPHERE / BOX / CYLINDER link: primitive_eval, the arithmetic of every other kernel.  Out of line,
// like robot_lookup_slow: 9 inlined copies (the first visit + 8 unrolled links) would nearly double the code of the
// kernel's extension instantiations, which trilinear robots run too.
__device__ __noinline__ float4 robot_primitive(const pvb_sdf_desc *dp, float qx, float qy, float qz) {
    const SdfOut o = primitive_eval(*dp, mk3(qx, qy, qz));
    return make_float4(o.val, o.grad.x, o.grad.y, o.grad.z);
}

// ----------------------------------------------------------------------------
// Swept queries (robot_swept_kernel / composed_swept_kernel, pvb_composed_query_swept): the minimum over a slab of
// configurations at every point.  The result is the per-configuration result (value, gradient, which) of the
// configuration c* such that (value, c, which) is lexicographically smallest: c* is the FIRST configuration attaining
// the minimum value, and which is that configuration's own argmin.

// The lexicographic order of two configurations' results at one point: a before b.  Configurations are distinct, so
// the sub-SDF index never decides.
__device__ __forceinline__ bool swept_before(float va, int ca, float vb, int cb) {
    return va < vb || (va == vb && ca < cb);
}

// The running result of one point.  cfg < 0: nothing folded yet.
struct SweptBest { float val; f3 grad; int cfg; int which; };

// Fold the result of a configuration (or the winner of a tile of configurations) into the point's running result.
// Configurations arrive in ascending order, so a later one replaces the running result only when STRICTLY smaller.
__device__ __forceinline__ void swept_fold(SweptBest &b, float val, f3 grad, int cfg, int which) {
    if (b.cfg < 0 || val < b.val) { b.val = val; b.grad = grad; b.cfg = cfg; b.which = which; }
}

// One lane of robot_swept_kernel: one (configuration, point) pair, its links visited nearest-sphere first (`pred`)
// and then in index order.  The prune threshold is the smaller of the lane's own running value and `bp`, the point's
// best value over the configurations of earlier tiles: a link is skipped only when a lower bound of its value is
// STRICTLY above the threshold, so it can neither be this configuration's argmin nor beat an earlier configuration --
// links whose value ties are always evaluated, and the visiting order never changes c* or which.
//   lb: the bounding-sphere bounds (rs_sphere_lb; +inf for slots beyond n_sdf, which are never visited once a link has
//   been evaluated, since values are finite); link(si, thr, o): transform the point into link si's frame, return false
//   when its exact AABB bound (margin included) is strictly above thr, else evaluate it into o = (value, link-frame
//   gradient).
// The result is (best, bg, bs): this configuration's per-configuration result whenever best <= bp; when best > bp it
// may differ from it, but then the configuration cannot win (its true minimum is above bp as well).  bs < 0: every
// link was pruned (best = +inf > bp).
template <class Link>
__device__ __forceinline__ void rs_swept_pair(const float (&lb)[8], int pred, float bp, const Link &link, float &best,
                                              f3 &bg, int &bs) {
    best = PVB_INF; bg = mk3(0.f, 0.f, 0.f); bs = -1;
    auto visit = [&](const int si) {
        float4 o;
        if (!link(si, fminf(best, bp), o)) return;
        if (bs < 0 || o.x < best || (o.x == best && si < bs)) { best = o.x; bg = mk3(o.y, o.z, o.w); bs = si; }
    };
    if (!(lb[pred] > bp)) visit(pred);
#pragma unroll
    for (int si = 0; si < 8; ++si)
        if (si != pred && !(lb[si] > fminf(best, bp))) visit(si);
}

// One link of the robot-family kernels evaluated at q in its frame: analytic primitive, trilinear interpolant or
// nearest voxel (kExt = false: nearest voxel only).
template <bool kExt>
__device__ __forceinline__ float4 rs_link_eval(const pvb_sdf_desc &d, f3 q) {
    return (kExt && d.kind != PVB_KIND_GRID)         ? robot_primitive(&d, q.x, q.y, q.z)
           : (kExt && (d.flags & PVB_GRID_TRILINEAR)) ? robot_lookup_trilinear(d, q)
                                                      : robot_lookup(d, q);
}

// The `link` of rs_swept_pair in the robot-family kernels: p carried into the link's frame by its rows r0..r2; false
// when thr + visit_margin is negative or the exact AABB bound is above it, else the link evaluated into o.
template <bool kExt>
__device__ __forceinline__ bool rs_link_visit(const pvb_sdf_desc &d, float visit_margin, const float4 &r0,
                                              const float4 &r1, const float4 &r2, f3 p, float thr, float4 &o) {
    const f3 q = composed_xform(r0, r1, r2, p);
    const float tm = thr + visit_margin;
    if (tm < 0.f || composed_aabb_lb2(d, q) > tm * tm) return false;
    o = rs_link_eval<kExt>(d, q);
    return true;
}

// The bounds of point p from the 8 links' bounding spheres (rs_sphere_lb) and their nearest-link keys (rs_bound_key),
// from one staged row of sphere centres ({x, y, z} of the 8 links back to back: 6 float4).  A link whose mask bit is
// clear gets +inf.
__device__ __forceinline__ void rs_point_bounds(const float4 *sph, const float *sph_rad, f3 p, int low3_off,
                                                unsigned mask, float (&lb)[8], float (&key)[8]) {
    float cen[24];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const float4 c4 = sph[j];
        cen[4 * j] = c4.x; cen[4 * j + 1] = c4.y; cen[4 * j + 2] = c4.z; cen[4 * j + 3] = c4.w;
    }
#pragma unroll
    for (int si = 0; si < 8; ++si) {
        lb[si] = ((mask >> si) & 1u) ? rs_sphere_lb(p, cen[3 * si], cen[3 * si + 1], cen[3 * si + 2], sph_rad[si])
                                     : PVB_INF;
        key[si] = rs_bound_key(lb[si], low3_off, si);
    }
}

// ----------------------------------------------------------------------------
// Clearance queries (robot_clearance_kernel / composed_clearance_kernel / clearance_finish_kernel,
// pvb_composed_query_clearance): for every configuration and every segment of points, the per-configuration result at
// the point i* that minimises (value, i) lexicographically -- the FIRST point of the segment attaining the minimum.
//
// A candidate (value v, point i of its segment) becomes one 64-bit key: an order-preserving image of v in the high
// word, i in the low word.  The unsigned order of keys is exactly the (value, i) order, so a 64-bit atomicMin over keys
// is an exact reduction whose result does not depend on the order in which candidates arrive (block count, block
// scheduling, SM count).  -0 is mapped to +0 first, so that the two compare equal as they do in torch; every NaN maps to
// the largest pattern, so a NaN value ranks above every number (+inf included), and ~0 ("no candidate yet") decodes to
// NaN.
__device__ __forceinline__ uint64_t clearance_key(float v, uint32_t i) {
    const uint32_t b = (uint32_t)__float_as_int(v == 0.f ? 0.f : v);
    const uint32_t h = v != v ? 0xffffffffu : ((b & 0x80000000u) ? ~b : (b | 0x80000000u));
    return ((uint64_t)h << 32) | i;
}

// The value of a key (+0 for a zero of either sign; a NaN for every NaN and for ~0).
__device__ __forceinline__ float clearance_key_value(uint64_t k) {
    const uint32_t h = (uint32_t)(k >> 32);
    return __int_as_float((int)((h & 0x80000000u) ? (h & 0x7fffffffu) : ~h));
}

// ----------------------------------------------------------------------------
// Self-clearance queries (robot_self_clearance_kernel / self_clearance_finish_kernel,
// pvb_composed_query_self_clearance): for configuration a, over every source sub-SDF i, every sub-SDF j that row i of
// the mask allows (bit j; the diagonal is cleared) and every link point k of i, the minimum of sdf_j(M_j(a) x) with
// x = W_i(a) link_pts[i][k] posed by composed_xform.  The minimum is taken over (value, i, k) lexicographically, and
// for that point the first allowed j attaining the value wins.
//
// One key per configuration: the value as in clearance_key, (i << 24) | k in the low word (k < 2^24, i < 8), so the
// unsigned order of keys is exactly the (value, i, k) order and every source of a configuration prunes against the
// best value any of them has reached.
__device__ __forceinline__ uint64_t self_clearance_key(float v, int i, int k) {
    return clearance_key(v, ((uint32_t)i << 24) | (uint32_t)k);
}

struct SelfClearanceOut { float val; f3 grad; int src; int point; int which; };

// The result of one configuration from its key: (i, k) decoded, x posed again, then every allowed sub-SDF of row i
// evaluated at x in index order (first index on ties) and the winner's gradient rotated back -- what
// composed_point of the composition of the allowed sub-SDFs gives at x.  ~0 (no allowed pair): +inf, 0, -1.
//   load_xf(s, r0, r1, r2) / load_inv(s, ...): rows of M_s / W_s of this configuration; load_pt(i, k): the link point;
//   eval(s, q): (value, sub-frame gradient) of sub-SDF s at q in its frame
template <class LoadXf, class LoadInv, class LoadPt, class Eval>
__device__ __forceinline__ SelfClearanceOut self_clearance_finish_one(uint64_t key, const unsigned char *masks,
                                                                      int n_sdf, const LoadXf &load_xf,
                                                                      const LoadInv &load_inv, const LoadPt &load_pt,
                                                                      const Eval &eval) {
    SelfClearanceOut o;
    if (key == ~0ull) {
        o.val = PVB_INF; o.grad = mk3(0.f, 0.f, 0.f); o.src = -1; o.point = -1; o.which = -1;
        return o;
    }
    const uint32_t low = (uint32_t)key;
    const int i = (int)(low >> 24), k = (int)(low & 0xffffffu);
    float4 w0, w1, w2;
    load_inv(i, w0, w1, w2);
    const f3 x = composed_xform(w0, w1, w2, load_pt(i, k));
    const unsigned mask = masks[i];
    float best = PVB_INF;
    f3 bg = mk3(0.f, 0.f, 0.f);
    int bs = -1;
    for (int s = 0; s < n_sdf; ++s) {
        if (!((mask >> s) & 1u)) continue;
        float4 r0, r1, r2;
        load_xf(s, r0, r1, r2);
        const float4 e = eval(s, composed_xform(r0, r1, r2, x));
        if (bs < 0 || e.x < best) { best = e.x; bg = mk3(e.y, e.z, e.w); bs = s; }
    }
    float4 r0, r1, r2;
    load_xf(max(bs, 0), r0, r1, r2);
    o.val = best; o.grad = composed_rotate_back(r0, r1, r2, bg); o.src = i; o.point = k; o.which = bs;
    return o;
}

// ----------------------------------------------------------------------------
// Collision-cost queries (robot_collision_cost_kernel / collision_cost_finish_kernel,
// pvb_composed_query_collision_cost): for configuration a and segment b of the points, with margin m,
//   cost[a, b]        = sum_n max(0, m - d)^2
//   twist[a, b, s, :] = sum over the points n whose argmin sub-SDF is s and d < m of
//                       (2 (m - d) g, 2 (m - d) (p x g))
// where (d, g, s) is the per-configuration result (value, object-frame gradient, first sub-SDF attaining it) at p.
//
// A segment of seg_len points is summed in chunks of collision_cost_chunk(seg_len) consecutive points.  The chunk
// depends on seg_len alone (whole multiples of 512 points, at most 256 chunks per segment; a shorter segment is one
// chunk), and so does the order of every sum: within a chunk, the points j = w, w + 8, w + 16, ... in ascending order
// per accumulator w = 0..7 (fp32), then the 8 accumulators in order (fp64, rounded to fp32 once per chunk), then the
// chunks in order (fp64).  No configuration tile, slab offset, grid size or SM count enters it.
constexpr int kCcWarps = 8;                       // accumulators per chunk: the warps of a block
__host__ __device__ inline long long collision_cost_chunk(long long seg_len) {
    const long long c = 512 * ((seg_len + 512 * 256 - 1) / (512 * 256));
    return c < seg_len ? c : (seg_len > 0 ? seg_len : 1);
}
__host__ __device__ inline long long collision_cost_chunks(long long seg_len) {
    return seg_len > 0 ? (seg_len + collision_cost_chunk(seg_len) - 1) / collision_cost_chunk(seg_len) : 0;
}

// a b - c d to within about one ulp of the result (Kahan's difference of products, two fused multiply-adds): the
// moment p x g cancels when p is nearly parallel to g, and the plain difference would then carry an error of the
// order of u |p| |g| instead of u |p x g|
__device__ __forceinline__ float cc_diff_of_products(float a, float b, float c, float d) {
    const float w = c * d;
    const float e = fmaf(-c, d, w);
    return fmaf(a, b, -w) + e;
}

// The terms of one contributing pair (d < m): cost (m - d)^2, then 2 (m - d) g and 2 (m - d) (p x g).
struct CollisionTerm { float cost; float tw[6]; };
__device__ __forceinline__ CollisionTerm collision_cost_term(float m, float d, f3 g, f3 p) {
    const float h = m - d, t = 2.f * h;
    CollisionTerm o;
    o.cost = h * h;
    o.tw[0] = t * g.x; o.tw[1] = t * g.y; o.tw[2] = t * g.z;
    o.tw[3] = t * cc_diff_of_products(p.y, g.z, p.z, g.y);
    o.tw[4] = t * cc_diff_of_products(p.z, g.x, p.x, g.z);
    o.tw[5] = t * cc_diff_of_products(p.x, g.y, p.y, g.x);
    return o;
}

// Whether a point can contribute for a configuration at all: some link's lower bound is below m.  A NaN bound (a
// transform that is not an isometry) or -inf (a link without a valid bound) always passes; the +inf bound of a slot
// beyond n_sdf never does.
__device__ __forceinline__ bool collision_cost_near(const float (&lb)[8], float m) {
    bool near = false;
#pragma unroll
    for (int si = 0; si < 8; ++si) near |= !(lb[si] >= m);
    return near;
}

// ----------------------------------------------------------------------------
// Self-collision-cost queries (robot_self_collision_cost_kernel, pvb_composed_query_self_collision_cost).
// Inputs: a composition of S sub-SDFs with transforms M_s(a), and W_s = _affine_inverse(M_s); link_points [S, K, 3],
// each row in its own sub-SDF's frame; allowed [S, S] bool (the diagonal is ignored); a margin m, rounded to fp32
// exactly as _collision_cost_margin does.  For configuration a, every source i and every point k:
//   * x = W_i(a) . link_points[i, k], posed with composed_xform.  This is the same posed point as in
//     pvb_transform_points_paired and self_clearance.
//   * (d, g, j) is what query_paired(..., return_which=True) of the composition of row i's allowed sub-SDFs gives at
//     x: the value, the object-frame gradient, and the first allowed sub-SDF attaining the value.  These are the
//     per-point values _composed_self_clearance already uses.
//   * When d < m, with h = m - d and tau = 2h (g, x x g):
//       cost[a] += h^2
//       twist[a, j] += tau.  The target moves.  This is the same term and sign as collision_cost_term.
//       twist[a, i] -= tau.  The source moves.  Its point travels with it, so d changes by +g . (v + w x x).
//   * twist[a, s] is therefore the derivative of the cost when sub-SDF s alone moves by an object-frame twist (v, w)
//     about the origin.  This is the convention of collision_cost, so RobotSDF.joint_gradient applies unchanged.
//   * A configuration with no allowed pair, or with no point below m, costs exactly 0 and has all-zero twists.
//
// Summation order (robot_self_collision_cost_kernel): one warp owns a configuration.  Lane l takes the points
// k = l, l + 32, l + 64, ... of every source, sources in ascending index order, and adds each term into its own fp32
// accumulators (cost, and the 6 S twist components); at the end the 32 lanes' accumulators are added in lane order in
// fp64 and rounded to fp32 once.  The order depends on K, S and allowed alone: not on the slab, the grid or the SM
// count, so repeated calls give identical bits and a slab reproduces the rows of the full call.
constexpr int kSccLanes = 32;                     // lanes of a configuration's warp: its accumulators

}  // namespace pvb
