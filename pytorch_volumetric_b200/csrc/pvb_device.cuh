// pvb_device.cuh -- device-side building blocks shared by the sm_90a kernels.
//
//   grid_eval      CachedSDF.__call__ for one point          (reference sdf.py:535-571)
//   bvh_closest    closest point on the mesh                 (Embree rtcPointQuery role, sdf.py:134)
//   bvh_parity     ray/triangle crossing parity              (count_intersections role, sdf.py:152-154)
//   mesh_eval      ObjectFactory._do_object_frame_closest_point epilogue (sdf.py:139-164)
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

__device__ __forceinline__ SdfOut sphere_eval(float radius, f3 p) {   // sdf.py:291-295
    const float r = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
    const float den = r + 1e-12f;
    SdfOut o;
    o.val = r - radius;
    o.grad = mk3(__fdiv_rn(p.x, den), __fdiv_rn(p.y, den), __fdiv_rn(p.z, den));
    return o;
}


// ----------------------------------------------------------------------------
// Composition primitives shared by the point-major and the configuration-major kernels (ComposedSDF.__call__,
// sdf.py:392-433): the rigid transform into a sub-frame, the exact rejection bound, one "consider this sub-SDF"
// step of the running argmin, and the gradient rotation back to the object frame.

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
// visiting order.
template <bool kMesh>
__device__ __forceinline__ void composed_consider(const pvb_sdf_desc &d, const NodeStage &st, int s, f3 q,
                                                  uint32_t mesh_mode, uint64_t idx, float &best, f3 &bg, int &bs) {
    SdfOut o;
    if (d.kind == PVB_KIND_GRID) {
        if ((d.flags & PVB_GRID_PRUNE_OK) && bs >= 0) {
            const float thr = best + d.prune_margin;
            if (thr < 0.f || composed_aabb_lb2(d, q) > thr * thr) return;
        }
        o = grid_eval<kMesh, true>(d, st, q, mesh_mode, idx, nullptr);
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

}  // namespace pvb
