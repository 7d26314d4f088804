/*
 * oracle/geom.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the geometry arithmetic that the reference obtains from
 * Open3D / Embree (third-party, not vendored in the reference, version
 * unpinned in pyproject.toml:54-61):
 *
 *   - RaycastingScene.compute_closest_points   (reference call site
 *     src/pytorch_volumetric/sdf.py:134)  -> orc_closest_points_*
 *   - RaycastingScene.count_intersections      (sdf.py:153)
 *                                              -> orc_count_intersections_*
 *
 * Embree's point query uses the closest-point-on-triangle routine of
 * C. Ericson, "Real-Time Collision Detection" section 5.1.5 in fp32; that
 * published algorithm is restated here.  Ties between equidistant triangles
 * are broken towards the lowest face index (Embree's own tie-break depends on
 * its BVH traversal order and cannot be reproduced -- "parity unpinned" for
 * the face id of exact ties; the distance is unaffected).
 *
 * Two evaluators are provided for each query:
 *   *_brute : O(N*T) exhaustive loop.  This is the checker the parity tests
 *             use: no acceleration structure, nothing to get wrong.
 *   *_bvh   : a plain binary median-split BVH + OpenMP, used ONLY as the
 *             timed CPU baseline in bench.py (so that the CPU arm is not a
 *             strawman) and cross-checked against *_brute in the CPU tests.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library.
 *
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp -shared).
 * -ffp-contract=off keeps every fp32 operation individually rounded, as
 * x86 Embree builds without FMA contraction across statements would.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct { float x, y, z; } v3;

static inline v3 v3sub(v3 a, v3 b) { v3 r = {a.x - b.x, a.y - b.y, a.z - b.z}; return r; }
static inline v3 v3add(v3 a, v3 b) { v3 r = {a.x + b.x, a.y + b.y, a.z + b.z}; return r; }
static inline v3 v3mul(v3 a, float s) { v3 r = {a.x * s, a.y * s, a.z * s}; return r; }
static inline float v3dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline v3 ldv(const float *p) { v3 r = {p[0], p[1], p[2]}; return r; }

/* Ericson RTCD 5.1.5 (the routine Embree's closest-point tutorial/user code
 * and Open3D's ClosestPointFunc use). */
static v3 closest_pt_triangle(v3 p, v3 a, v3 b, v3 c)
{
    const v3 ab = v3sub(b, a), ac = v3sub(c, a), ap = v3sub(p, a);
    const float d1 = v3dot(ab, ap), d2 = v3dot(ac, ap);
    if (d1 <= 0.f && d2 <= 0.f) return a;

    const v3 bp = v3sub(p, b);
    const float d3 = v3dot(ab, bp), d4 = v3dot(ac, bp);
    if (d3 >= 0.f && d4 <= d3) return b;

    const float vc = d1 * d4 - d3 * d2;
    if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
        const float v = d1 / (d1 - d3);
        return v3add(a, v3mul(ab, v));
    }

    const v3 cp = v3sub(p, c);
    const float d5 = v3dot(ab, cp), d6 = v3dot(ac, cp);
    if (d6 >= 0.f && d5 <= d6) return c;

    const float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
        const float w = d2 / (d2 - d6);
        return v3add(a, v3mul(ac, w));
    }

    const float va = d3 * d6 - d5 * d4;
    if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) {
        const float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        return v3add(b, v3mul(v3sub(c, b), w));
    }

    const float denom = 1.f / (va + vb + vc);
    const float v = vb * denom, w = vc * denom;
    return v3add(a, v3add(v3mul(ab, v), v3mul(ac, w)));
}

/* Ray/triangle hit test used for the parity count (sdf.py:152-154).  Embree's
 * exact fp32 intersector cannot be reproduced; the oracle evaluates the
 * Moller-Trumbore predicate in fp64 on the fp32 inputs, i.e. the
 * mathematically intended answer: hit iff the ray o + t*d, t in [0, inf),
 * crosses the closed triangle. */
static int ray_hits_triangle(const double o[3], const double d[3], v3 a, v3 b, v3 c)
{
    const double e1[3] = {(double)b.x - a.x, (double)b.y - a.y, (double)b.z - a.z};
    const double e2[3] = {(double)c.x - a.x, (double)c.y - a.y, (double)c.z - a.z};
    const double pv[3] = {d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0]};
    const double det = e1[0] * pv[0] + e1[1] * pv[1] + e1[2] * pv[2];
    if (det == 0.0) return 0;
    const double inv = 1.0 / det;
    const double tv[3] = {o[0] - a.x, o[1] - a.y, o[2] - a.z};
    const double u = (tv[0] * pv[0] + tv[1] * pv[1] + tv[2] * pv[2]) * inv;
    if (u < 0.0 || u > 1.0) return 0;
    const double qv[3] = {tv[1] * e1[2] - tv[2] * e1[1], tv[2] * e1[0] - tv[0] * e1[2], tv[0] * e1[1] - tv[1] * e1[0]};
    const double v = (d[0] * qv[0] + d[1] * qv[1] + d[2] * qv[2]) * inv;
    if (v < 0.0 || u + v > 1.0) return 0;
    const double t = (e2[0] * qv[0] + e2[1] * qv[1] + e2[2] * qv[2]) * inv;
    return t >= 0.0;
}

/* ------------------------------------------------------------------ brute */

/* verts: V x 3 fp32, faces: T x 3 int32, pts: N x 3 fp32.
 * out_closest N x 3, out_dist2 N (squared distance, fp32), out_face N int32. */
void orc_closest_points_brute(const float *verts, const int32_t *faces, int64_t T,
                              const float *pts, int64_t N,
                              float *out_closest, float *out_dist2, int32_t *out_face)
{
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < N; ++i) {
        const v3 p = ldv(pts + 3 * i);
        float best = INFINITY;
        int32_t bf = -1;
        v3 bc = {NAN, NAN, NAN};
        for (int64_t t = 0; t < T; ++t) {
            const v3 a = ldv(verts + 3 * (int64_t)faces[3 * t]);
            const v3 b = ldv(verts + 3 * (int64_t)faces[3 * t + 1]);
            const v3 c = ldv(verts + 3 * (int64_t)faces[3 * t + 2]);
            const v3 q = closest_pt_triangle(p, a, b, c);
            const v3 g = v3sub(q, p);
            const float d2 = v3dot(g, g);
            if (d2 < best) { best = d2; bf = (int32_t)t; bc = q; }
        }
        out_closest[3 * i] = bc.x; out_closest[3 * i + 1] = bc.y; out_closest[3 * i + 2] = bc.z;
        out_dist2[i] = best;
        out_face[i] = bf;
    }
}

/* rays: N x 6 fp32 (origin, direction); out_count N int32. */
void orc_count_intersections_brute(const float *verts, const int32_t *faces, int64_t T,
                                   const float *rays, int64_t N, int32_t *out_count)
{
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < N; ++i) {
        const double o[3] = {rays[6 * i], rays[6 * i + 1], rays[6 * i + 2]};
        const double d[3] = {rays[6 * i + 3], rays[6 * i + 4], rays[6 * i + 5]};
        int32_t cnt = 0;
        for (int64_t t = 0; t < T; ++t) {
            const v3 a = ldv(verts + 3 * (int64_t)faces[3 * t]);
            const v3 b = ldv(verts + 3 * (int64_t)faces[3 * t + 1]);
            const v3 c = ldv(verts + 3 * (int64_t)faces[3 * t + 2]);
            cnt += ray_hits_triangle(o, d, a, b, c);
        }
        out_count[i] = cnt;
    }
}

/* -------------------------------------------------------------------- bvh */
/* Plain binary BVH (median split on the longest centroid axis, <= 4
 * triangles per leaf).  Timing baseline only. */

typedef struct {
    float lo[3], hi[3];
    int32_t left, right;   /* children; leaf if left < 0 */
    int32_t start, count;  /* triangle range for leaves */
} bnode;

typedef struct {
    bnode *nodes; int32_t n_nodes;
    int32_t *order;        /* triangle permutation */
    float *tri;            /* T x 9, permuted triangle vertices */
    int64_t T;
} obvh;

static const float *g_cent; static int g_axis;
static int cmp_axis(const void *a, const void *b)
{
    const float ca = g_cent[3 * (int64_t)(*(const int32_t *)a) + g_axis];
    const float cb = g_cent[3 * (int64_t)(*(const int32_t *)b) + g_axis];
    return (ca > cb) - (ca < cb);
}

static int32_t build_rec(obvh *bv, const float *tri9, const float *cent, int32_t start, int32_t count)
{
    const int32_t id = bv->n_nodes++;
    bnode *n = &bv->nodes[id];
    float clo[3] = {INFINITY, INFINITY, INFINITY}, chi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int k = 0; k < 3; ++k) { n->lo[k] = INFINITY; n->hi[k] = -INFINITY; }
    for (int32_t i = start; i < start + count; ++i) {
        const int32_t t = bv->order[i];
        for (int v = 0; v < 3; ++v)
            for (int k = 0; k < 3; ++k) {
                const float x = tri9[9 * (int64_t)t + 3 * v + k];
                if (x < n->lo[k]) n->lo[k] = x;
                if (x > n->hi[k]) n->hi[k] = x;
            }
        for (int k = 0; k < 3; ++k) {
            const float c = cent[3 * (int64_t)t + k];
            if (c < clo[k]) clo[k] = c;
            if (c > chi[k]) chi[k] = c;
        }
    }
    n->start = start; n->count = count; n->left = n->right = -1;
    if (count <= 4) return id;
    int ax = 0;
    if (chi[1] - clo[1] > chi[ax] - clo[ax]) ax = 1;
    if (chi[2] - clo[2] > chi[ax] - clo[ax]) ax = 2;
    g_cent = cent; g_axis = ax;
    qsort(bv->order + start, (size_t)count, sizeof(int32_t), cmp_axis);
    const int32_t half = count / 2;
    const int32_t l = build_rec(bv, tri9, cent, start, half);
    const int32_t r = build_rec(bv, tri9, cent, start + half, count - half);
    bv->nodes[id].left = l; bv->nodes[id].right = r;
    return id;
}

void *orc_bvh_create(const float *verts, const int32_t *faces, int64_t T)
{
    obvh *bv = (obvh *)calloc(1, sizeof(obvh));
    bv->T = T;
    bv->nodes = (bnode *)malloc(sizeof(bnode) * (size_t)(2 * T + 1));
    bv->order = (int32_t *)malloc(sizeof(int32_t) * (size_t)T);
    float *tri9 = (float *)calloc(1, sizeof(float) * 9 * (size_t)T);
    float *cent = (float *)calloc(1, sizeof(float) * 3 * (size_t)T);
    for (int64_t t = 0; t < T; ++t) {
        bv->order[t] = (int32_t)t;
        for (int v = 0; v < 3; ++v)
            for (int k = 0; k < 3; ++k)
                tri9[9 * t + 3 * v + k] = verts[3 * (int64_t)faces[3 * t + v] + k];
        for (int k = 0; k < 3; ++k)
            cent[3 * t + k] = (tri9[9 * t + k] + tri9[9 * t + 3 + k] + tri9[9 * t + 6 + k]) * (1.f / 3.f);
    }
    build_rec(bv, tri9, cent, 0, (int32_t)T);
    bv->tri = (float *)malloc(sizeof(float) * 9 * (size_t)T);
    for (int64_t i = 0; i < T; ++i) memcpy(bv->tri + 9 * i, tri9 + 9 * (int64_t)bv->order[i], 9 * sizeof(float));
    free(tri9); free(cent);
    return bv;
}

void orc_bvh_destroy(void *h)
{
    obvh *bv = (obvh *)h;
    if (!bv) return;
    free(bv->nodes); free(bv->order); free(bv->tri); free(bv);
}

static inline float box_dist2(const bnode *n, v3 p)
{
    const float dx = fmaxf(fmaxf(n->lo[0] - p.x, 0.f), p.x - n->hi[0]);
    const float dy = fmaxf(fmaxf(n->lo[1] - p.y, 0.f), p.y - n->hi[1]);
    const float dz = fmaxf(fmaxf(n->lo[2] - p.z, 0.f), p.z - n->hi[2]);
    return dx * dx + dy * dy + dz * dz;
}

void orc_closest_points_bvh(const void *h, const float *pts, int64_t N,
                            float *out_closest, float *out_dist2, int32_t *out_face)
{
    const obvh *bv = (const obvh *)h;
#pragma omp parallel for schedule(dynamic, 1024)
    for (int64_t i = 0; i < N; ++i) {
        const v3 p = ldv(pts + 3 * i);
        float best = INFINITY; int32_t bf = -1; v3 bc = {NAN, NAN, NAN};
        int32_t stack[128]; float sd[128]; int sp = 0;
        stack[sp] = 0; sd[sp++] = box_dist2(&bv->nodes[0], p);
        while (sp) {
            const int32_t id = stack[--sp];
            /* conservative prune: box distance is a lower bound up to fp32
             * rounding; the (1 - 1e-5) factor keeps it strictly safe */
            if (sd[sp] * (1.f - 1e-5f) > best) continue;
            const bnode *n = &bv->nodes[id];
            if (n->left < 0) {
                for (int32_t k = n->start; k < n->start + n->count; ++k) {
                    const float *t9 = bv->tri + 9 * (int64_t)k;
                    const v3 q = closest_pt_triangle(p, ldv(t9), ldv(t9 + 3), ldv(t9 + 6));
                    const v3 g = v3sub(q, p);
                    const float d2 = v3dot(g, g);
                    const int32_t f = bv->order[k];
                    if (d2 < best || (d2 == best && f < bf)) { best = d2; bf = f; bc = q; }
                }
            } else {
                const float dl = box_dist2(&bv->nodes[n->left], p);
                const float dr = box_dist2(&bv->nodes[n->right], p);
                if (dl < dr) {
                    stack[sp] = n->right; sd[sp++] = dr;
                    stack[sp] = n->left; sd[sp++] = dl;
                } else {
                    stack[sp] = n->left; sd[sp++] = dl;
                    stack[sp] = n->right; sd[sp++] = dr;
                }
            }
        }
        out_closest[3 * i] = bc.x; out_closest[3 * i + 1] = bc.y; out_closest[3 * i + 2] = bc.z;
        out_dist2[i] = best; out_face[i] = bf;
    }
}

static inline int ray_box(const bnode *n, const double o[3], const double inv[3])
{
    double t0 = 0.0, t1 = INFINITY;
    for (int k = 0; k < 3; ++k) {
        /* boxes padded by a relative epsilon so that fp64 slabs on fp32 boxes
         * never cull a triangle the exact test would count */
        const double pad = 1e-6 * (fabs((double)n->lo[k]) + fabs((double)n->hi[k]) + 1e-3);
        double a = ((double)n->lo[k] - pad - o[k]) * inv[k];
        double b = ((double)n->hi[k] + pad - o[k]) * inv[k];
        if (a > b) { const double s = a; a = b; b = s; }
        if (a > t0) t0 = a;
        if (b < t1) t1 = b;
        if (t0 > t1) return 0;
    }
    return 1;
}

void orc_count_intersections_bvh(const void *h, const float *rays, int64_t N, int32_t *out_count)
{
    const obvh *bv = (const obvh *)h;
#pragma omp parallel for schedule(dynamic, 1024)
    for (int64_t i = 0; i < N; ++i) {
        const double o[3] = {rays[6 * i], rays[6 * i + 1], rays[6 * i + 2]};
        const double d[3] = {rays[6 * i + 3], rays[6 * i + 4], rays[6 * i + 5]};
        double inv[3];
        for (int k = 0; k < 3; ++k) inv[k] = 1.0 / (d[k] == 0.0 ? 1e-300 : d[k]);
        int32_t cnt = 0;
        int32_t stack[128]; int sp = 0;
        stack[sp++] = 0;
        while (sp) {
            const bnode *n = &bv->nodes[stack[--sp]];
            if (!ray_box(n, o, inv)) continue;
            if (n->left < 0) {
                for (int32_t k = n->start; k < n->start + n->count; ++k) {
                    const float *t9 = bv->tri + 9 * (int64_t)k;
                    cnt += ray_hits_triangle(o, d, ldv(t9), ldv(t9 + 3), ldv(t9 + 6));
                }
            } else {
                stack[sp++] = n->left;
                stack[sp++] = n->right;
            }
        }
        out_count[i] = cnt;
    }
}

/* Threads used by the parallel loops from now on (no-op without OpenMP or for n < 1). */
void orc_set_num_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
