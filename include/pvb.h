/*
 * pvb.h -- C ABI of libpvb.so, the H100 (sm_90a) signed-distance query library.
 *
 * The reference (UM-ARM-Lab/pytorch_volumetric) is pure Python and has no FFI
 * of its own; each entry point below replaces the body of one reference
 * operator (file:line in the reference repository) and is what a binding for that
 * operator would call.  See INTEGRATION.md for the ctypes stub a maintainer
 * would add on the reference side.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary
 *   - every "const float* pts" style argument below is a DEVICE pointer unless
 *     its comment says HOST; descriptors (pvb_sdf_desc) are HOST structs that
 *     hold device pointers
 *   - all launches go to the caller's stream (`stream` is a cudaStream_t
 *     passed as void*; NULL = legacy default stream); no allocation and no
 *     synchronisation inside query calls
 *   - fp32, C-contiguous; points are [n,3] AoS exactly as torch stores them
 *   - return value: 0 on success, negative pvb_status otherwise, with a
 *     thread-local message behind pvb_last_error()
 */
#ifndef PVB_H
#define PVB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PVB_VERSION 100

typedef enum pvb_status {
    PVB_OK = 0,
    PVB_ERR_INVALID = -1,   /* bad argument */
    PVB_ERR_CUDA = -2,      /* a CUDA runtime call or launch failed */
    PVB_ERR_CAPACITY = -3   /* caller-provided buffer too small */
} pvb_status;

/* sub-SDF kinds understood by the fused kernels.  BOX and CYLINDER are an EXTENSION (not reference behaviour): the
 * analytic URDF primitives, exact Euclidean SDFs centred at the origin (pvb_device.cuh box_eval / cylinder_eval).
 * Honoured by pvb_composed_query, _paired, _multi, _multicast (where the point-serial robot kernel runs, see
 * PVB_GRID_TRILINEAR) and pvb_chamfer.  Every entry point taking descriptors refuses a kind outside 0..4. */
enum { PVB_KIND_GRID = 0, PVB_KIND_MESH = 1, PVB_KIND_SPHERE = 2, PVB_KIND_BOX = 3, PVB_KIND_CYLINDER = 4 };

/* pvb_sdf_desc.flags */
enum {
    PVB_GRID_INDEX_FP32 = 1u << 0, /* voxel index arithmetic in fp32 (range given as Python floats);
                                      default is fp64, the dtype torch infers for numpy ranges */
    PVB_GRID_OOB_GT     = 1u << 1, /* OutOfBoundsStrategy.LOOKUP_GT_SDF: out-of-range points take the
                                      mesh query (mesh fields must be filled); default BOUNDING_BOX */
    PVB_GRID_PRUNE_OK   = 1u << 2, /* table verified to satisfy val >= dist(voxel centre, bb) - prune_margin:
                                      composed kernels may skip lookups that provably cannot win the min.  On
                                      SPHERE / BOX / CYLINDER: the same bound holds for the primitive and its
                                      bb_min / bb_max (prune_margin = inradius + fp32 slack) */
    PVB_GRID_TRILINEAR  = 1u << 4, /* EXTENSION (not reference behaviour): value = trilinear interpolation of the
                                      8 surrounding voxel values, gradient = analytic gradient of that interpolant
                                      (cell-wise finite differences).  Honoured by pvb_grid_lookup,
                                      pvb_composed_query, pvb_composed_query_multi and (where the point-serial
                                      robot kernel runs: <= 8 GRID or primitive sub-SDFs, >= PVB_ROBOT_MIN_CFG
                                      configurations)
                                      pvb_composed_query_multicast; needs the bounding-box rule (not
                                      PVB_GRID_OOB_GT).  pvb_chamfer rejects it (PVB_ERR_INVALID). */
    PVB_MESH_CLOSED     = 1u << 3  /* every directed edge is matched by its reverse (closed, consistently oriented
                                      surface): crossing parity is direction independent, so the sign test may use
                                      the exact axis-aligned walk instead of the reference's diagonal ray */
};

/* pvb_mesh_query mode flags */
enum {
    PVB_MESH_SIGNED         = 1u << 0, /* ray-parity inside test + sign (sdf.py:146-157) */
    PVB_MESH_SURFACE_NORMAL = 1u << 1, /* |d| < 1e-3 -> gradient = face normal (sdf.py:162-164) */
    PVB_MESH_DEFAULT        = 3u,
    PVB_MESH_WINDING        = 1u << 2  /* EXTENSION (not reference behaviour): with PVB_MESH_SIGNED, inside/outside from
                                          the generalized winding number |w| > 1/2 (hierarchical first-order evaluation,
                                          Barill et al. 2018) instead of crossing parity -- robust on open / self-
                                          intersecting meshes; needs pvb_sdf_desc.wn_nodes */
};

/*
 * One queryable object.  240 bytes (pvb_sizeof_sdf_desc()), POD, host-resident (device pointers
 * inside); the composed kernels take a host array of these by value.
 *
 * GRID part  = CachedSDF state (sdf.py:521-525): interleaved table
 *              {val, gx, gy, gz} per voxel in C order (last axis fastest),
 *              grid geometry, the mesh AABB used by the BOUNDING_BOX
 *              out-of-range rule (sdf.py:555-571).
 * MESH part  = ObjectFactory state (sdf.py:115-120): BVH4 nodes + leaf-ordered
 *              triangles from pvb_bvh_build, fp32 face normals in ORIGINAL
 *              face order, ray "destination" bbox(padding=1.0).max (sdf.py:147).
 * SPHERE     = SphereSDF radius (sdf.py:285-299); bb_min / bb_max = -/+radius.
 * BOX        = EXTENSION: half extents h in bb_max, bb_min = -h.
 * CYLINDER   = EXTENSION: axis along z, radius in `radius`, bb_min / bb_max = (-r, -r, -h) / (r, r, h) with h the
 *              half length.
 * Primitives set PVB_GRID_PRUNE_OK with prune_margin = inradius (sphere r, box min h, cylinder min(r, h)) + slack.
 */
typedef struct pvb_sdf_desc {
    int32_t kind;
    uint32_t flags;
    /* ---- grid ---- */
    const void *table;          /* device float4[n0*n1*n2] */
    int32_t dims[3];
    int32_t _pad0;
    double min64[3];            /* fp64 index mode: round((double(p) - min64) / res64) */
    double res64[3];
    float min32[3];             /* fp32 index mode: rintf((p - min32) / res32) */
    float res32[3];
    float valid_lo[3];          /* inclusive fp32 bounds equivalent to all(min <= p <= max) */
    float valid_hi[3];
    float bb_min[3];            /* surface AABB, fp32 (primitives: their box, see above) */
    float bb_max[3];
    float prune_margin;         /* see PVB_GRID_PRUNE_OK */
    /* ---- mesh ---- */
    int32_t n_nodes;
    const void *nodes;          /* device pvb_bvh4_node[n_nodes] */
    const void *tris;           /* device float4[3*n_tris] */
    const float *face_normals;  /* device float[3*n_tris], original face order */
    int32_t n_tris;
    float ray_far[3];
    uint32_t ray_seed;          /* seed of the deterministic stand-in for sdf.py:149's jitter */
    /* ---- sphere, cylinder ---- */
    float radius;
    /* ---- grid: fast index path ----
     * k = rintf((p - min32) * inv_res32) is taken as the voxel index when |q - k| <= idx_certain (the fp32
     * estimate provably rounds the same way as the exact formula); otherwise the exact formula above runs. */
    float inv_res32[3];
    float idx_certain[3];
    /* ---- mesh: winding-number extension ----
     * device float4[8 * n_nodes]: per node, for each of the 4 children {area-weighted centroid xyz, bounding
     * radius} then {sum of area vectors xyz, 0}; NULL unless PVB_MESH_WINDING is used */
    const void *wn_nodes;
} pvb_sdf_desc;

/* BVH4 node, 128 bytes: SoA child boxes + child links.
 * child >= 0: inner node index; child < 0 and != INT32_MIN: leaf, ~child =
 * (first_triangle << 2) | (count - 1), count in 1..4; INT32_MIN: empty slot. */
typedef struct pvb_bvh4_node {
    float lox[4], loy[4], loz[4];
    float hix[4], hiy[4], hiz[4];
    int32_t child[4];
    int32_t _pad[4];
} pvb_bvh4_node;

const char *pvb_last_error(void);
int pvb_version(void);
/* sizeof the structs above as compiled, so a binding can verify its mirror */
int pvb_sizeof_sdf_desc(void);
int pvb_sizeof_bvh4_node(void);

/* ---- measurement hook (bench.py's roofline; no reference counterpart) ----
 * pvb_timing_enable(1): every query entry point below brackets its DOMINANT kernel launch (the tree walk, the
 * lookup, the composed kernel, the chamfer partial sums) with a pair of CUDA events on the caller's stream.
 * pvb_timing_last_ms waits for the stop event of the most recent such launch on the current device and returns
 * that one launch's device time.  Off by default. */
int pvb_timing_enable(int on);
int pvb_timing_last_ms(float *ms_out /* HOST */);

/* ---- mesh preprocessing (HOST -> HOST), replaces RaycastingScene construction, sdf.py:115-118 ---- */
int64_t pvb_bvh_max_nodes(int64_t n_faces);
/* verts HOST float[n_verts*3], faces HOST int32[n_faces*3];
 * nodes_out HOST pvb_bvh4_node[node_capacity]; tris_out HOST float[n_faces*12]
 * (3 x {x,y,z,w}; w of vertex 0 carries the original face index as int bits). */
int pvb_bvh_build(const float *verts, int64_t n_verts, const int32_t *faces, int64_t n_faces,
                  void *nodes_out, int64_t node_capacity, float *tris_out,
                  int64_t *n_nodes_out, int32_t *max_depth_out);

/* ---- ObjectFactory._do_object_frame_closest_point, sdf.py:122-172 (MeshSDF.__call__, sdf.py:312-329) ----
 * out_dist[n], out_grad[n*3] required; out_closest[n*3], out_face[n] (int32, original index),
 * out_normal[n*3] optional (NULL to skip). */
int pvb_mesh_query(const pvb_sdf_desc *mesh, const float *pts, int64_t n, uint32_t mode,
                   float *out_dist, float *out_grad, float *out_closest, int32_t *out_face,
                   float *out_normal, void *workspace, int64_t workspace_bytes, void *stream);
/* Optional DEVICE scratch for the tree-walk kernels (pvb_mesh_query, pvb_chamfer): with at least
 * pvb_query_workspace(n) bytes, large batches are spatially binned (counting sort into Morton cells) and walked
 * in that order, which keeps warps coherent; results land in the original slots.  0 / NULL (or a pointer that is
 * not 16-byte aligned) = walk in input order. */
int64_t pvb_query_workspace(int64_t n);

/* ---- CachedSDF.__call__ (sdf.py:535-571) and outside_surface (sdf.py:593-602) ----
 * out_val / out_grad may be NULL when only occupancy is wanted; out_outside (uint8, 0/1)
 * may be NULL; out_index (int64 ravelled key, -1 if out of range) may be NULL. */
int pvb_grid_lookup(const pvb_sdf_desc *grid, const float *pts, int64_t n,
                    float *out_val, float *out_grad, uint8_t *out_outside, float surface_level,
                    int64_t *out_index, void *stream);

/* ---- SphereSDF.__call__, sdf.py:291-295 ---- */
int pvb_sphere_query(float radius, const float *pts, int64_t n, float *out_val, float *out_grad, void *stream);

/* ---- ComposedSDF.__call__ / RobotSDF.__call__ (sdf.py:392-433, model_to_sdf.py:117-125) ----
 * descs: HOST array of n_sdf (<= 128) pvb_sdf_desc, passed to the kernel by value (constant bank); xforms: DEVICE float[n_sdf*n_cfg][16] object->sub-frame
 * 4x4 row-major, sub-SDF-major (sdf.py:385-390).  The winning gradient is mapped back with
 * g_obj = g_link @ M[:3,:3]: the reference's link_frame_to_obj_frame[i].transform_normals
 * (sdf.py:380-383, 409) is g @ inv(inv(M)[:3,:3]), and the two inversions cancel;
 * pts DEVICE [n_pts,3]; out_val [n_cfg*n_pts], out_grad [n_cfg*n_pts*3]; out_which optional
 * int32 argmin index.  cfg_begin/cfg_count select a contiguous slab of configurations (multi-GPU
 * sharding); outputs are indexed relative to cfg_begin.  needs_mesh != 0 when any descriptor is a MESH or a
 * GRID with PVB_GRID_OOB_GT (selects the instantiation that contains the tree walk). */
int pvb_composed_query(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                       int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                       const float *pts, int64_t n_pts, uint32_t mesh_mode,
                       float *out_val, float *out_grad, int32_t *out_which, void *stream);

/* ---- EXTENSION: paired query, every configuration at its own points ----
 * The reference has no such operator; its equivalent is the diagonal of ComposedSDF.__call__ (sdf.py:392-433) over
 * points [|A|, n_pts, 3], which costs |A| times the work and memory.  Configuration cfg_begin + c is evaluated at
 * pts[c][0 .. n_pts) only: pts DEVICE [cfg_count][n_pts][3], out_val [cfg_count * n_pts], out_grad
 * [cfg_count * n_pts * 3], out_which optional; everything else as pvb_composed_query.  Results are bit-identical to
 * pvb_composed_query(pts + 3 * c * n_pts, n_pts, cfg_begin + c, cfg_count = 1) for every c, including the mesh ray
 * jitter (seeded by the absolute configuration index), and so, for GRID and SPHERE sets, to the diagonal of the cross
 * product.  PVB_ERR_INVALID also when cfg_count * n_pts overflows int64_t. */
int pvb_composed_query_paired(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                              int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                              const float *pts, int64_t n_pts, uint32_t mesh_mode,
                              float *out_val, float *out_grad, int32_t *out_which, void *stream);

/* ---- EXTENSION: swept query, the minimum over the configurations at every point ----
 * The reference has no such operator; its equivalent is the minimum over dim 0 of ComposedSDF.__call__'s result
 * (sdf.py:392-433), which materialises 16 * cfg_count * n_pts bytes.  For point i, the result is the
 * per-configuration result (pvb_composed_query: value, gradient, which) of the configuration c* that minimises
 * (value, c, which) lexicographically over [cfg_begin, cfg_begin + cfg_count): the FIRST configuration attaining the
 * minimum value.  Bit-identical to that reduction of pvb_composed_query's results, for every set it accepts.
 * out_val [n_pts], out_grad [n_pts * 3]; out_cfg [n_pts] (the absolute configuration index c*) and out_which [n_pts]
 * (the sub-SDF index) are optional; everything else as pvb_composed_query.  PVB_ERR_INVALID also when cfg_count < 1
 * and n_pts > 0: there is no minimum over an empty set.  n_pts == 0 does nothing. */
int pvb_composed_query_swept(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                             int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                             const float *pts, int64_t n_pts, uint32_t mesh_mode,
                             float *out_val, float *out_grad, int32_t *out_cfg, int32_t *out_which, void *stream);

/* ---- EXTENSION: clearance query, the minimum over the points of a segment for every configuration ----
 * The reference has no such operator; its equivalent is the minimum over the point dimension of ComposedSDF.__call__'s
 * result (sdf.py:392-433), which materialises 16 * cfg_count * n_seg * seg_len bytes.  pts DEVICE [n_seg][seg_len][3]:
 * segment b is pts[b].  For configuration cfg_begin + c and segment b, the result is the per-configuration result
 * (pvb_composed_query: value, gradient, which) at the point i* of the segment that minimises (value, i)
 * lexicographically: the FIRST point of the segment attaining the minimum value.  -0 and +0 compare equal; a NaN value
 * ranks above every number (+inf included), so i* is a NaN point only when every point of the segment is NaN, and then
 * the first one.  Bit-identical to that reduction of pvb_composed_query's results over the flat points, for every set
 * it accepts.
 * keys DEVICE scratch of cfg_count * n_seg entries (the library initialises it).  out_val [cfg_count * n_seg],
 * out_grad [cfg_count * n_seg * 3], configuration-major (entry c * n_seg + b); out_point (i*, the index within the
 * segment) and out_which (the sub-SDF index) are optional; everything else as pvb_composed_query.  PVB_ERR_INVALID also
 * when seg_len == 0 with cfg_count >= 1 and n_seg >= 1 (no minimum over an empty segment), when cfg_count < 1 with
 * points, and when seg_len >= 2^31.  n_seg == 0 does nothing. */
int pvb_composed_query_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                                 int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                 const float *pts, int64_t n_seg, int64_t seg_len, uint32_t mesh_mode,
                                 uint64_t *keys, float *out_val, float *out_grad,
                                 int32_t *out_point, int32_t *out_which, void *stream);

/* ---- EXTENSION: paired clearance query, every configuration against its own points ----
 * The reference has no such operator; its equivalent is the per-configuration clearance over each configuration's own
 * cloud, pvb_composed_query_clearance(pts[c], cfg_begin + c, 1) for every c.  pts DEVICE [cfg_count][n_seg][seg_len][3]:
 * segment b of configuration cfg_begin + c is pts[c][b].  Entry c * n_seg + b of every output is bit-identical to entry
 * b of that per-configuration call (value, gradient, point i* within the segment, sub-SDF), mesh ray jitter included:
 * the jitter index of pts[c][b][i] is (cfg_begin + c) * n_seg * seg_len + b * seg_len + i, as in the paired and the
 * per-configuration query.  Equivalently, the first-point (value, i) minimum of pvb_composed_query_paired's results over
 * each segment; -0 == +0 and a NaN value ranks above every number, as in pvb_composed_query_clearance.
 * Arguments and refusals are those of pvb_composed_query_clearance (keys: device scratch of cfg_count * n_seg entries
 * that the library initialises), plus PVB_ERR_INVALID when cfg_count * n_seg * seg_len overflows int64. */
int pvb_composed_query_paired_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh,
                                        const float *xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                        const float *pts, int64_t n_seg, int64_t seg_len, uint32_t mesh_mode,
                                        uint64_t *keys, float *out_val, float *out_grad,
                                        int32_t *out_point, int32_t *out_which, void *stream);

/* ---- EXTENSION: self-clearance query, every configuration's smallest distance between its own sub-SDFs ----
 * The reference has no such operator.  M_s(a) = xforms[s * n_cfg + a] (object -> sub-frame, as every composed query
 * reads it) and W_s(a) = inv_xforms[s * n_cfg + a], the same layout (sub-frame -> object frame; the caller computes
 * it, ComposedSDF caches _affine_inverse(M)).  link_pts DEVICE [n_sdf][K][3]: K points of every sub-SDF in its own
 * frame.  allowed HOST uint8_t[n_sdf]: bit j of row i lets the points of i be tested against sub-SDF j; the diagonal
 * is ignored.  For configuration cfg_begin + c: over every i, every allowed j and every k, the minimum of
 * sdf_j(M_j(a) x) with x = W_i(a) link_pts[i][k] posed by the arithmetic of pvb_transform_points_paired.  The minimum
 * is taken over (value, i, k) lexicographically; for that point the first allowed j attaining the value wins (the
 * composition's first-index rule); -0 == +0 and a NaN value ranks above every number, as in
 * pvb_composed_query_clearance.  out_val [cfg_count], out_grad [cfg_count * 3] (the object-frame gradient
 * pvb_composed_query_paired of the allowed sub-composition reports at x); optional out_src (i), out_point (k),
 * out_which (j).  A configuration without an allowed pair gets +inf, a zero gradient and indices -1.  Bit-identical to
 * the composition route: per source i, its points posed by pvb_transform_points_paired with W_i, then
 * pvb_composed_query_paired_clearance on the allowed sub-SDFs and their transform rows, reduced over i by (value, i).
 * keys: device scratch of cfg_count entries that the library initialises.
 * Serves the sets pvb_composed_query_paired_clearance runs fused: at most 8 GRID sub-SDFs with the bounding-box rule
 * (nearest or trilinear) or primitives.  PVB_ERR_INVALID for every other set (mesh, LOOKUP_GT_SDF grids, more than 8
 * sub-SDFs: callers compose the route above), for K < 1 or K >= 2^24, bits of allowed beyond n_sdf, cfg_count < 1,
 * null inv_xforms, allowed or keys, and the argument checks of pvb_composed_query. */
int pvb_composed_query_self_clearance(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                      const float *inv_xforms, int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                      const float *link_pts, int64_t K, const uint8_t *allowed, uint64_t *keys,
                                      float *out_val, float *out_grad, int32_t *out_src, int32_t *out_point,
                                      int32_t *out_which, void *stream);

/* ---- EXTENSION: collision-cost query, a hinge cost over a cloud and its twist gradient for every configuration ----
 * The reference has no such operator.  pts DEVICE [n_seg][seg_len][3] (object frame): segment b is pts[b].  For
 * configuration a = cfg_begin + c, segment b and margin m, with (d, g, s) the per-configuration result of
 * pvb_composed_query at point p (value, object-frame gradient, first sub-SDF attaining the value):
 *   out_cost[c * n_seg + b]                 = sum over p of max(0, m - d)^2   (0 for an empty segment)
 *   out_twist[((c * n_seg + b) * n_sdf + s) * 6 + k], k = 0..5
 *                                            = sum over the p with argmin s and d < m of 2 (m - d) (g, p x g),
 * the derivative of the cost when sub-SDF s alone moves by an object-frame twist (v, w) about the origin (its material
 * points moving at v + w x p).  Every (d, g, s) that enters a sum is bit-identical to pvb_composed_query's; a pair is
 * skipped only when a lower bound of its value is >= m.  The sums are deterministic: no atomics, and the order of every
 * (configuration, segment) sum depends on seg_len alone (pvb_device.cuh collision_cost_chunk), so a slab reproduces
 * the rows of a larger call bit for bit; they are not bit-identical to a composition of pvb_composed_query.
 * workspace DEVICE, at least pvb_collision_cost_workspace(n_sdf, cfg_count, n_seg, seg_len) bytes, 4-byte aligned
 * (may be NULL when that is 0); pvb_collision_cost_workspace returns -1 for negative sizes or an overflow.
 * Serves the sets pvb_composed_query_self_clearance serves: at most 8 GRID sub-SDFs with the bounding-box rule
 * (nearest or trilinear) or primitives.  PVB_ERR_INVALID for every other set (mesh, LOOKUP_GT_SDF grids, more than 8
 * sub-SDFs: callers compose pvb_composed_query), for a margin that is not finite, cfg_count < 1 with points,
 * seg_len >= 2^31, a workspace that is too small, null outputs with segments and configurations, and the argument
 * checks of pvb_composed_query.  n_seg == 0 does nothing. */
int64_t pvb_collision_cost_workspace(int32_t n_sdf, int32_t cfg_count, int64_t n_seg, int64_t seg_len);
int pvb_composed_query_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms, int32_t n_cfg,
                                      int32_t cfg_begin, int32_t cfg_count, const float *pts, int64_t n_seg,
                                      int64_t seg_len, float margin, void *workspace, int64_t workspace_bytes,
                                      float *out_cost, float *out_twist, void *stream);

/* ---- EXTENSION: paired collision-cost query, each configuration's hinge cost over its OWN cloud ----
 * The reference has no such operator.  pts DEVICE [cfg_count][n_seg][seg_len][3] (object frame): configuration
 * cfg_begin + c is evaluated at pts[c] only.  Row c * n_seg + b of out_cost and out_twist (layouts of
 * pvb_composed_query_collision_cost) is pvb_composed_query_collision_cost of configuration cfg_begin + c alone
 * (cfg_count = 1) over pts[c], segment b, bit for bit: the same (d, g, s) per point -- pvb_composed_query_paired's --,
 * the same terms and the same summation order, which depends on seg_len alone (pvb_device.cuh collision_cost_chunk).
 * So the sums are deterministic, repeated calls give identical bits and a slab reproduces the rows of a larger call.
 * workspace DEVICE, at least pvb_collision_cost_workspace(n_sdf, cfg_count, n_seg, seg_len) bytes, 4-byte aligned
 * (may be NULL when that is 0).  Serves the sets pvb_composed_query_collision_cost serves: at most 8 GRID sub-SDFs with
 * the bounding-box rule (nearest or trilinear) or primitives.  PVB_ERR_INVALID for every other set (mesh, LOOKUP_GT_SDF
 * grids, more than 8 sub-SDFs: callers compose pvb_composed_query_paired), for a margin that is not finite,
 * cfg_count < 1 with points, seg_len >= 2^31, cfg_count * n_seg * seg_len overflowing int64, a workspace that is too
 * small, null outputs with segments and configurations, and the argument checks of pvb_composed_query.  n_seg == 0
 * does nothing. */
int pvb_composed_query_paired_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                             int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count, const float *pts,
                                             int64_t n_seg, int64_t seg_len, float margin, void *workspace,
                                             int64_t workspace_bytes, float *out_cost, float *out_twist,
                                             void *stream);

/* ---- EXTENSION: self-collision-cost query, a hinge cost between every configuration's own links and its twists ----
 * The reference has no such operator.  xforms, inv_xforms, link_pts and allowed as in
 * pvb_composed_query_self_clearance.  The definition:
 *   Inputs: a composition of S sub-SDFs with transforms M_s(a), and W_s = _affine_inverse(M_s); link_points [S, K, 3],
 *   each row in its own sub-SDF's frame; allowed [S, S] bool (the diagonal is ignored); a margin m, rounded to fp32
 *   exactly as _collision_cost_margin does.
 *   For configuration a, every source i and every point k:
 *   - x = W_i(a) . link_points[i, k], posed with composed_xform.  This is the same posed point as in
 *     pvb_transform_points_paired and self_clearance.
 *   - (d, g, j) is what query_paired(..., return_which=True) of the composition of row i's allowed sub-SDFs gives at x:
 *     the value, the object-frame gradient, and the first allowed sub-SDF attaining the value.  These are the
 *     per-point values _composed_self_clearance already uses.
 *   - When d < m, with h = m - d and tau = 2h (g, x x g):
 *     - cost[a] += h^2
 *     - twist[a, j] += tau.  The target moves.  This is the same term and sign as collision_cost_term.
 *     - twist[a, i] -= tau.  The source moves.  Its point travels with it, so d changes by +g . (v + w x x).
 *   - twist[a, s] is therefore the derivative of the cost when sub-SDF s alone moves by an object-frame twist (v, w)
 *     about the origin.  This is the convention of collision_cost, so RobotSDF.joint_gradient applies unchanged.
 *   - A configuration with no allowed pair, or with no point below m, costs exactly 0 and has all-zero twists.
 * out_cost [cfg_count] and out_twist [cfg_count * n_sdf * 6] (k = 0..5 of sub-SDF s at (c * n_sdf + s) * 6 + k) for
 * configuration cfg_begin + c.  Every (d, g, j) that enters a sum is bit-identical to the per-point query's; a pair is
 * skipped only when a lower bound of its value is >= m.  The sums are deterministic: no atomics, and their order
 * depends on K, n_sdf and allowed alone (pvb_device.cuh), so repeated calls give identical bits and a slab reproduces
 * the rows of a larger call; they are not bit-identical to a composition of per-source queries.  No workspace.
 * Serves the sets pvb_composed_query_self_clearance serves: at most 8 GRID sub-SDFs with the bounding-box rule
 * (nearest or trilinear) or primitives.  PVB_ERR_INVALID for every other set (mesh, LOOKUP_GT_SDF grids, more than 8
 * sub-SDFs: callers compose the per-source paired queries), for K < 1 or K >= 2^24, bits of allowed beyond n_sdf, a
 * margin that is not finite, cfg_count < 1, null inv_xforms, allowed or outputs, and the argument checks of
 * pvb_composed_query. */
int pvb_composed_query_self_collision_cost(const pvb_sdf_desc *descs, int32_t n_sdf, const float *xforms,
                                           const float *inv_xforms, int32_t n_cfg, int32_t cfg_begin,
                                           int32_t cfg_count, const float *link_pts, int64_t K,
                                           const uint8_t *allowed, float margin, float *out_cost, float *out_twist,
                                           void *stream);

/* ---- EXTENSION: scene queries, every configuration's link points against one static scene SDF ----
 * The reference has no such operator.  The robot: a composition of n_sdf <= 255 sub-SDFs whose inverse transforms
 * W_s(a) = _affine_inverse(M_s(a)) are inv_xforms [n_sdf][n_cfg][4][4] (device); link_pts [n_sdf][K][3] (device), each
 * row in its own sub-SDF's frame, 1 <= K < 2^24; links [n_sdf] (HOST memory), nonzero for the sources tested.  The
 * robot's own sub-SDFs are never evaluated, so they may be of any kind.  The scene: n_scene <= 128 descriptors (host
 * array, device tables) with their one configuration of object->sub-frame transforms scene_xforms [n_scene][4][4]
 * (device), in the robot's object frame; a bare SDF is one descriptor under the identity.  For configuration a, every
 * tested source i and point k: x = W_i(a) . link_pts[i][k] (posed as pvb_transform_points_paired poses), and (d, g)
 * the scene's value and object-frame gradient at x, evaluated with the scene composition's one-point sequence
 * (pvb_composed_query at x gives the same bits).
 * Clearance: out_val / out_grad [cfg_count] / [cfg_count * 3] hold the minimum over (d, i, k) lexicographically (-0 ==
 * +0, NaN above every number) and its gradient; out_link / out_point (each may be null) its i and k.  A configuration
 * without a tested source gets +inf, a zero gradient and -1, -1.
 * Collision cost with margin m: when d < m, h = m - d and tau = 2h (g, x x g): cost[a] += h^2 and twist[a, i] -= tau
 * (the source moves, its point with it; the static scene takes no term).  out_cost [cfg_count], out_twist
 * [cfg_count * n_sdf * 6] (k = 0..5 of source s at (c * n_sdf + s) * 6 + k); a configuration with nothing inside the
 * margin costs exactly 0, and every untested source's row is 0.  The sums are deterministic, without atomics or
 * workspace; their order depends on K, n_sdf and links alone (pvb_device.cuh), so a slab reproduces the rows of a
 * larger call bit for bit.
 * Both serve scenes of GRID sub-SDFs with the bounding-box rule (nearest or trilinear) and primitives.
 * PVB_ERR_INVALID for mesh or LOOKUP_GT_SDF scene sub-SDFs (callers query the scene at the posed points), more than
 * 128 scene or 255 robot sub-SDFs, K < 1 or K >= 2^24, null inv_xforms, links or outputs, an empty or invalid slab,
 * a margin that is not finite, and the descriptor checks of pvb_composed_query. */
int pvb_composed_query_scene_clearance(const pvb_sdf_desc *scene, int32_t n_scene, const float *scene_xforms,
                                       const float *inv_xforms, int32_t n_sdf, int32_t n_cfg, int32_t cfg_begin,
                                       int32_t cfg_count, const float *link_pts, int64_t K, const uint8_t *links,
                                       float *out_val, float *out_grad, int32_t *out_link, int32_t *out_point,
                                       void *stream);
int pvb_composed_query_scene_collision_cost(const pvb_sdf_desc *scene, int32_t n_scene, const float *scene_xforms,
                                            const float *inv_xforms, int32_t n_sdf, int32_t n_cfg, int32_t cfg_begin,
                                            int32_t cfg_count, const float *link_pts, int64_t K, const uint8_t *links,
                                            float margin, float *out_cost, float *out_twist, void *stream);

/* ---- the same query with the result slab stored to several destinations from the kernel epilogue ----
 * Multi-GPU re-assembly of a configuration-sharded RobotSDF result (model_to_sdf.py:117-125 returns the full
 * (|A|, N) tensors): every rank evaluates its slab [cfg_begin, cfg_begin + cfg_count) and writes it straight into
 * the full-size result buffer of every rank -- its own and the peer-mapped ones (pvb_ipc_open) -- so the NVLink
 * traffic overlaps the lookups instead of following them as a separate all-gather.
 * targets: HOST array of n_targets (1..PVB_MAX_TARGETS) DEVICE pointer pairs, each already advanced to the slab
 * (element cfg_begin * n_pts of that rank's full buffer); target 0 conventionally is the local buffer.  The caller
 * orders the launch after the peers' previous readers and publishes completion (stream-ordered collective or
 * event) before anyone reads. */
#define PVB_MAX_TARGETS 8
typedef struct pvb_out_target {
    float *val;  /* [cfg_count * n_pts]     */
    float *grad; /* [cfg_count * n_pts * 3] */
} pvb_out_target;
int pvb_composed_query_multi(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                             int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                             const float *pts, int64_t n_pts, uint32_t mesh_mode,
                             const pvb_out_target *targets, int32_t n_targets, int32_t *out_which, void *stream);

/* ---- the same, stored through an NVLS MULTICAST mapping ----
 * mc_val / mc_grad are multicast addresses (cuMulticast* / torch symmetric memory) of the full-size result buffers,
 * already advanced to the slab: the kernel epilogue issues one multimem.st per 16-byte chunk and the NVSwitch
 * replicates it into every bound GPU's buffer (the sender emits each byte once instead of once per peer).  Needs
 * <= 16 GRID sub-SDFs with the bounding-box out-of-range rule (a RobotSDF of cached links); sets with trilinear or
 * primitive sub-SDFs only where the point-serial robot kernel runs (<= 8 sub-SDFs, >= PVB_ROBOT_MIN_CFG configurations). */
int pvb_composed_query_multicast(const pvb_sdf_desc *descs, int32_t n_sdf, int32_t needs_mesh, const float *xforms,
                                 int32_t n_cfg, int32_t cfg_begin, int32_t cfg_count,
                                 const float *pts, int64_t n_pts, uint32_t mesh_mode,
                                 float *mc_val, float *mc_grad, void *stream);

/* ---- RobotSDF.set_joint_configuration, model_to_sdf.py:82-115 (forward kinematics of a serial chain) ----
 * For every configuration a and mesh link s: out[(slot_s * n_cfg + a)] = mesh_from_link_s @ inverse(FK_frame(s)(q_a)),
 * the 4x4 row-major object->mesh-frame matrix pvb_composed_query reads (sub-SDF-major).  FK: T_f = T_{f-1} @ origin_f
 * @ motion_f(q[q_index_f]); revolute = Rodrigues rotation about `axis` (unit), prismatic = translation along it.
 * frames / links: HOST arrays (passed to the kernel by value); links sorted by frame; q DEVICE float[n_cfg][n_joints];
 * out_xforms DEVICE float[n_links * n_cfg][16]. */
#define PVB_FK_MAX_FRAMES 32
#define PVB_FK_MAX_LINKS 16
enum { PVB_FK_FIXED = 0, PVB_FK_REVOLUTE = 1, PVB_FK_PRISMATIC = 2 };
typedef struct pvb_fk_frame {
    float origin[12];      /* joint origin in the parent frame, rows of [R | t] */
    float axis[3];
    int32_t joint_type;    /* PVB_FK_* */
    int32_t q_index;       /* column of q this joint reads (ignored for fixed joints) */
    int32_t _pad[3];
} pvb_fk_frame;
typedef struct pvb_fk_link {
    float mesh_from_link[12]; /* inverse of the visual offset (<visual><origin>), rows of [A | t] */
    int32_t frame;            /* frame whose pose carries this mesh */
    int32_t slot;             /* sub-SDF index s of the output */
    int32_t _pad[2];
} pvb_fk_link;
int pvb_fk_serial(const pvb_fk_frame *frames, int32_t n_frames, const pvb_fk_link *links, int32_t n_links,
                  const float *q, int32_t n_cfg, int32_t n_joints, float *out_xforms, void *stream);

/* ---- the same for a kinematic tree (kinematics.Chain) ----
 * T_f = T_{parents[f]} @ origin_f @ motion_f(q[q_index_f]), the root's parent pose the identity; the output layout,
 * the links and the rest of the arguments are those of pvb_fk_serial.  parents: HOST int32[n_frames] in depth-first
 * pre-order: parents[0] == -1, and for f > 0 parents[f] is f - 1 or an ancestor of f - 1.  pvb_fk_serial is this
 * walk with parents[f] = f - 1. */
#define PVB_FK_TREE_MAX_FRAMES 64
#define PVB_FK_TREE_MAX_LINKS 64
int pvb_fk_tree(const pvb_fk_frame *frames, const int32_t *parents, int32_t n_frames, const pvb_fk_link *links,
                int32_t n_links, const float *q, int32_t n_cfg, int32_t n_joints, float *out_xforms, void *stream);

/* ---- peer-visible device buffers (one process per GPU, same node) ----
 * pvb_ipc_alloc: cudaMalloc on the current device (IPC handles need a whole allocation, not a slice of a caching
 * allocator's segment); pvb_ipc_export fills a 64-byte handle another PROCESS passes to pvb_ipc_open to map the
 * buffer (peer access is enabled on first use).  pvb_ipc_close unmaps, pvb_ipc_free releases the allocation. */
#define PVB_IPC_HANDLE_BYTES 64
int pvb_ipc_alloc(int64_t bytes, void **out_ptr);
int pvb_ipc_free(void *ptr);
int pvb_ipc_export(void *ptr, unsigned char *handle /* [PVB_IPC_HANDLE_BYTES] */);
int pvb_ipc_open(const unsigned char *handle, void **out_ptr);
int pvb_ipc_close(void *ptr);
/* cudaMemcpyAsync between any two device pointers of the node (local or peer-mapped), on `stream`: the copy-engine
 * push of a finished result slab into the peers' buffers (sharded_robot_query(gather="dma")). */
int pvb_memcpy_async(void *dst, const void *src, int64_t bytes, void *stream);

/* ---- batch_chamfer_dist, chamfer.py:79-94 ----
 * world_to_object DEVICE float[n_tf][16]; pts DEVICE [n_pts,3] world frame;
 * workspace DEVICE float[n_tf * pvb_chamfer_workspace(n_pts)]; out DEVICE float[n_tf]
 * = mean_i (scale * d_i)^2 with d the unsigned distance to `obj` (mesh) or the value of
 * `obj` (grid / sphere). */
int64_t pvb_chamfer_workspace(int64_t n_pts);
int pvb_chamfer(const pvb_sdf_desc *obj, const float *world_to_object, int32_t n_tf,
                const float *pts, int64_t n_pts, float scale, float *workspace, float *out,
                void *sort_workspace, int64_t sort_workspace_bytes, void *stream);

/* ---- sample_mesh_points, sdf.py:650-658 (area-uniform surface samples) ----
 * verts64 DEVICE double[n_verts*3]; faces DEVICE int32[n_faces*3]; cum_counts DEVICE int64[n_faces]
 * inclusive cumulative sample count per face (stratified allocation);
 * out_pts DEVICE double[n*3]; out_face DEVICE int32[n]. */
int pvb_mesh_sample(const double *verts64, const int32_t *faces, int64_t n_faces, const int64_t *cum_counts,
                    int64_t n, uint64_t seed, double *out_pts, int32_t *out_face, void *stream);

/* ---- voxel containers: VoxelGrid / ExpandingVoxelGrid / voxel_down_sample (voxel.py:42-171) over the value-range
 * view TorchMultidimView (sdf.py:264; voxel.py:55-64, 88-91) ----
 * Grid geometry: d in 1..3 coordinates per point, per-axis min64 / res64 (HOST double[d]) and dims (HOST int32[d]);
 * fp32_mode != 0 evaluates the index in fp32 (ranges given as Python floats / float32 numpy), else in fp64 (float64
 * numpy ranges) -- the dtype torch infers for the range tensors.  Cell of a point: round((p - min) / res), half to even
 * like torch.round; valid when every index is in [0, dim).  Flat indices are C order (last axis fastest).
 *   pvb_voxel_index    out_index[n] int64 flat cell or -1                       (ensure_index_key + ravel_multi_index)
 *   pvb_voxel_scatter  data[cell(p_i)] = values[i] (values == NULL: `scalar`)   (view[pts] = value, voxel.py:90-91)
 *   pvb_voxel_gather   out[i] = data[cell(p_i)] or `invalid`; out_valid optional (view[pts], voxel.py:87-88)
 *   pvb_compact_nonempty  ascending flat indices of the cells with data != empty (get_known_pos_and_values,
 *                      voxel.py:59-65; the compaction behind voxel_down_sample, voxel.py:166-167); out_count DEVICE
 *                      int64[1] receives the number found (also when capacity is too small: call again);
 *                      workspace DEVICE, pvb_compact_workspace(n) bytes.
 * elem_bytes: 4 = float32 grid, 1 = bool / uint8 grid.  All pointers DEVICE unless marked HOST. */
int pvb_voxel_index(int32_t d, const double *min64, const double *res64, const int32_t *dims, int32_t fp32_mode,
                    const float *pts, int64_t n, int64_t *out_index, void *stream);
int pvb_voxel_scatter(int32_t d, const double *min64, const double *res64, const int32_t *dims, int32_t fp32_mode,
                      const float *pts, int64_t n, int32_t elem_bytes, const void *values, double scalar, void *data,
                      void *stream);
int pvb_voxel_gather(int32_t d, const double *min64, const double *res64, const int32_t *dims, int32_t fp32_mode,
                     const float *pts, int64_t n, int32_t elem_bytes, const void *data, double invalid, void *out,
                     uint8_t *out_valid, void *stream);
int64_t pvb_compact_workspace(int64_t n);
int pvb_compact_nonempty(const void *data, int64_t n, int32_t elem_bytes, double empty, void *workspace,
                         int64_t capacity, int64_t *out_index, int64_t *out_count, void *stream);

/* ---- occupancy distance transform: OccupancySDF (sdf.py) ----
 * occ DEVICE uint8 [nx][ny][nz] (C order, z fastest; nonzero = occupied), dims HOST int32[3] = {nx, ny, nz}, each
 * 2..1024.  For every voxel c: its site s(c), the voxel of the OTHER state (occupied for a free c, free for an occupied
 * c) at the smallest squared distance D(c) = |c - s|^2 in integer cell units, ties to the smallest flat C-order index
 * (exact: integer arithmetic throughout).  Outputs, each DEVICE and each optional (not all NULL):
 *   out_sqdist int32 [n_vox]  D(c)
 *   out_site   int32 [n_vox]  flat index of s(c)
 *   out_table  float [n_vox][4], 16-byte aligned: the CachedSDF record {val, gx, gy, gz} with sigma = +1 for a free
 *              voxel and -1 for an occupied one, r32 = resolution and q = sqrt_rn(float(D)), every operation rounded to
 *              nearest once: val = sigma (r32 * (q - 0.5)), g_k = sigma (float(c_k - s_k) / q).  The zero level lies
 *              on the faces between occupied and free voxels.
 * A grid without an occupied or without a free voxel has no field: D = -1, site = -1, val = sigma inf, gradient 0.
 * workspace DEVICE, pvb_occupancy_sdf_workspace(dims) bytes (48 per voxel), 8-byte aligned; nothing is allocated.
 * PVB_ERR_INVALID before any device work: dims outside 2..1024, a resolution that is not finite and positive, a
 * missing or short workspace, occ NULL, every output NULL.  pvb_occupancy_sdf_workspace returns -1 for such dims. */
int64_t pvb_occupancy_sdf_workspace(const int32_t *dims);
int pvb_occupancy_sdf(const uint8_t *occ, const int32_t *dims, float resolution, void *workspace,
                      int64_t workspace_bytes, int32_t *out_sqdist, int32_t *out_site, float *out_table, void *stream);

/* ---- depth images: depth_to_points, depth_occupancy, OccupancySDF.from_depth (sdf.py) ----
 * depth DEVICE float [V][H][W], z-depth in metres, row-major; V 1..64, H and W 1..32768.  A pixel is valid when its
 * depth d is finite, d > 0 and d <= max_depth (+inf allowed); any other pixel carries no information.
 * intrinsics HOST float [V][4] = {fx, fy, cx, cy}: fx, fy finite and positive, cx, cy finite.  The camera follows the
 * OpenCV convention (x right, y down, z forward); pixel (row i, column j) is centred at u = j, v = i.
 * cam_to_world / world_to_cam HOST float [V][12]: the rows [R | t] of a rigid transform, finite.
 * Every fp32 operation rounds to nearest once, in the order written; (float)i is exact.
 *
 * pvb_depth_points: out_points DEVICE float [V][H][W][3].  A valid pixel (i, j) of depth d gives
 *   x = ((float)j - cx) * d / fx,  y = ((float)i - cy) * d / fy  (subtract, multiply, divide), p_cam = (x, y, d),
 *   world = R p_cam + t, row k as fma(R_k0, x, fma(R_k1, y, fma(R_k2, d, t_k))) (composed_xform);
 * an invalid pixel gives (NaN, NaN, NaN).
 *
 * pvb_depth_carve: out_state DEVICE uint8 [nx][ny][nz] (C order, z fastest), dims HOST int32[3] each 2..1024, lo HOST
 * float[3] finite.  Voxel (ix, iy, iz) has its centre c_k = lo_k + (float)i_k * resolution (multiply, then add).  Per
 * view, p = world_to_cam c (the same FMA chain); the view says nothing when p.z <= 0, when the pixel
 *   (row floor(fy * p.y / p.z + cy + 0.5), column floor(fx * p.x / p.z + cx + 0.5))  (multiply, divide, add, add)
 * lies outside the image, or when that pixel is invalid; otherwise it says free when p.z < d - free_margin.  The
 * voxel's state is 0 (free) when any view says free and 2 (unknown) otherwise; the order of the views does not
 * matter.  Occupied voxels (1) are written afterwards by pvb_voxel_scatter of the valid points: hits win over free.
 *
 * PVB_ERR_INVALID before any device work: V, H or W out of range, null pointers, a focal length that is not finite
 * and positive, a principal point or transform entry that is not finite, max_depth <= 0 or NaN; for the carve also
 * dims outside 2..1024, a resolution that is not finite and positive, a free_margin that is negative or not finite
 * and a lo that is not finite. */
int pvb_depth_points(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                     const float *cam_to_world, float max_depth, float *out_points, void *stream);
int pvb_depth_carve(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                    const float *world_to_cam, float max_depth, float free_margin, const float *lo, float resolution,
                    const int32_t *dims, uint8_t *out_state, void *stream);

/* ---- occupancy maps: OccupancyMap.integrate (sdf.py) ----
 * pvb_depth_integrate: one observation of the V views of one call, fused into a log-odds occupancy grid on the
 * lattice, depth images, views and checks of pvb_depth_carve.
 * log_odds DEVICE int16 [nx][ny][nz]: log-odds in units of 1/1024; -32768 marks a voxel never observed.
 * hits DEVICE uint8 [nx][ny][nz]: nonzero where a valid pixel's point falls into the voxel.  The caller writes it
 *   with pvb_voxel_scatter (value 1) of all V*H*W points of pvb_depth_points (an invalid pixel's NaN point falls into
 *   no voxel); the kernel reads it and writes 0 back, so it is all zero when the call returns.
 * params HOST int32[4] = {hit, miss, clamp_lo, clamp_hi} in 1/1024 units, with
 *   -32767 <= clamp_lo <= miss < 0 < hit <= clamp_hi <= 32767.
 * Per voxel, in int32 arithmetic, with L = 0 for a voxel never observed:
 *   hit (hits nonzero):                                  L = min(L + hit, clamp_hi)
 *   else free (some view says free, as pvb_depth_carve):  L = max(L + miss, clamp_lo)
 *   else:                                                the stored value is unchanged (-32768 stays -32768).
 * Each voxel receives at most one update per call; the result depends on neither the view order nor the thread
 * order.  Frames taken at different times go in separate calls.
 * PVB_ERR_INVALID before any device work: pvb_depth_carve's cases, null hits, log_odds or params, and parameters
 * outside the order above. */
int pvb_depth_integrate(const float *depth, int32_t V, int32_t H, int32_t W, const float *intrinsics,
                        const float *world_to_cam, float max_depth, float free_margin, const float *lo,
                        float resolution, const int32_t *dims, uint8_t *hits, int16_t *log_odds,
                        const int32_t *params, void *stream);

/* ---- ray-cast point clouds: ray_occupancy, OccupancySDF.from_rays, OccupancyMap.integrate_points (sdf.py) ----
 * A ray is a sensor origin o and a return p, fp32 world points on pvb_depth_carve's lattice (voxel i centred at
 * lo + i * resolution, dims HOST int32[3] each 2..1024, lo HOST float[3] finite).  Every fp32 operation rounds to
 * nearest once, in the order written; fma, sqrt, min, max and floor are the IEEE operations, (float)i is exact.
 *
 * Valid ray: d = p - o per axis, l = sqrt(fma(dz, dz, fma(dy, dy, dx * dx))); the ray is valid when all six
 * coordinates of o and p are finite and 0 < l <= max_range with l finite (+inf max_range allowed).  An invalid ray
 * (a NaN row pads a ragged scan; l = 0 is a LiDAR's "no return" in the sensor frame) says nothing: no hit, no free
 * voxel.  Returns beyond max_range are dropped.
 * Free voxels: the face-connected (6-connected) walk of the segment o + t d, 0 <= t <= t_end, t_end = (l - m) / l with
 * m = free_margin; nothing when l <= m.  In lattice coordinates a_k = (o_k - lo_k) / resolution + 0.5 and
 * u_k = d_k / resolution, voxel i covers [i, i + 1).
 *   clip: t_lo = 0, t_hi = t_end; per axis with u_k != 0, t0 = -a_k / u_k and t1 = (n_k - a_k) / u_k give
 *     t_lo = max(t_lo, min(t0, t1)), t_hi = min(t_hi, max(t0, t1)); an axis with u_k == 0 needs 0 <= a_k < n_k.  No
 *     voxel unless t_lo < t_hi.
 *   start: i_k = floor(fma(t_lo, u_k, a_k)) clamped to 0..n_k - 1.
 *   boundaries: tb_k = ((float)(i_k + (u_k > 0)) - a_k) / u_k (subtract, divide), recomputed from the index after
 *     every step, +inf when u_k == 0; no step accumulates rounding.
 *   step: visit the voxel; take the axis of the smallest tb (ties: x, then y, then z); stop when that tb >= t_end;
 *     move its index one voxel towards u_k's sign; stop when it leaves 0..n_k - 1.
 *   Every index moves one way only: no voxel twice, at most n_x + n_y + n_z voxels per ray (also a hard loop bound).
 *
 * pvb_ray_carve: points DEVICE float [n_rays][3]; origins DEVICE float [n_rays / rays_per_origin][3], ray t taking
 * origin t / rays_per_origin.  Writes 2 into marks DEVICE uint8 [nx][ny][nz] (C order) on every free voxel of every
 * valid ray and leaves every other byte as it is; writes out_points DEVICE float [n_rays][3]: p for a valid ray and
 * (NaN, NaN, NaN) otherwise.  The caller then scatters out_points with pvb_voxel_scatter (value 1), so hits win over
 * free.  Every carve write stores the same value: the result depends on neither the ray order nor the thread order.
 * The origins are not read on the host (a non-finite origin makes its rays invalid), so the call does not
 * synchronise.
 * pvb_occupancy_apply: one observation from such marks into pvb_depth_integrate's log_odds grid: per voxel, mark 1
 * applies the hit update, mark 2 the free update and 0 nothing (any other mark nothing), then every mark is set to 0,
 * so marks is all zero when the call returns.  params as pvb_depth_integrate's.
 *
 * PVB_ERR_INVALID before any device work: null pointers, n_rays < 1, n_rays >= 2^31, a rays_per_origin < 1 or one
 * that does not divide n_rays, max_range <= 0 or NaN, dims outside 2..1024, a resolution that is not finite and
 * positive, a free_margin that is negative or not finite, a lo that is not finite; for the apply, null pointers, dims
 * outside 2..1024 and parameters outside pvb_depth_integrate's order. */
int pvb_ray_carve(const float *points, int64_t n_rays, int64_t rays_per_origin, const float *origins,
                  float max_range, float free_margin, const float *lo, float resolution, const int32_t *dims,
                  uint8_t *marks, float *out_points, void *stream);
int pvb_occupancy_apply(uint8_t *marks, int16_t *log_odds, const int32_t *dims, const int32_t *params, void *stream);

/* ---- rigid transform helpers used by the generic (unfused) composition path ---- */
/* out[b][i] = xforms[b] applied to pts[i] (pts DEVICE [n_pts][3], out DEVICE [n_tf][n_pts][3]), the FMA chain of the
 * composed kernels' transform; any n_tf >= 0, PVB_ERR_INVALID when n_tf * n_pts * 3 overflows int64 */
int pvb_transform_points(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts,
                         float *out, void *stream);
/* paired: out[b][i] = xforms[b] applied to pts[b][i] (pts / out DEVICE [n_tf][n_pts][3]), same arithmetic as the
 * composed kernels' transform -- the generic path of the paired query (pvb_composed_query_paired) */
int pvb_transform_points_paired(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts,
                                float *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PVB_H */
