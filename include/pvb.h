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

/* sub-SDF kinds understood by the fused kernels */
enum { PVB_KIND_GRID = 0, PVB_KIND_MESH = 1, PVB_KIND_SPHERE = 2 };

/* pvb_sdf_desc.flags */
enum {
    PVB_GRID_INDEX_FP32 = 1u << 0, /* voxel index arithmetic in fp32 (range given as Python floats);
                                      default is fp64, the dtype torch infers for numpy ranges */
    PVB_GRID_OOB_GT     = 1u << 1, /* OutOfBoundsStrategy.LOOKUP_GT_SDF: out-of-range points take the
                                      mesh query (mesh fields must be filled); default BOUNDING_BOX */
    PVB_GRID_PRUNE_OK   = 1u << 2, /* table verified to satisfy val >= dist(voxel centre, bb) - prune_margin:
                                      composed kernels may skip lookups that provably cannot win the min */
    PVB_GRID_TRILINEAR  = 1u << 4, /* EXTENSION (not reference behaviour): value = trilinear interpolation of the
                                      8 surrounding voxel values, gradient = analytic gradient of that interpolant
                                      (cell-wise finite differences).  pvb_grid_lookup only. */
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
 * SPHERE     = SphereSDF radius (sdf.py:285-299).
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
    float bb_min[3];            /* surface AABB, fp32 */
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
    /* ---- sphere ---- */
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
 * <= 16 GRID sub-SDFs with the bounding-box out-of-range rule (a RobotSDF of cached links). */
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

/* ---- rigid transform helpers used by the generic (unfused) composition path ---- */
int pvb_transform_points(const float *xforms, int32_t n_tf, const float *pts, int64_t n_pts,
                         float *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PVB_H */
