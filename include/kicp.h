/*
 * kicp.h — C ABI of the H100-native kinematic-icp registration hot path (libkicp_b200.so).
 *
 * The reference (PRBonn/kinematic-icp @ 07c2851, v0.1.1) has no FFI: its hot path is a C++ value API
 * (SURVEY.md §8(b)).  This header is the boundary a binding for that path would bind; every entry point cites
 * the reference interface it replaces (paths relative to the reference root).  The C++ facade in
 * kinematic-icp_b200/cpp/ (same class names, namespaces and signatures as the reference headers) sits on top
 * of exactly these functions, so the ROS 2 nodes keep including "kinematic_icp/pipeline/KinematicICP.hpp" unchanged.
 *
 * Conventions
 *   - plain pointers and sizes only; every function returns an int status (KICP_OK == 0);
 *   - points are row-major xyz doubles (std::vector<Eigen::Vector3d> is layout-compatible: 3 contiguous doubles);
 *   - a pose is double[7] = {qx, qy, qz, qw, tx, ty, tz} — Eigen::Quaterniond coefficient order followed by the
 *     translation, i.e. the two members of Sophus::SE3d;
 *   - host pointers unless the name says "device"; calls are synchronous unless the name says "async";
 *   - there is NO CPU fallback: without a CUDA device every call fails with KICP_ERR_CUDA.
 */
#ifndef KICP_H_
#define KICP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KICP_VERSION 100
#define KICP_MAX_ITERATIONS 64 /* upper bound accepted for max_num_iterations (reference default: 10) */

enum kicp_status {
    KICP_OK = 0,
    KICP_ERR_CUDA = 1,        /* CUDA runtime error (no device, launch failure, out of memory); see kicp_last_error */
    KICP_ERR_INVALID = 2,     /* bad argument */
    KICP_ERR_UNSUPPORTED = 3, /* e.g. max_points_per_voxel > 255 */
    KICP_ERR_NCCL = 4,
    KICP_ERR_CAPACITY = 5,
    /* The reference divides by the correspondence count with no guard (Registration.cpp:119-125): with zero
     * correspondences its pose becomes NaN.  We stay drop-in (the returned pose IS NaN) and also say so. */
    KICP_WARN_NO_CORRESPONDENCES = 16
};

#define KICP_DTYPE_F64 0 /* std::vector<Eigen::Vector3d> storage */
#define KICP_DTYPE_F32 1 /* PointCloud2 FLOAT32 fields */

typedef struct kicp_ctx kicp_ctx;   /* one GPU: device id, stream, scratch, optional NCCL communicator */
typedef struct kicp_map kicp_map;   /* kiss_icp::VoxelHashMap resident in HBM */
typedef struct kicp_scan kicp_scan; /* a scan (the `frame` argument of ComputeRobotMotion) resident in HBM */

/* kinematic_icp::KinematicRegistration's public fields (registration/Registration.hpp:45-49).  max_num_threads_
 * has no GPU meaning and is not carried. */
typedef struct kicp_reg_params {
    int32_t max_num_iterations;                   /* Registration.hpp:45, default 10 (pipeline/KinematicICP.hpp:52) */
    int32_t use_adaptive_odometry_regularization; /* Registration.hpp:48, default true (KinematicICP.hpp:55) */
    double convergence_criterion;                 /* Registration.hpp:46, default 1e-3 (KinematicICP.hpp:53) */
    double fixed_regularization;                  /* Registration.hpp:49, default 0.0 (KinematicICP.hpp:56) */
} kicp_reg_params;

/* Result of one registration.  sums[j] are the normal-equation sums of solve j BEFORE the /N normalisation
 * (Registration.cpp:110-118): {JTJ00, JTJ01, JTJ11, JTr0, JTr1, N, sum |r|^2, 0}; dx[j] = (d, theta). */
typedef struct kicp_reg_result {
    double pose[7];          /* the SE3d ComputeRobotMotion returns */
    double beta;             /* odometry regularisation actually used (Registration.cpp:171-177) */
    double last_dx_norm;
    int32_t iterations;      /* number of ComputePerturbation solves == DataAssociation passes executed */
    int32_t status;          /* KICP_OK or KICP_WARN_NO_CORRESPONDENCES */
    double sums[KICP_MAX_ITERATIONS][8];
    double dx[KICP_MAX_ITERATIONS][2];
} kicp_reg_result;

const char *kicp_status_string(int status);
/* Thread-local text of the last failure (CUDA / NCCL error string and the call site). */
const char *kicp_last_error(void);

/* ---- context ------------------------------------------------------------------------------------------- */
int kicp_ctx_create(int device, kicp_ctx **out);
int kicp_ctx_destroy(kicp_ctx *ctx);
int kicp_ctx_synchronize(kicp_ctx *ctx);
/* The CUDA stream (cudaStream_t) all work of this context is enqueued on — so a caller can time it with events. */
void *kicp_ctx_stream(kicp_ctx *ctx);
/* Number of this library's kernels launched on the context since creation (bench.py reports gpu_launches). */
int64_t kicp_ctx_launch_count(kicp_ctx *ctx);
/* Ordering with a caller's CUDA stream (`stream` is a cudaStream_t of the context's device; 0, cudaStreamLegacy and
 * cudaStreamPerThread are accepted).  The context stream is non-blocking, so a producer or consumer on another stream must be ordered
 * explicitly.  Each call records an event the context owns on one stream and makes the other wait for it; neither waits on the host.
 *   kicp_ctx_wait_stream: the context's later work waits for everything enqueued on `stream` so far (call it before handing the
 *                         library device memory that `stream` writes);
 *   kicp_stream_wait_ctx: `stream`'s later work waits for everything enqueued on the context so far (call it before `stream` reads
 *                         what an "async" device output wrote, or reuses memory a registration reads in place).
 * Errors: KICP_ERR_INVALID for a null ctx; KICP_ERR_CUDA for a stream the runtime rejects. */
int kicp_ctx_wait_stream(kicp_ctx *ctx, void *stream);
int kicp_stream_wait_ctx(kicp_ctx *ctx, void *stream);
/* Options: "persistent" 1 = all IRLS iterations of a registration inside ONE cooperative launch (default), 0 = one launch per
 * iteration; "stats" 1 = count hash probes / candidate points / 128-byte lines on the device (bench.py's touched-bytes figure);
 * "ctas_per_sm" = cap of the resident CTAs per SM the grid is sized for (0 = occupancy limit); "nn_cache" = between IRLS
 * passes every point keeps its two nearest candidates together with a certificate (a lower bound on the distance to every other
 * candidate) and a pass re-searches only the points whose certificate the pose update broke (exact, see DESIGN.md): 1 = for
 * scans of 49152 points or more (default: smaller scans gain nothing from the extra phase), 2 = always, 0 = never; "overlap_upload" 1 = the
 * host-pointer entry points overlap the frame's upload with the first pass (default); "spin_timeout_ms" = bound of every
 * device-side wait (upload flags, peers of the fused exchange; default 20000); "frame_sync" 1 = kicp_register_frame reads the
 * survivor counts back in the middle of a frame (legacy order; default 0 = ONE host synchronisation per frame, at its end).
 * "downsample_order" sets the output order of every VoxelDownsample on the context (kicp_voxel_downsample and both down-samples
 * of kicp_register_frame / kicp_register_staged_frame): 0 = the order of first occurrence (default), 1 = the iteration order of
 * the tsl::robin_map that KISS-ICP v1.2.0's VoxelDownsample fills (reserved for the down-sample's input count, the library's
 * 3-prime XOR hash, robin-hood insertion in input order), so that a frame picks the source points and builds the map the
 * library's own pipeline does.  Mode 1 restates that container from memory and is UNPINNED exactly as the test oracle's mode 1
 * is: pinning it means checking both against the library.  It accepts at most 2^28 points per down-sample (KICP_ERR_INVALID
 * beyond).  Other values fail with KICP_ERR_INVALID.
 * "correspondences" 1 = every frame call (kicp_register_frame, kicp_register_staged_frame, _sensors and the _segments variants) also
 * evaluates the registration source at the returned pose against the map BEFORE the frame's Update, by the rules of
 * kicp_map_correspondences: two more kernel launches per frame, the pose read from the device result block and the source count from
 * the device, and no further host synchronisation (the statistics come back with the frame's).  Read them with
 * kicp_frame_correspondences / kicp_frame_correspondences_device.  The first frame (empty map) has no inliers and fitness 0; a frame
 * that returns KICP_WARN_NO_CORRESPONDENCES is evaluated at its NaN pose, so every distance is DBL_MAX and a finite tau gives no
 * inliers (the map stays untouched as always); with "frame_sync" 1 the count is the one read back mid-frame.  0 (default) = no launch,
 * no allocation, nothing of any result changes.
 * Unknown names fail with KICP_ERR_INVALID.
 * Every setting but "downsample_order" computes the same result up to the summation order. */
int kicp_ctx_set_option(kicp_ctx *ctx, const char *name, int32_t value);
/* Per-kernel device timing with CUDA events recorded on the context stream around (a) the set-up of each registration
 * (k_reg_init, multi-launch path only) and (b) every launch of the registration kernel.  Only
 * launches that did work are counted in assoc_* (a launch issued after convergence exits at its first instruction
 * and is reported under idle_*).  kicp_ctx_profile_end synchronises the stream. */
typedef struct kicp_profile {
    double assoc_ms;          /* summed duration of the association launches that did work */
    int64_t assoc_launches;
    double idle_ms;           /* launches issued after convergence (early exit) */
    int64_t idle_launches;
    double prep_ms;           /* set-up launches, summed over registrations (0 on the persistent path) */
    int64_t registrations;
    int64_t assoc_iterations; /* IRLS iterations executed by those launches (a persistent launch runs several) */
} kicp_profile;
int kicp_ctx_profile_begin(kicp_ctx *ctx);
int kicp_ctx_profile_end(kicp_ctx *ctx, kicp_profile *out);
/* Pinned host memory for truly asynchronous copies (std::vector storage works too, just slower). */
int kicp_host_alloc(uint64_t bytes, void **out);
int kicp_host_free(void *p);

/* ---- kiss_icp::VoxelHashMap (KISS-ICP v1.2.0 core/VoxelHashMap.hpp; used by the reference at
 *      pipeline/KinematicICP.hpp:79,88,92, pipeline/KinematicICP.cpp:79, registration/Registration.cpp:74,157) --- */
/* VoxelHashMap(voxel_size, max_distance, max_points_per_voxel) */
int kicp_map_create(kicp_ctx *ctx, double voxel_size, double max_distance, uint32_t max_points_per_voxel, kicp_map **out);
int kicp_map_destroy(kicp_map *map);
/* Pre-size the map's device storage for `voxels` occupied voxels (like tsl::robin_map::reserve on the reference's
 * map_ member).  Optional: kicp_map_create already sizes for a disc of radius max_distance, and the storage doubles
 * when exceeded — but growth re-allocates, which is the one slow (milliseconds) event of a drive. */
int kicp_map_reserve(kicp_map *map, int64_t voxels);
int kicp_map_clear(kicp_map *map);                         /* Clear(), KinematicICP.hpp:88 */
int kicp_map_empty(kicp_map *map, int32_t *empty);         /* Empty(), Registration.cpp:157 */
int kicp_map_num_points(kicp_map *map, int64_t *n);
int kicp_map_num_voxels(kicp_map *map, int64_t *n);
int kicp_map_add_points(kicp_map *map, const double *xyz, int64_t n);                /* AddPoints(points) */
int kicp_map_remove_far(kicp_map *map, const double origin[3]);                      /* RemovePointsFarFromLocation */
int kicp_map_update(kicp_map *map, const double *xyz, int64_t n, const double origin[3]); /* Update(points, origin) */
/* Update(points, pose): transform by pose, AddPoints, evict around pose.translation()  (KinematicICP.cpp:79) */
int kicp_map_update_pose(kicp_map *map, const double *xyz, int64_t n, const double pose[7]);
/* Pointcloud(), KinematicICP.hpp:92.  *n receives the count; fails with KICP_ERR_CAPACITY if cap is too small. */
int kicp_map_pointcloud(kicp_map *map, double *out_xyz, int64_t cap, int64_t *n);
/* Pointcloud() as the records EigenToPointCloud2 (ros/.../utils/RosUtils.cpp:41-63) builds from it: x, y, z FLOAT32 at byte
 * offsets 0, 4, 8, point_step 12, in kicp_map_pointcloud's order; each coordinate is static_cast<float> as on x86-64, NaN bits
 * included.  out_xyz: any host memory, n*3 floats (page-locked is fastest).  *n receives the count; KICP_ERR_CAPACITY if cap < n. */
int kicp_map_pointcloud_f32(kicp_map *map, float *out_xyz, int64_t cap, int64_t *n);
/* Pointcloud() (dtype KICP_DTYPE_F64: xyz doubles) or kicp_map_pointcloud_f32's records (KICP_DTYPE_F32) in the same order and the
 * same bytes, written by the packing kernel straight into `out`: device memory of the context's device for cap points, aligned to
 * the element size (never NULL).  Enqueued on the context stream with no host synchronisation; order a reader on another stream with
 * kicp_stream_wait_ctx.  *n receives the map's point count (known on the host).  Errors: KICP_ERR_CAPACITY when cap < *n (nothing
 * enqueued); KICP_ERR_INVALID for a null argument, another dtype, or `out` that is not such memory or misaligned. */
int kicp_map_pointcloud_device_async(kicp_map *map, void *out, int32_t dtype, int64_t cap, int64_t *n);
/* The same records kept up to date incrementally, for a node that publishes the local map every frame: the map owns a page-locked
 * buffer of them, and each call writes into it only the records that changed since the previous call, decided on the device.
 *   - Content: after the call, the n 12-byte records at *records are, as a multiset and bit for bit, those kicp_map_pointcloud_f32
 *     returns at that moment.  Their order is unspecified.
 *   - Stability: a record whose point is still in the map keeps its position unless it is moved to fill a hole.  Holes are filled
 *     first by new records, then by records moved from the tail, so the buffer stays dense.  A call after which nothing changed
 *     (including a frame that returned KICP_WARN_NO_CORRESPONDENCES) writes nothing.
 *   - Cost: at most 12 * written bytes cross PCIe, plus a few words, and the host synchronises once.
 *   - Lifetime: the bytes change only inside this call; the pointer stays valid until the next call on the same map or
 *     kicp_map_destroy.  When the map outgrows the buffer, the call allocates a larger one (the pointer changes) and writes all n
 *     records.  Clear, load and every update need no hook: the next call sees what is gone and what is new.  The first call
 *     allocates the state; a map that never calls this pays nothing.
 * stats may be NULL. */
typedef struct kicp_map_live_stats {
    int64_t added;     /* records of points stored since the previous call */
    int64_t removed;   /* records of points gone since the previous call (evicted voxels, Clear, load) */
    int64_t moved;     /* surviving records relocated to fill holes */
    int64_t rewritten; /* surviving positions whose bytes changed (a voxel evicted and re-created at the same key between calls) */
    int64_t written;   /* records that crossed PCIe in this call: added + moved + rewritten, or n after the buffer grew */
} kicp_map_live_stats;
int kicp_map_pointcloud_f32_live(kicp_map *map, const float **records, int64_t *n, kicp_map_live_stats *stats);
/* Voxel-grouped dump: keys[V][3], counts[V], points[total][3] in per-voxel insertion order (tests, checkpoints). */
int kicp_map_export_voxels(kicp_map *map, int32_t *keys, int32_t *counts, double *points, int64_t cap_voxels,
                           int64_t cap_points, int64_t *num_voxels, int64_t *num_points);
/* Bulk load of a voxel-grouped map (replaces the content): the inverse of kicp_map_export_voxels. */
int kicp_map_load_voxels(kicp_map *map, const int32_t *keys, const int32_t *counts, const double *points,
                         int64_t num_voxels);
/* ---- a frozen prior inside the map: a map has P prior voxels (0 by default), the first P voxels in its block order (the order of
 *      kicp_map_export_voxels and kicp_map_pointcloud).  Every reader (registration, nearest, correspondences, pose search, planar
 *      alignment, the exports) sees one map: the prior voxels followed by the live ones.
 *   - Prior voxels are read-only: while frozen their keys, counts and point bytes do not change, and they stay at positions [0, P).
 *   - Insertion: every AddPoints (host and _device variants, both Updates, the frame path's Update in both synchronisation orders)
 *     drops a point whose voxel key is a prior voxel's; every other point follows the reference's rule, which looks only inside the
 *     point's own voxel.  The live voxels are therefore exactly the map the same calls build from an empty map, fed only the points
 *     that were not dropped.
 *   - Eviction: prior voxels never die; live voxels die by the reference's rule (first point >= max_distance from the origin).
 *   - The frame path's map-update policy is unchanged: NEVER skips the whole Update, ALWAYS and GATED apply it to the live voxels, and
 *     GATED's "the map held no points" is about the whole map.
 *   - kicp_map_clear and kicp_map_load_voxels reset P to 0 ("load, then freeze" is two calls); so does the facade's SetPose, which
 *     clears the map as the reference does.  A map that never freezes runs exactly the code, launches and bytes it ran before.
 *   - Cost while frozen: an Update compacts and re-inserts only the live voxels, plus one device copy of a snapshot of the prior's
 *     hash table (16 bytes a slot, 4 to 8 slots per voxel of capacity); freezing copies the prior once into the spare block arrays.
 * kicp_map_freeze: every voxel now in the map becomes prior (P = number of voxels); a second freeze also takes in the live voxels
 * added since.  kicp_map_thaw: P = 0, the voxels stay as ordinary ones (the next eviction may remove them).  Both synchronise.
 * kicp_map_pointcloud_f32_live still diffs the whole map.  Errors: KICP_ERR_INVALID for a null argument, named by kicp_last_error. */
int kicp_map_freeze(kicp_map *map);
int kicp_map_thaw(kicp_map *map);
/* the prior's voxel and point counts (0, 0 when nothing is frozen) */
int kicp_map_prior_size(kicp_map *map, int64_t *voxels, int64_t *points);
#define KICP_MAP_LAYER_ALL 0   /* every voxel: kicp_map_pointcloud's points */
#define KICP_MAP_LAYER_PRIOR 1 /* the frozen prior voxels [0, P) */
#define KICP_MAP_LAYER_LIVE 2  /* the voxels after them */
/* kicp_map_pointcloud (dtype KICP_DTYPE_F64) or kicp_map_pointcloud_f32 (KICP_DTYPE_F32) of one layer: ALL is PRIOR followed by LIVE,
 * byte for byte.  A node that localises on a prior publishes PRIOR once and LIVE every frame.  *n receives the layer's point count.
 * The _device_async form packs into device memory as kicp_map_pointcloud_device_async does.  Errors: KICP_ERR_INVALID for a null
 * argument, a layer or dtype outside the values above, or (device) `out` that is not such memory, named by kicp_last_error;
 * KICP_ERR_CAPACITY when cap < *n (nothing copied). */
int kicp_map_pointcloud_layer(kicp_map *map, int32_t layer, int32_t dtype, void *out, int64_t cap, int64_t *n);
int kicp_map_pointcloud_layer_device_async(kicp_map *map, int32_t layer, int32_t dtype, void *out, int64_t cap, int64_t *n);

/* ---- free-space clearing: live voxels that a cloud's rays pass through leave the map (a van that drove off, a door that opened).
 *      Inputs: the map (voxel size v, max_distance D, P prior voxels), n points p_i in a frame F, a pose T (F -> map) and a sensor
 *      origin s in F, and the parameters below.  Plain IEEE double arithmetic with no contraction throughout:
 *   1. o = T s and q_i = T p_i, the transform kicp_map_update_pose applies, bit for bit.
 *   2. K(x) is the map's voxel key per axis (INT_MIN for a non-finite or huge value).  A ray is CAST when no coordinate of K(o) or
 *      K(q_i) is INT_MIN; other rays do nothing.
 *   3. Hit: a cast ray hits its end voxel K(q_i).
 *   4. Misses: d = q_i - o, L = sqrt(dx*dx + dy*dy + dz*dz) (added in x, y, z order), t_end = min(L - end_margin, D) / L.  No voxel is
 *      visited when L == 0 or t_end <= 0.  Otherwise a 3-D DDA runs from k = K(o).  Per axis j: d_j > 0: step +1,
 *      tmax_j = ((k_j + 1) * v - o_j) / d_j, tdelta_j = v / d_j; d_j < 0: step -1, tmax_j = (k_j * v - o_j) / d_j, tdelta_j = -v / d_j;
 *      d_j == 0: tmax_j = +inf (k_j + 1 and k_j * v in double).  Visit k; then at most |K(q_i) - K(o)|_1 times: take the axis j of the
 *      smallest tmax (the lowest index on ties), stop if tmax_j >= t_end, else k_j += step_j, tmax_j += tdelta_j and visit k.  A visited
 *      voxel that is in the map and is not K(q_i) gets one miss from this ray.
 *   5. Decision (occupancy off; kicp_map_set_occupancy below keeps evidence across calls): a LIVE voxel (block index >= P) with at
 *      least min_misses misses and no hit is cleared.  A prior voxel that meets the condition is kept (prior voxels are read-only, kicp_map_freeze) and counted in prior_contradicted: its prior is going stale.
 *   6. Removal: cleared voxels leave through the eviction's stable compaction; the survivors keep their relative order, so the exports
 *      after the call are determined bit for bit.
 *      The result depends only on integer counts: not on the order of the rays or on the launch shape.
 *      Cost: one ray per point, one hash probe per voxel visited (up to about 3 D / v per ray); the map keeps one flag word per voxel
 *      of capacity, allocated by its first clearing (a map that never clears allocates nothing). ------------------------------- */
typedef struct kicp_free_space_params {
    double end_margin;  /* metres cut from the end of every ray (>= 0, finite): keeps the voxels just before a hit */
    int32_t min_misses; /* misses a live voxel needs to be cleared (>= 1; kicp_ctx_set_free_space: 0 = off) */
} kicp_free_space_params;
typedef struct kicp_free_space_stats {
    int64_t rays;               /* rays cast */
    int64_t visits;             /* voxels visited, summed over the cast rays */
    int64_t cleared_voxels;     /* live voxels cleared */
    int64_t cleared_points;     /* the points they held */
    int64_t prior_contradicted; /* prior voxels that met the condition and were kept */
} kicp_free_space_stats;
/* The rule above for n host points at xyz.  Synchronous, with one host synchronisation; the host mirrors are current when it returns.
 * `stats` may be NULL.  Errors: KICP_ERR_INVALID, with kicp_last_error naming the argument, for a null map, pose, sensor_origin or params,
 * xyz == NULL with n > 0, n < 0 or n >= 2^40, a non-finite pose or origin, an end_margin that is NaN, negative or infinite, or
 * min_misses < 1. */
int kicp_map_clear_free_space(kicp_map *map, const double *xyz, int64_t n, const double pose[7], const double sensor_origin[3],
                              const kicp_free_space_params *params, kicp_free_space_stats *stats);
/* The same for n device points in kicp_map_nearest_device_async's layout and validation rules (packed float64 read in place, other
 * layouts widened once into the map's buffer); synchronous like the host variant. */
int kicp_map_clear_free_space_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                     int32_t offset_y, int32_t offset_z, const double pose[7], const double sensor_origin[3],
                                     const kicp_free_space_params *params, kicp_free_space_stats *stats);
/* ---- occupancy evidence: a setting of the MAP (not of the context: the evidence is map state and survives evictions, growth and
 *      freezes) that gives step 5 above a memory across clearing calls.  One clearing call is kicp_map_clear_free_space[_device] or
 *      the frame path's clearing after an applied Update (kicp_ctx_set_free_space); steps 1-4 give every voxel b its hit_b and miss_b,
 *      and free_b = !hit_b && miss_b >= min_misses is the condition of step 5.
 *   Off (the default, or after kicp_map_set_occupancy(map, NULL)): step 5 as above.
 *   On: every LIVE voxel (block index >= P) carries an int32 evidence e_b, updated once per clearing call:
 *     hit_b:  e_b = min(e_b + hit_gain, max_evidence);
 *     else free_b: e_b = e_b - miss_loss, and the voxel is cleared when e_b <= 0 (it leaves through step 6 and is counted in
 *             cleared_voxels / cleared_points);
 *     else:   unchanged.
 *   Prior voxels keep their evidence while frozen; prior_contradicted counts free_b as above.  A voxel gets `initial` when an insert
 *   creates it (every AddPoints / Update variant and the frame path), when kicp_map_load_voxels loads it, and when it is in the map at
 *   a kicp_map_set_occupancy call (every set call resets all voxels to `initial`); a voxel evicted by distance and created again starts
 *   again at `initial`.  kicp_map_freeze freezes the prior voxels' evidence with them and kicp_map_thaw resumes it; kicp_map_clear (and
 *   the facade's SetPose) empties the map and keeps the setting.  Only clearing calls change evidence: an Update without clearing
 *   leaves it alone, and a node that clears once per sensor updates it once per such call.  The result depends only on integer counts
 *   (not on ray order or launch shape), and {1, 0, 1, 1} gives the memoryless rule's exports and statistics byte for byte.
 *   Cost: two int32 per block of capacity (the evidence and its compaction target), allocated by the set call; no extra launch in the
 *   clearing calls or the inserts (kicp_map_load_voxels adds one fill). -------------------------------------------------------------- */
typedef struct kicp_occupancy_params {
    int32_t initial;      /* evidence of a new voxel: 1 <= initial <= max_evidence */
    int32_t hit_gain;     /* added when a ray ends in the voxel: 0 <= hit_gain <= 2^24 */
    int32_t miss_loss;    /* subtracted when the voxel is free in a call: 1 <= miss_loss <= 2^24 */
    int32_t max_evidence; /* the cap of the evidence: max_evidence <= 2^24 (with these bounds int32 arithmetic cannot overflow) */
} kicp_occupancy_params;
/* Turns occupancy on with `params` (every voxel now in the map, prior included, starts at params->initial) or off with NULL (the
 * arrays are freed).  Synchronous.  Errors: KICP_ERR_INVALID, with kicp_last_error naming the field, for a value out of range, or a
 * null map; the previous setting is kept. */
int kicp_map_set_occupancy(kicp_map *map, const kicp_occupancy_params *params);
/* The evidence of every voxel in kicp_map_export_voxels' block order (prior first): *n = the voxel count, then n int32 copied to
 * `evidence` with one host synchronisation.  Errors: KICP_ERR_INVALID when occupancy is off or for a null map or n (evidence may be
 * NULL when the map is empty), KICP_ERR_CAPACITY when cap < *n (nothing copied). */
int kicp_map_export_occupancy(kicp_map *map, int32_t *evidence, int64_t cap, int64_t *n);
/* GetClosestNeighbor(query) for n queries: (closest point, distance); (0,0,0), DBL_MAX when nothing is found. */
int kicp_map_nearest(kicp_map *map, const double *queries, int64_t n, double *out_points, double *out_dist);
/* ---- the map operators on clouds in device memory.  `data` holds n points of device memory of the context's device in the layout of
 *      kicp_scan_attach_device (dtype KICP_DTYPE_F64 or KICP_DTYPE_F32, point_step 0 = tightly packed x,y,z, else the byte stride
 *      with the field offsets), with no alignment required.  Each returns bit for bit what its host variant returns for the same
 *      points, float32 fields widened exactly to double.  Packed float64 points are read in place; any other layout is first widened
 *      by one more kernel into the map's own buffer.  Errors: KICP_ERR_INVALID for a null map or argument, n < 0, a bad layout, and
 *      any pointer that is not device memory of the context's device (host memory, page-locked included, another GPU's memory, null),
 *      checked at both ends of its range before any work; kicp_last_error names the argument.  None of them discards a frame staged
 *      by kicp_frame_stage. */
/* AddPoints, Update(points, origin), Update(points, pose): the host synchronises once, as in the host variants, and the caller's
 * memory is free to change when they return. */
int kicp_map_add_points_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                               int32_t offset_y, int32_t offset_z);
int kicp_map_update_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                           int32_t offset_y, int32_t offset_z, const double origin[3]);
int kicp_map_update_pose_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                int32_t offset_y, int32_t offset_z, const double pose[7]);
/* GetClosestNeighbor for n device queries, by the rules of kicp_map_nearest: n x 3 doubles to out_points and n doubles to out_dist,
 * device memory of the context's device aligned to 8 bytes.  Enqueued on the context stream with no host synchronisation: order a
 * producer of the queries first (kicp_ctx_wait_stream), a reader of the results after (kicp_stream_wait_ctx), and leave the queries
 * unchanged until then (or kicp_ctx_synchronize): they are read in place. */
int kicp_map_nearest_device_async(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                  int32_t offset_y, int32_t offset_z, double *out_points, double *out_dist);

/* ---- correspondences at a pose: how well a cloud fits the map at a pose, for instance how well a frame registered.
 *      The reference's DataAssociation (registration/Registration.cpp:62-81) and the sums of ComputePerturbation (:86-118) evaluated
 *      once at the pose T.  For source points p_i, i < n, a gate tau and the map:
 *        q_i = T * p_i                          (the transform kicp_map_update_pose applies, bit for bit)
 *        (n_i, d_i) = GetClosestNeighbor(q_i)   (kicp_map_nearest's rules and bits: (0,0,0), DBL_MAX for an empty neighbourhood)
 *        inlier_i = d_i < tau                   (Registration.cpp:75; a NaN distance is not an inlier)
 *      Over the inliers, with J = [R e_x | R (-p_y, p_x, 0)] and r = q_i - n_i (Registration.cpp:89-95):
 *        sum_sq = sum |r|^2, jtj = {JTJ00, JTJ01, JTJ11}, jtr = {JTr0, JTr1}: ComputePerturbation's sums at T before the /N
 *        normalisation, in the layout of the first five entries of kicp_reg_result.sums.
 *      The sums are reduced in a fixed order (per-CTA partials, then one CTA adds them in index order, no floating-point atomics), so
 *      repeated calls on the same inputs give the same bits.  The library derives no covariance from them (INTEGRATION.md shows one
 *      way a node can). ------------------------------------------------------------------------------------------------------- */
typedef struct kicp_corr_stats {
    int64_t n_points;   /* n */
    int64_t n_inliers;
    double fitness;     /* n_inliers / n_points, 0 when n_points == 0 */
    double inlier_rmse; /* sqrt(sum_sq / n_inliers), 0 without inliers */
    double sum_sq;
    double jtj[3];
    double jtr[2];
} kicp_corr_stats;
/* n host points at xyz, pose double[7]; host outputs, each of which may be NULL: out_points n x 3 doubles (n_i), out_dist n doubles,
 * out_inlier n bytes (1 = inlier), stats.  Mirrors kicp_map_nearest: one host synchronisation.  Errors: KICP_ERR_INVALID (kicp_last_error
 * names the argument) for a null map or pose, n < 0, and xyz == NULL with n > 0. */
int kicp_map_correspondences(kicp_map *map, const double *xyz, int64_t n, const double pose[7], double tau, double *out_points,
                             double *out_dist, uint8_t *out_inlier, kicp_corr_stats *stats);
/* The same for n device points in kicp_map_nearest_device_async's layout and validation rules, enqueued on the context stream with no
 * host synchronisation.  Outputs may each be NULL: out_points / out_dist device memory of the context's device aligned to 8 bytes,
 * out_inlier n bytes of such memory, stats device memory of the context's device or page-locked host memory (kicp_host_alloc),
 * written on the context stream (valid after kicp_ctx_synchronize, or on a stream ordered by kicp_stream_wait_ctx). */
int kicp_map_correspondences_device_async(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                          int32_t offset_y, int32_t offset_z, const double pose[7], double tau, double *out_points,
                                          double *out_dist, uint8_t *out_inlier, kicp_corr_stats *stats);

/* ---- relocalisation: where a cloud fits the map around a prior pose (planar offsets x, y, yaw) ----------------------------------
 * A hypothesis is an integer lattice point L = (ix, iy, ipsi) in units of u = step / 2^(levels-1) (the finest step).  Its pose is
 * prior * Delta, Delta = (Rz(ipsi * u_yaw), (ix * u_x, iy * u_y, 0)), composed on the host as the C++ facade's Sophus product does
 * (q = normalize(q_prior * (0, 0, sin(psi/2), cos(psi/2))), t = t_prior + q_prior * (x, y, 0)).  Its score is n_inliers (GetClosestNeighbor
 * distance d < tau) and sum_sq (sum of d^2 over the inliers): the count and the distances are kicp_map_correspondences' at that pose
 * bit for bit; sum_sq is added in an order of its own (fixed, so equal inputs give equal bits) and agrees with that report's sum to
 * rounding.
 * Ranking key: more inliers, smaller sum_sq, smaller |ipsi|, smaller ix^2 + iy^2, then (ipsi, ix, iy) lexicographic.
 * Level 0 scores every lattice point of the box |x| <= half_extent[0] (likewise y, yaw) on the level-0 steps; level l >= 1 scores the
 * 26 neighbours at the level's step (step / 2^l) of each of the `keep` best hypotheses so far, skipping points already scored. */
typedef struct kicp_pose_search_params {
    double half_extent[3]; /* x, y (m), yaw (rad) of level 0 around the prior; >= 0, yaw <= pi */
    double step[3];        /* level-0 lattice steps, > 0 */
    double tau;            /* inlier gate d < tau, > 0 */
    int32_t levels;        /* 1..8 */
    int32_t keep;          /* 1..64 */
} kicp_pose_search_params;
typedef struct kicp_pose_hypothesis {
    double pose[7];     /* prior * Delta */
    double offset[3];   /* x, y, yaw */
    int32_t lattice[3]; /* ix, iy, ipsi in units of step / 2^(levels-1) */
    int32_t level;      /* the level that scored it */
    int64_t n_inliers;
    double fitness;     /* n_inliers / n, 0 for n == 0 */
    double inlier_rmse; /* sqrt(sum_sq / n_inliers), 0 without inliers */
    double sum_sq;
} kicp_pose_hypothesis;
/* The best min(keep, n_scored) hypotheses by the key, over every distinct lattice point scored in the call, into out[0 .. *n_out)
 * (cap >= keep entries); *n_scored (may be NULL) = the number of lattice points scored.  n host points in the robot base frame.
 * Synchronous: one host synchronisation per level.  The map, a staged frame and the last frame's clouds and report are unchanged.
 * n == 0 and an empty map are valid (every score (0, 0): the keep lattice points nearest the prior by the key).  KICP_ERR_INVALID,
 * with kicp_last_error naming the argument, before any device work: a null map, prior, params, out or n_out; n < 0,
 * n >= 2^40 (2^30 for device points) or xyz NULL with n > 0; a non-finite prior or parameter; a bound above; cap < keep; more than 4 194 304 level-0 hypotheses; lattice coordinates
 * beyond int32. */
int kicp_map_pose_search(kicp_map *map, const double *xyz, int64_t n, const double prior[7], const kicp_pose_search_params *params,
                         kicp_pose_hypothesis *out, int32_t cap, int32_t *n_out, int64_t *n_scored);
/* The same for n device points in kicp_map_nearest_device_async's layout and validation rules (packed float64 read in place, other
 * layouts widened once into a buffer the map owns); the caller orders their producer before the call (kicp_ctx_wait_stream). */
int kicp_map_pose_search_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                int32_t offset_y, int32_t offset_z, const double prior[7], const kicp_pose_search_params *params,
                                kicp_pose_hypothesis *out, int32_t cap, int32_t *n_out, int64_t *n_scored);

/* ---- planar alignment: Gauss-Newton in (x, y, yaw) of a cloud against the map from up to 64 starting poses -------------------
 * Each starting pose T0 is aligned on its own: T = T0; for at most max_iterations steps, the inliers at T (q = T p, (nb, d) =
 * GetClosestNeighbor(q), d < tau, r = q - nb, J = [R e_x | R e_y | R (-p_y, p_x, 0)]) give A = J^T J / N and b = J^T r / N, dx =
 * -A^-1 b by a fixed LDL^T, and T = T * Delta with Delta = (R_q, (dx0, dx1, 0)), q = normalize((0, 0, dx2/2, 1)) (a turn by
 * 2 atan(dx2/2): no trigonometry, the same fixed point).  It stops with CONVERGED when |dx| < convergence (after that step),
 * NO_CORRESPONDENCES when no point is an inlier (n == 0 and an empty map included), SINGULAR when a pivot of the factorisation is not
 * positive and finite or dx is not finite (both with T unchanged), else MAX_ITERATIONS.  The report is taken at the returned pose:
 * n_inliers and the per-point distances are kicp_map_correspondences' at that pose exactly; the sums are added in an order that
 * depends on n only, so an alignment's bits do not depend on the other starting poses of the call. */
#define KICP_ALIGN_CONVERGED 0
#define KICP_ALIGN_MAX_ITERATIONS 1
#define KICP_ALIGN_NO_CORRESPONDENCES 2
#define KICP_ALIGN_SINGULAR 3
typedef struct kicp_planar_align_params {
    double tau;             /* inlier gate d < tau: finite, > 0 */
    double convergence;     /* stop when |dx| < convergence: finite, >= 0 (the reference's convergence_criterion: 1e-3) */
    int32_t max_iterations; /* 1..KICP_MAX_ITERATIONS (the reference's max_num_iterations: 10) */
} kicp_planar_align_params;
typedef struct kicp_planar_alignment {
    double pose[7];     /* the returned pose T */
    int32_t status;     /* KICP_ALIGN_* */
    int32_t iterations; /* updates applied */
    double last_step;   /* |dx| of the last update, 0 without one */
    int64_t n_inliers;  /* at pose */
    double fitness;     /* n_inliers / n, 0 for n == 0 */
    double inlier_rmse; /* sqrt(sum_sq / n_inliers), 0 without inliers */
    double sum_sq;      /* sum of |r|^2 over the inliers */
    double jtj[6];      /* J^T J over (x, y, yaw), unnormalised: {00, 01, 02, 11, 12, 22} */
    double jtr[3];      /* J^T r, unnormalised */
} kicp_planar_alignment;
/* n host points in the robot base frame (n < 2^40), n_initial (1..64) starting poses initial[7 * k .. 7 * k + 6] -> out[k].
 * Synchronous: one host synchronisation.  The map, a staged frame and the last frame's clouds and report are unchanged.
 * KICP_ERR_INVALID, with kicp_last_error naming the argument, before any device work: a null map, initial, params or out; xyz NULL
 * with n > 0; n < 0 or n >= 2^40; n_initial outside 1..64; a non-finite starting pose; a parameter outside its range above. */
int kicp_map_align_planar(kicp_map *map, const double *xyz, int64_t n, const double *initial, int32_t n_initial,
                          const kicp_planar_align_params *params, kicp_planar_alignment *out);
/* The same for n device points in kicp_map_nearest_device_async's layout and validation rules (packed float64 read in place, other
 * layouts widened once into a buffer the map owns); the caller orders their producer before the call (kicp_ctx_wait_stream). */
int kicp_map_align_planar_device(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                 int32_t offset_y, int32_t offset_z, const double *initial, int32_t n_initial,
                                 const kicp_planar_align_params *params, kicp_planar_alignment *out);

/* ---- kinematic_icp::KinematicRegistration::ComputeRobotMotion (registration/Registration.hpp:39-43,
 *      registration/Registration.cpp:151-190; single call site pipeline/KinematicICP.cpp:68-72) -------------- */
/* frame: n host points in the robot base frame.  Returns last_robot_pose * relative_wheel_odometry when the map is
 * empty (Registration.cpp:157).  `result` may be NULL. */
int kicp_register(kicp_map *map, const double *frame_xyz, int64_t n, const double last_robot_pose[7],
                  const double relative_wheel_odometry[7], double max_correspondence_distance,
                  const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result);

/* Same computation with the scan already resident in HBM, enqueued without a host synchronisation: `result` is
 * written by an asynchronous device-to-host copy and is valid after kicp_ctx_synchronize (pinned memory from
 * kicp_host_alloc keeps the copy asynchronous). */
int kicp_scan_create(kicp_ctx *ctx, int64_t capacity, kicp_scan **out);
int kicp_scan_destroy(kicp_scan *scan);
int kicp_scan_upload(kicp_scan *scan, const double *xyz, int64_t n);       /* synchronous host -> HBM copy */
int kicp_scan_upload_async(kicp_scan *scan, const double *xyz, int64_t n); /* enqueued on the context stream */
/* The same two uploads for a frame held as float32 or float64 x,y,z fields at a byte stride (dtype / point_step / offsets as in
 * kicp_frame_input below; point_step 0 = tightly packed): the bytes cross PCIe as they are — half the traffic for the float32
 * clouds the reference's callers actually hold (RosUtils.cpp:30-39 widens float32 PointCloud2 fields to double) — and the
 * registration kernel widens while it reads.  Field offsets and point_step must be multiples of the field width. */
int kicp_scan_upload_points(kicp_scan *scan, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                            int32_t offset_y, int32_t offset_z);
int kicp_scan_upload_points_async(kicp_scan *scan, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                  int32_t offset_y, int32_t offset_z);
/* kicp_register for such a frame (host pointer). */
int kicp_register_points(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                         int32_t offset_y, int32_t offset_z, const double last_robot_pose[7],
                         const double relative_wheel_odometry[7], double max_correspondence_distance,
                         const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result);
int kicp_register_scan_async(kicp_map *map, kicp_scan *scan, const double last_robot_pose[7],
                             const double relative_wheel_odometry[7], double max_correspondence_distance,
                             const kicp_reg_params *params, kicp_reg_result *result);
/* Zero-copy scan: the scan refers to n points of the caller's device memory (of the context's device) in the layout of
 * kicp_scan_upload_points, until the next upload or attach on that scan; kicp_register_scan_async and
 * kicp_register_scan_sharded_async read it in place.  In addition to the layout rules, `data` must be aligned to the field width.
 * Nothing is enqueued: order the producer first (kicp_ctx_wait_stream), and leave the memory unchanged until the registrations that
 * read it have completed (kicp_ctx_synchronize, or kicp_stream_wait_ctx on the stream that will change it).  The scan keeps its own
 * buffer for later uploads, and kicp_scan_destroy never frees attached memory.  Errors: KICP_ERR_INVALID for a null scan, n < 0,
 * a bad layout, and data that is not device memory of the context's device (host memory, page-locked included, or another GPU's),
 * null or misaligned; a failing attach leaves the scan as it was. */
int kicp_scan_attach_device(kicp_scan *scan, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                            int32_t offset_y, int32_t offset_z);

/* ---- front end of KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:38-44,54-59; KISS-ICP v1.2.0) ---------------- */
/* kiss_icp::VoxelDownsample(frame, voxel_size): the first point (input order) of every voxel, in input order (with context option
 * "downsample_order" 1: in the library's robin_map order). */
int kicp_voxel_downsample(kicp_ctx *ctx, const double *xyz, int64_t n, double voxel_size, double *out_xyz, int64_t cap,
                          int64_t *m);
/* kiss_icp::Preprocessor::Preprocess(frame, timestamps, relative_motion) — de-skew with exp((s-1) log(relative_motion))
 * when `deskew` and stamps are given (n_stamps == n), keep min_range < |p| < max_range — followed by the transform of
 * the survivors by lidar_to_base (KinematicICP.cpp:59).  Pass the identity pose to get Preprocess alone. */
int kicp_preprocess(kicp_ctx *ctx, const double *xyz, int64_t n, const double *stamps, int64_t n_stamps,
                    const double relative_motion[7], const double lidar_to_base[7], double max_range, double min_range,
                    int32_t deskew, double *out_xyz, int64_t cap, int64_t *m);
/* The two on a cloud in device memory (`data` ... `offset_z` as for kicp_map_add_points_device; `stamps`, when read, n doubles of
 * device memory): bit for bit what kicp_voxel_downsample (with either "downsample_order") and kicp_preprocess return for the same
 * points, float32 fields widened exactly to double, as packed xyz doubles to `out`, device memory of the context's device aligned to 8
 * bytes for min(cap, n) points.  The host synchronises once and the caller's memory is free to change when they return; `out` is
 * complete then.  *m receives the count; KICP_ERR_CAPACITY when it exceeds cap, with `out` left unwritten.  Errors: KICP_ERR_INVALID
 * as for kicp_map_add_points_device, and for kicp_preprocess_device n_stamps != n with deskew.  Like their host variants (and when
 * they fail) they discard a frame staged by kicp_frame_stage. */
int kicp_voxel_downsample_device(kicp_ctx *ctx, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                 int32_t offset_y, int32_t offset_z, double voxel_size, double *out, int64_t cap, int64_t *m);
int kicp_preprocess_device(kicp_ctx *ctx, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                           int32_t offset_y, int32_t offset_z, const double *stamps, int64_t n_stamps, const double relative_motion[7],
                           const double lidar_to_base[7], double max_range, double min_range, int32_t deskew, double *out, int64_t cap,
                           int64_t *m);

/* ---- whole frame: KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:48-85) as ONE call, the frame staying in HBM
 *      from ingest to map update: ingest (float32/float64 fields at a PointCloud2-style stride, RosUtils.cpp:30-39) ->
 *      Preprocess (de-skew by `deskew_motion` = lidar_to_base^-1 * relative_odometry * lidar_to_base, range filter) ->
 *      transform to base -> VoxelDownsample(0.5 vs) -> VoxelDownsample(1.5 vs) -> ComputeRobotMotion(source, map,
 *      last_pose, relative_odometry, tau) -> map.Update(frame_downsample, new_pose).  The scalar CorrespondenceThreshold
 *      stays with the caller (tau in, pose out).  out_frame / out_source receive the two clouds RegisterFrame returns
 *      (preprocessed frame in base, registration source); either may be NULL to skip its download.  On zero
 *      correspondences the pose is NaN like the reference's, KICP_WARN_NO_CORRESPONDENCES is returned and the map is
 *      left untouched.  The host synchronises with the device ONCE per frame, at its end: the survivor counts of the
 *      filters, the pose and the map's bookkeeping all stay on the device in between (with out_frame / out_source buffers
 *      smaller than in->n points, or option "frame_sync", the counts are read back mid-frame instead, so that
 *      KICP_ERR_CAPACITY can be reported before the map changes). ------------------------------------------------- */
typedef struct kicp_frame_input {
    const void *data;   /* host pointer: n points */
    int64_t n;
    int32_t dtype;      /* KICP_DTYPE_F64 (std::vector<Eigen::Vector3d>) or KICP_DTYPE_F32 (PointCloud2 FLOAT32 fields) */
    int32_t point_step; /* bytes between consecutive points; 0 = tightly packed x,y,z (offsets ignored) */
    int32_t offset_x, offset_y, offset_z; /* byte offsets of the fields inside a point (used when point_step > 0) */
    const double *stamps; /* per-point times in any affine scale (normalised to [0,1] on the device, like          */
    int64_t n_stamps;     /* TimeStampHandler.cpp:129-135 does); 0 = no de-skewing                                 */
} kicp_frame_input;
typedef struct kicp_frame_params {
    double max_range, min_range; /* kiss_icp::Preprocessor, pipeline/KinematicICP.hpp:40-41 */
    int32_t deskew;              /* pipeline::Config::deskew */
    double voxel_size;           /* pipeline::Config::voxel_size: the two down-sample sizes are 0.5x and 1.5x of it */
    int32_t stage_clouds;        /* flags: keep the two clouds in context-owned pinned host memory (KICP_STAGE_* below) */
    kicp_reg_params reg;
} kicp_frame_params;
#define KICP_STAGE_F64 1 /* the two clouds as doubles, read by kicp_frame_clouds (any other bit but KICP_STAGE_F32 means this too) */
#define KICP_STAGE_F32 2 /* the two clouds as float32 records (the rule of kicp_map_pointcloud_f32), read by kicp_frame_clouds_f32 */
int kicp_register_frame(kicp_map *map, const kicp_frame_input *in, const double deskew_motion[7], const double lidar_to_base[7],
                        const double last_pose[7], const double relative_odometry[7], double tau, const kicp_frame_params *fp,
                        double out_pose[7], double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source,
                        int64_t cap_source, int64_t *n_source, kicp_reg_result *result);
/* The two clouds of the last kicp_register_frame on this context (fp->stage_clouds & KICP_STAGE_F64 or out_* given): pointers into
 * context-owned pinned host memory, valid until the next front-end call on the same context.  Lets a caller build its
 * own containers in one pass instead of pre-sizing worst-case output buffers. */
int kicp_frame_clouds(kicp_ctx *ctx, const double **frame, int64_t *n_frame, const double **source, int64_t *n_source);
/* The same two clouds as the float32 records EigenToPointCloud2 builds (fp->stage_clouds & KICP_STAGE_F32): x, y, z at byte offsets
 * 0, 4, 8, point_step 12, each coordinate static_cast<float> as on x86-64, NaN bits included.  They are encoded on the device after
 * the front end and before the registration (one more kernel launch per frame) and 12 bytes per point cross PCIe; the copies, the
 * counts, KICP_ERR_CAPACITY, the NaN-pose rule and the lifetime are kicp_frame_clouds'.  Counts are 0 for a frame without the flag. */
int kicp_frame_clouds_f32(kicp_ctx *ctx, const float **frame, int64_t *n_frame, const float **source, int64_t *n_source);
/* The same two clouds where the frame left them, in context-owned device memory: dtype KICP_DTYPE_F64 gives the preprocessed frame in
 * base and the registration source as packed xyz doubles (no staging flag needed), KICP_DTYPE_F32 the float32 records of
 * kicp_frame_clouds_f32 (frames with KICP_STAGE_F32; counts 0 without it).  Bytes and counts are those kicp_frame_clouds /
 * kicp_frame_clouds_f32 deliver for the same frame.  Valid after a kicp_register_frame / kicp_register_staged_frame that returned
 * KICP_OK or KICP_WARN_NO_CORRESPONDENCES, until the next front-end call on the context (after any other outcome the counts are 0).
 * The frame call has synchronised, so any stream may read them; this call is not a front-end call and discards no staged frame.
 * Errors: KICP_ERR_INVALID for a null argument or another dtype. */
int kicp_frame_clouds_device(kicp_ctx *ctx, int32_t dtype, const void **frame, int64_t *n_frame, const void **source,
                             int64_t *n_source);
/* With option "correspondences" 1: the kicp_corr_stats of the last frame call on the context, its registration source evaluated at the
 * returned pose against the map before that frame's Update.  All counts are 0 (and every field) when the option was off for that frame
 * or the frame failed (any status but KICP_OK and KICP_WARN_NO_CORRESPONDENCES).  Errors: KICP_ERR_INVALID for a null argument,
 * named by kicp_last_error. */
int kicp_frame_correspondences(kicp_ctx *ctx, kicp_corr_stats *stats);
/* The per-point results of that evaluation in context-owned device memory, one row per source point (kicp_frame_clouds_device's
 * source, in its order): points n x 3 doubles, dist n doubles, inlier n bytes.  Lifetime and discard rules are kicp_frame_clouds_device's;
 * *n is 0 when the option was off or the frame failed.  Errors: KICP_ERR_INVALID for a null argument, named by kicp_last_error. */
int kicp_frame_correspondences_device(kicp_ctx *ctx, const double **points, const double **dist, const uint8_t **inlier, int64_t *n);

/* ---- the frame path's map-update policy: whether a frame call (kicp_register_frame, kicp_register_staged_frame, _sensors and the
 *      _segments variants) ends with the reference's Update(frame_downsample, new_pose), decided on the device within the frame's one
 *      host synchronisation.  NEVER registers frames against a map that must not change (a map restored with kicp_map_load_voxels);
 *      GATED inserts only frames whose correspondence report shows that they fit.  The pose, kicp_reg_result, the frame's status, the
 *      two clouds and the report are those of ALWAYS: the policy decides only whether the map changes. --------------------------- */
#define KICP_MAP_UPDATE_ALWAYS 0 /* default: Update after every frame whose registration ended KICP_OK (the reference's behaviour) */
#define KICP_MAP_UPDATE_NEVER 1  /* register against the map as it is: never insert, never evict */
#define KICP_MAP_UPDATE_GATED 2  /* Update only when the frame's correspondence report passes the thresholds below */
typedef struct kicp_map_update_policy {
    int32_t mode;            /* KICP_MAP_UPDATE_* */
    int64_t min_inliers;     /* GATED: n_inliers >= min_inliers (>= 0) */
    double min_fitness;      /* GATED: fitness >= min_fitness (in [0, 1]) */
    double max_inlier_rmse;  /* GATED: inlier_rmse <= max_inlier_rmse (> 0; +inf allowed) */
} kicp_map_update_policy;
/* The policy of every later frame call on the context (default {ALWAYS, 0, 0.0, +inf}); the thresholds are ignored outside GATED.
 * The outcome of a frame, in order: NEVER gives KICP_FRAME_UPDATE_SKIPPED; a registration status other than KICP_OK gives
 * NO_CORRESPONDENCES; ALWAYS gives APPLIED; GATED gives APPLIED when the map held no points when the frame began (else no map could
 * ever be built under a gate: the first frame has fitness 0), or when st.n_inliers >= min_inliers, st.fitness >= min_fitness and
 * st.inlier_rmse <= max_inlier_rmse, where st is the kicp_corr_stats kicp_frame_correspondences returns for that frame, bit for bit;
 * REJECTED otherwise.  GATED evaluates the report even with option "correspondences" 0 (two more launches, and the report is readable
 * as if the option were on) and adds one single-thread gate launch; NEVER drops the map's launches.  With option "frame_sync" 1 (or
 * caller buffers smaller than the frame) the host applies the same rule to the report it has read back.  GATED applies the full Update,
 * eviction included: it protects a live map; a prior map wider than max_distance is kept by NEVER, or by freezing it
 * (kicp_map_freeze), after which ALWAYS and GATED update only the live voxels beside it.
 * Errors: KICP_ERR_INVALID, with kicp_last_error naming the field, for a null argument, a mode outside 0..2, min_inliers < 0, a
 * min_fitness that is NaN or outside [0, 1], or a max_inlier_rmse that is NaN or not > 0; the previous policy is kept. */
int kicp_ctx_set_map_update(kicp_ctx *ctx, const kicp_map_update_policy *policy);
#define KICP_FRAME_UPDATE_APPLIED 0            /* the map was updated with the frame */
#define KICP_FRAME_UPDATE_NO_CORRESPONDENCES 1 /* NaN pose: the map is untouched, as under every policy */
#define KICP_FRAME_UPDATE_REJECTED 2           /* GATED, thresholds not met: the map is untouched */
#define KICP_FRAME_UPDATE_SKIPPED 3            /* NEVER: the map is untouched */
#define KICP_FRAME_UPDATE_NONE 4               /* no frame call yet, the last one failed, or another front-end call came after it */
/* The outcome of the last frame call on the context (KICP_FRAME_UPDATE_*), with the report's lifetime: valid after a frame call that
 * returned KICP_OK or KICP_WARN_NO_CORRESPONDENCES, until the next front-end call.  Not a front-end call.  Errors: KICP_ERR_INVALID for
 * a null argument, named by kicp_last_error. */
int kicp_frame_map_update(kicp_ctx *ctx, int32_t *outcome);
/* Free-space clearing in the frame path (the rule of kicp_map_clear_free_space; default {0.0, 0}: off).  With min_misses >= 1 the
 * single-sensor frame calls (kicp_register_frame, kicp_register_staged_frame, kicp_register_staged_frame_segments) clear the map after
 * an Update whose outcome is KICP_FRAME_UPDATE_APPLIED: the points are frame_downsample (the cloud the Update inserts) in the base frame,
 * the pose is the returned pose and the origin the translation of lidar_to_base.  The rays run against the map after the insert; a
 * voxel the same Update evicts by distance counts as evicted, not cleared.  In the single-synchronisation order this is one memset and
 * two more launches within the frame's one host synchronisation; the read-back order (option "frame_sync" 1, or small caller buffers)
 * calls kicp_map_clear_free_space after its Update and gives the same map.  NEVER, a GATED rejection and a NaN pose leave the map
 * untouched as before.  The multi-sensor calls (kicp_register_staged_sensors[_segments]) fail with KICP_ERR_INVALID while it is on (the
 * down-sampled frame no longer knows which sensor a point came from): they consume the staged frame and leave the map unchanged; such a
 * node calls kicp_map_clear_free_space once per sensor with that sensor's cloud.  Errors: KICP_ERR_INVALID, with kicp_last_error naming
 * the field, for a null argument, an end_margin that is NaN, negative or infinite, or min_misses < 0; the previous setting is kept. */
int kicp_ctx_set_free_space(kicp_ctx *ctx, const kicp_free_space_params *params);
/* The statistics of the last frame call's clearing, with the correspondence report's lifetime: all zero when the option was off, the
 * Update was not applied or the frame failed.  Not a front-end call.  Errors: KICP_ERR_INVALID for a null argument. */
int kicp_frame_free_space(kicp_ctx *ctx, kicp_free_space_stats *stats);

/* ---- the same frame in two steps, for a caller that needs the sweep's time range before it has the relative odometry (the
 *      online server: ProcessTimestamps -> wheel-odometry lookup over [begin, end] -> RegisterFrame,
 *      ros/.../server/LidarOdometryServer.cpp:186-210). ---------------------------------------------------------------- */
/* PointField datatypes of a per-point time field (sensor_msgs/msg/PointField) */
#define KICP_STAMP_NONE 0
#define KICP_STAMP_UINT32 6
#define KICP_STAMP_FLOAT32 7
#define KICP_STAMP_FLOAT64 8
/* Stage a frame: its records are uploaded once and decoded on the device (x, y, z as kicp_register_frame's ingest; with
 * stamp_datatype != KICP_STAMP_NONE also the time field at byte `stamp_offset` of every record, in seconds, with the nanosecond
 * rule of TimeStampHandler.cpp:42-104: a value whose rounded integer part has more than 10 digits is multiplied by 1e-9 — bit
 * for bit what kicp/pointcloud2.hpp extract_timestamps returns).  The host synchronises once and receives
 * stamp_range = {min, max} of the stamps in seconds and *n_stamps = their count (0, with stamp_range = {0, 0}, when the frame
 * has none).  A frame without a time field may carry host stamps in in->stamps (n_stamps == n); their {min, max} is reduced on
 * the device the same way.  The field may sit at any byte offset (no alignment needed) but needs point_step > 0.
 * Errors: KICP_ERR_UNSUPPORTED for any other stamp_datatype; KICP_ERR_INVALID for a field outside point_step, a field with
 * point_step == 0, a field together with host stamps, and everything kicp_register_frame rejects in `in`.
 * The staged frame stays on the context's device until kicp_register_staged_frame consumes it.  Any other front-end call on
 * the context (kicp_register_frame, kicp_preprocess, kicp_voxel_downsample, another kicp_frame_stage or
 * kicp_frame_stage_laser_scan, also a failing one) discards it. */
int kicp_frame_stage(kicp_ctx *ctx, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset, double stamp_range[2],
                     int64_t *n_stamps);
/* kicp_frame_stage for a frame already in GPU memory: in->data (n records) and in->stamps (n_stamps doubles) are device memory of the
 * context's device, read in place by the ingest kernel (packed float64 x,y,z without a time field: one device-to-device copy; host
 * stamps: copied device to device).  Same validation, staging and discard rules, the same staged frame bit for bit, the same kernel
 * launches and one host synchronisation; after it returns the staged frame no longer depends on the caller's memory.  Order the
 * producer first (kicp_ctx_wait_stream).  No alignment is needed.  Errors: those of kicp_frame_stage, and KICP_ERR_INVALID when a
 * pointer is not device memory of the context's device (host memory, page-locked included, or another GPU's); a failing call discards
 * a staged frame as kicp_frame_stage does. */
int kicp_frame_stage_device(kicp_ctx *ctx, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset,
                            double stamp_range[2], int64_t *n_stamps);
/* kicp_register_frame on the staged frame of map's context, same arguments without `in`, same results: the same pose, result
 * block, clouds and map as kicp_register_frame given the same points and stamps (host-decoded by extract_timestamps), the same
 * "frame_sync", KICP_ERR_CAPACITY, kicp_frame_clouds and NaN-pose rules, one host synchronisation.  De-skewing uses the staged
 * stamps when fp->deskew is set and the frame has any.  The call consumes the staged frame whatever it returns; without one it
 * fails with KICP_ERR_INVALID, as it does (consuming the frame) on a frame of several sensors staged by kicp_frame_stage_sensors. */
int kicp_register_staged_frame(kicp_map *map, const double deskew_motion[7], const double lidar_to_base[7], const double last_pose[7],
                               const double relative_odometry[7], double tau, const kicp_frame_params *fp, double out_pose[7],
                               double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source, int64_t cap_source,
                               int64_t *n_source, kicp_reg_result *result);

/* ---- 2D LiDAR: a sensor_msgs/LaserScan staged as the frame laser_geometry's projectLaser(scan, cloud, -1.0,
 *      channel_option::Timestamp) makes of it (the reference's use_2d_lidar, ros/src/kinematic_icp_ros/nodes/online_node.cpp). ---- */
typedef struct kicp_laser_scan { /* sensor_msgs/msg/LaserScan without header and intensities */
    const float *ranges;         /* host pointer, n beams (page-locked is fastest) */
    int64_t n;
    float angle_min, angle_max, angle_increment;
    float time_increment, range_min, range_max;
} kicp_laser_scan;
/* Stage the scan: exactly what kicp_frame_stage stages for projectLaser(scan)'s records (FLOAT32 x, y, z at 0, 4, 8 and a FLOAT32
 * `stamps` field at 12, point_step 16): beam i is kept iff range_min <= ranges[i] < range_max; its point is r * (cos, sin) of
 * angle_min + i * angle_increment narrowed to float, z = 0; its stamp is (float)i * time_increment, decoded as kicp_frame_stage decodes
 * a FLOAT32 time field.  Kept beams stay in beam order.  The ranges cross PCIe once (4 bytes per beam); the projection, the range test,
 * the stamps and the compaction run in one kernel; the host synchronises once.  *n_points receives the kept count (also the stamp
 * count) and stamp_range their {min, max} in seconds ({0, 0} when nothing is kept).  The cos / sin table is the C library's, computed
 * on the host and cached on the context like the projector's: recomputed only when n, angle_min or angle_max differ from the cached
 * scan's (a changed angle_increment alone keeps the old table, as laser_geometry does).  Errors: KICP_ERR_INVALID for a null
 * argument, n < 0 or n > 2^30 - 1, and ranges == NULL with n > 0 (any float values are accepted); KICP_ERR_CAPACITY when the host
 * cannot hold the table.  The staging rules are
 * kicp_frame_stage's: kicp_register_staged_frame consumes the scan, any other front-end call (kicp_frame_stage included) discards it,
 * and a failing call stages nothing. */
int kicp_frame_stage_laser_scan(kicp_ctx *ctx, const kicp_laser_scan *scan, double stamp_range[2], int64_t *n_points);
/* kicp_frame_stage_laser_scan with scan->ranges in device memory of the context's device, 4-byte aligned, read in place by the
 * projection kernel.  The cos / sin table, its cache and key rules, the staging rules and the one host synchronisation are
 * kicp_frame_stage_laser_scan's.  Order the producer first (kicp_ctx_wait_stream).  Errors: those of kicp_frame_stage_laser_scan, and
 * KICP_ERR_INVALID for ranges that are not such memory or misaligned (a failing call discards a staged frame). */
int kicp_frame_stage_laser_scan_device(kicp_ctx *ctx, const kicp_laser_scan *scan, double stamp_range[2], int64_t *n_points);

/* ---- several LiDARs in one frame: K sensors (PointCloud2-style records or LaserScans, host or device memory) staged with one call,
 *      each de-skewed in its own frame with its own motion and extrinsic over one common sweep window, then registered as one frame.
 *      The frame is defined as follows.
 *        1. Common window: T0, T1 = min, max of stamp + time_offset over the stamped points of all sensors.  A stamped point is
 *           normalised as s = (stamp + time_offset - T0) / (T1 - T0).
 *        2. Per-sensor Preprocess: a point of sensor k is de-skewed in sensor k's frame with exp((s - 1) log(deskew_motion_k)),
 *           range-tested there and transformed to base by lidar_to_base_k.  A sensor without stamps is not de-skewed, and
 *           fp->deskew == 0 turns de-skewing off for all sensors.
 *        3. The kept points are concatenated in sensor order, then input order (kept-beam order for a LaserScan); from there the
 *           frame is kicp_register_frame's: both down-samples, registration, map update, the two clouds.
 *      One sensor with time_offset 0 gives bit for bit what kicp_frame_stage (or _laser_scan, or _device) followed by
 *      kicp_register_staged_frame gives. ------------------------------------------------------------------------------------------ */
#define KICP_MAX_SENSORS 8
#define KICP_SENSOR_POINTS 0     /* `points` with stamp_datatype / stamp_offset, as kicp_frame_stage takes them */
#define KICP_SENSOR_LASER_SCAN 1 /* `scan`, as kicp_frame_stage_laser_scan takes it */
typedef struct kicp_sensor_input {
    int32_t kind;                            /* KICP_SENSOR_POINTS or KICP_SENSOR_LASER_SCAN */
    int32_t device;                          /* 0: host memory; 1: device memory of the context's device (the _device rules) */
    kicp_frame_input points;                 /* kind KICP_SENSOR_POINTS */
    int32_t stamp_datatype, stamp_offset;    /* kind KICP_SENSOR_POINTS: kicp_frame_stage's time field */
    kicp_laser_scan scan;                    /* kind KICP_SENSOR_LASER_SCAN */
    double time_offset;                      /* seconds added to every stamp of the sensor: 0 for absolute stamps, the header stamp for
                                                relative ones (a LaserScan's beam times, an Ouster `t`); must be finite */
} kicp_sensor_input;
typedef struct kicp_sensor_stats {
    int64_t n_points;      /* points staged (records, or kept beams) */
    int64_t n_stamps;      /* their stamps (0: the sensor has none) */
    double stamp_range[2]; /* {min, max} of its stamps on the common clock, {0, 0} without stamps */
} kicp_sensor_stats;
/* Stage k sensors (1 <= k <= KICP_MAX_SENSORS): each is ingested on the device at its own place of the staged frame (records by the
 * ingest of kicp_frame_stage, LaserScans by the projection of kicp_frame_stage_laser_scan, whose cos / sin table is cached per sensor
 * index), then one reduction puts the stamps on the common clock and finds the window.  The host synchronises once.  stamp_range
 * receives {T0, T1} ({0, 0} when no sensor has stamps); stats (k entries, may be NULL) the per-sensor counts and ranges.
 * Errors: KICP_ERR_INVALID for k outside [1, KICP_MAX_SENSORS], a null argument, another kind, a non-finite time_offset, more than
 * 2^30 - 1 points in all, and whatever kicp_frame_stage / _device or kicp_frame_stage_laser_scan / _device reject in a sensor (the
 * error text names sensors[i]); KICP_ERR_UNSUPPORTED for a stamp datatype they do not support.  The staging rules are kicp_frame_stage's:
 * any other front-end call discards the staged frame and a failing call stages nothing. */
int kicp_frame_stage_sensors(kicp_ctx *ctx, const kicp_sensor_input *sensors, int32_t k, double stamp_range[2],
                             kicp_sensor_stats *stats);
/* kicp_register_staged_frame for a frame of k sensors: sensor i is de-skewed with deskew_motions[i] (lidar_to_base_i^-1 *
 * relative_odometry * lidar_to_base_i for the reference's rule) and moved to base by lidar_to_bases[i].  A frame staged by
 * kicp_frame_stage or kicp_frame_stage_laser_scan (or their _device variants) is a frame of one sensor with time_offset 0.  Outputs,
 * rules and results are kicp_register_staged_frame's.  The call consumes the staged frame whatever it returns; without one, or with
 * k different from the staged frame's sensor count, it fails with KICP_ERR_INVALID.  kicp_register_staged_frame on a frame of more
 * than one sensor fails with KICP_ERR_INVALID (and consumes it). */
int kicp_register_staged_sensors(kicp_map *map, int32_t k, const double deskew_motions[][7], const double lidar_to_bases[][7],
                                 const double last_pose[7], const double relative_odometry[7], double tau, const kicp_frame_params *fp,
                                 double out_pose[7], double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source,
                                 int64_t cap_source, int64_t *n_source, kicp_reg_result *result);

/* ---- de-skew along sampled odometry: instead of one motion over the sweep, each sensor of a staged frame carries 1 to
 *      KICP_MAX_DESKEW_SEGMENTS contiguous time segments, each with constant velocity, so that a robot that turns or brakes during the
 *      sweep (or during the longer common window of several unsynchronised sensors) is de-skewed along the path its odometry saw.
 *      A segment {t_begin, t_end, motion, to_end}:
 *        - t_begin < t_end are seconds on the staged frame's clock: the clock of stamp_range and kicp_sensor_stats, time offsets added;
 *        - motion is the sensor-frame motion from t_begin to t_end;
 *        - to_end is the sensor-frame motion from t_end to the window end T1: the identity for the segment that ends at T1.
 *      A sensor's segments are contiguous (t_end of one == t_begin of the next, exactly).  For a stamped point at time t, with
 *      fp->deskew set:
 *        1. j = the largest index with t_begin_j <= t.  The segments must cover the common window [T0, T1].
 *        2. u = (t - t_begin_j) / (t_end_j - t_begin_j).
 *        3. p' = to_end_j^-1 * exp((u - 1) log(motion_j)) * p: the point in the sensor frame at t_end_j, then in the frame at T1
 *           (a motion M from a to b takes a point from b's frame to a's, so the de-skew applies exp((s - 1) log M) = M^-1 at s = 0 to
 *           bring an early point forward, and to_end^-1 here).  log and the inverse are taken once per segment on the host; to_end
 *           is skipped when it is exactly {0, 0, 0, 1, 0, 0, 0}.
 *        4. Then the range test on p', the transform by lidar_to_base, and the rest of kicp_register_staged_frame unchanged.
 *      Unstamped sensors, and fp->deskew == 0, are not de-skewed.  The library composes no poses: callers pass sensor-frame segments
 *      (the C++ facade's kicp/deskew_segments.hpp and the Python deskew_segments build them from odometry samples).
 *      One segment [T0, T1] (the doubles stamp_range returned) with motion = deskew_motion and an identity to_end gives bit for bit
 *      what kicp_register_staged_frame / kicp_register_staged_sensors give. ------------------------------------------------------ */
#define KICP_MAX_DESKEW_SEGMENTS 64
typedef struct kicp_deskew_segment {
    double t_begin, t_end; /* seconds on the staged frame's clock, t_begin < t_end */
    double motion[7];      /* sensor-frame motion from t_begin to t_end */
    double to_end[7];      /* sensor-frame motion from t_end to T1 */
} kicp_deskew_segment;
/* kicp_register_staged_frame with the de-skew of n_segments segments; relative_odometry keeps its role in the motion model and the
 * threshold.  Any staging route (records, LaserScans, _device variants) of one sensor.  The staging rules, outputs, frame_sync,
 * KICP_ERR_CAPACITY and a NaN pose are kicp_register_staged_frame's; the call consumes the staged frame whatever it returns.
 * KICP_ERR_INVALID, with kicp_last_error naming the argument, for a null pointer, a segment count outside [1, 64], non-finite times or
 * poses, t_begin >= t_end, a gap or overlap between segments, segments that do not cover [T0, T1] of a stamped frame with de-skew on,
 * no staged frame or one of several sensors.  A failing call leaves the map unchanged. */
int kicp_register_staged_frame_segments(kicp_map *map, int32_t n_segments, const kicp_deskew_segment *segments,
                                        const double lidar_to_base[7], const double last_pose[7], const double relative_odometry[7],
                                        double tau, const kicp_frame_params *fp, double out_pose[7], double *out_frame, int64_t cap_frame,
                                        int64_t *n_frame, double *out_source, int64_t cap_source, int64_t *n_source,
                                        kicp_reg_result *result);
/* kicp_register_staged_sensors with sensor i de-skewed by its n_segments[i] segments at segments[i] (every table covers the common
 * window when the sensor is stamped and de-skew is on); otherwise as kicp_register_staged_frame_segments. */
int kicp_register_staged_sensors_segments(kicp_map *map, int32_t k, const int32_t n_segments[], const kicp_deskew_segment *const segments[],
                                          const double lidar_to_bases[][7], const double last_pose[7], const double relative_odometry[7],
                                          double tau, const kicp_frame_params *fp, double out_pose[7], double *out_frame,
                                          int64_t cap_frame, int64_t *n_frame, double *out_source, int64_t cap_source, int64_t *n_source,
                                          kicp_reg_result *result);

/* ---- multi-GPU: the scan's points shard by contiguous index range, the map is replicated, and each IRLS
 *      iteration ends with one sum-allreduce of the 8 accumulated doubles (SURVEY.md §8(e)). ------------------- */
#define KICP_UNIQUE_ID_BYTES 128
int kicp_comm_unique_id(uint8_t id[KICP_UNIQUE_ID_BYTES]); /* ncclGetUniqueId on rank 0; broadcast it out of band */
int kicp_comm_init(kicp_ctx *ctx, const uint8_t id[KICP_UNIQUE_ID_BYTES], int32_t nranks, int32_t rank);
int kicp_comm_destroy(kicp_ctx *ctx);
/* Fused exchange over NVLink peer memory (preferred over NCCL when available): every rank allocates a mailbox and
 * publishes its CUDA-IPC handle; after kicp_comm_p2p_init the sharded registration runs as ONE persistent kernel per GPU
 * whose grid barrier also writes the 8 partial sums into every peer's mailbox and waits for theirs — no collective
 * kernels, no extra launches.  All ranks must issue the same sequence of sharded registrations. */
#define KICP_IPC_HANDLE_BYTES 64
#define KICP_MAX_RANKS 8
int kicp_comm_p2p_handle(kicp_ctx *ctx, uint8_t handle[KICP_IPC_HANDLE_BYTES]);
int kicp_comm_p2p_init(kicp_ctx *ctx, const uint8_t *handles /* nranks x 64 bytes, rank order */, int32_t nranks, int32_t rank);
/* Every rank calls this with ITS shard (frame_xyz / n are the local range).  All ranks return the same pose. */
int kicp_register_sharded(kicp_map *map, const double *frame_xyz, int64_t n_local, const double last_robot_pose[7],
                          const double relative_wheel_odometry[7], double max_correspondence_distance,
                          const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result);
int kicp_register_points_sharded(kicp_map *map, const void *data, int64_t n_local, int32_t dtype, int32_t point_step, int32_t offset_x,
                                 int32_t offset_y, int32_t offset_z, const double last_robot_pose[7],
                                 const double relative_wheel_odometry[7], double max_correspondence_distance,
                                 const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result);
int kicp_register_scan_sharded_async(kicp_map *map, kicp_scan *scan_shard, const double last_robot_pose[7],
                                     const double relative_wheel_odometry[7], double max_correspondence_distance,
                                     const kicp_reg_params *params, kicp_reg_result *result);

#ifdef __cplusplus
}
#endif
#endif /* KICP_H_ */
