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
/* Options: "persistent" 1 = all IRLS iterations of a registration inside ONE cooperative launch (default), 0 = one launch per
 * iteration; "stats" 1 = count hash probes / candidate points / 128-byte lines on the device (bench.py's touched-bytes figure);
 * "ctas_per_sm" = cap of the resident CTAs per SM the grid is sized for (0 = occupancy limit); "nn_cache" = between IRLS
 * passes every point keeps its two nearest candidates together with a certificate (a lower bound on the distance to every other
 * candidate) and a pass re-searches only the points whose certificate the pose update broke (exact, see DESIGN.md): 1 = for
 * scans of 49152 points or more (default: smaller scans gain nothing from the extra phase), 2 = always, 0 = never; "overlap_upload" 1 = the
 * host-pointer entry points overlap the frame's upload with the first pass (default); "spin_timeout_ms" = bound of every
 * device-side wait (upload flags, peers of the fused exchange; default 20000); "frame_sync" 1 = kicp_register_frame reads the
 * survivor counts back in the middle of a frame (legacy order; default 0 = ONE host synchronisation per frame, at its end).
 * Unknown names fail with KICP_ERR_INVALID.
 * Every setting computes the same result up to the summation order. */
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
/* Voxel-grouped dump: keys[V][3], counts[V], points[total][3] in per-voxel insertion order (tests, checkpoints). */
int kicp_map_export_voxels(kicp_map *map, int32_t *keys, int32_t *counts, double *points, int64_t cap_voxels,
                           int64_t cap_points, int64_t *num_voxels, int64_t *num_points);
/* Bulk load of a voxel-grouped map (replaces the content): the inverse of kicp_map_export_voxels. */
int kicp_map_load_voxels(kicp_map *map, const int32_t *keys, const int32_t *counts, const double *points,
                         int64_t num_voxels);
/* GetClosestNeighbor(query) for n queries: (closest point, distance); (0,0,0), DBL_MAX when nothing is found. */
int kicp_map_nearest(kicp_map *map, const double *queries, int64_t n, double *out_points, double *out_dist);

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

/* ---- front end of KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:38-44,54-59; KISS-ICP v1.2.0) ---------------- */
/* kiss_icp::VoxelDownsample(frame, voxel_size): the first point (input order) of every voxel, in input order. */
int kicp_voxel_downsample(kicp_ctx *ctx, const double *xyz, int64_t n, double voxel_size, double *out_xyz, int64_t cap,
                          int64_t *m);
/* kiss_icp::Preprocessor::Preprocess(frame, timestamps, relative_motion) — de-skew with exp((s-1) log(relative_motion))
 * when `deskew` and stamps are given (n_stamps == n), keep min_range < |p| < max_range — followed by the transform of
 * the survivors by lidar_to_base (KinematicICP.cpp:59).  Pass the identity pose to get Preprocess alone. */
int kicp_preprocess(kicp_ctx *ctx, const double *xyz, int64_t n, const double *stamps, int64_t n_stamps,
                    const double relative_motion[7], const double lidar_to_base[7], double max_range, double min_range,
                    int32_t deskew, double *out_xyz, int64_t cap, int64_t *m);

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
    int32_t stage_clouds;        /* keep the two clouds in context-owned pinned host memory for kicp_frame_clouds() */
    kicp_reg_params reg;
} kicp_frame_params;
int kicp_register_frame(kicp_map *map, const kicp_frame_input *in, const double deskew_motion[7], const double lidar_to_base[7],
                        const double last_pose[7], const double relative_odometry[7], double tau, const kicp_frame_params *fp,
                        double out_pose[7], double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source,
                        int64_t cap_source, int64_t *n_source, kicp_reg_result *result);
/* The two clouds of the last kicp_register_frame on this context (fp->stage_clouds != 0 or out_* given): pointers into
 * context-owned pinned host memory, valid until the next front-end call on the same context.  Lets a caller build its
 * own containers in one pass instead of pre-sizing worst-case output buffers. */
int kicp_frame_clouds(kicp_ctx *ctx, const double **frame, int64_t *n_frame, const double **source, int64_t *n_source);

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
