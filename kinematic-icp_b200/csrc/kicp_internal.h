// Internal definitions shared by the translation units of libkicp_b200.so.  Not installed.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "kicp.h"

#define KICP_SLOT_EMPTY 0xFFFFFFFFu
#define KICP_SLOT_LOCKED 0xFFFFFFFEu
#define KICP_PSTRIDE 4    // doubles per stored map point: {x, y, z, pad} = one 32-byte sector, two 16-byte loads
#define KICP_UPLOAD_CHUNKS 8
#define KICP_MAX_CAP 255  // max_points_per_voxel: the count shares the slot's meta word (low 8 bits)

// ---------------------------------------------------------------------------------------------------------
// HBM layout of the voxel map (kiss_icp::VoxelHashMap on the device)
//
//   slots[nslots]      int4 {kx, ky, kz, meta}   open-addressed, linear probing, nslots = 2^k, load <= 0.25
//                                                meta = (block << 8) | count, 0xFFFFFFFF = empty
//   blk[blocks_cap]    int4 {kx, ky, kz, count}  one header per occupied voxel ("block"), dense [0, num_blocks)
//   pts[blocks_cap * cap * 4] double             block b owns points [b*cap, b*cap + count), insertion order;
//                                                each point is {x, y, z, pad}: exactly one 32-byte sector
//   blocks [0, prior_blocks) are a frozen prior when there is one (kicp_map_freeze): read-only, never evicted, never moved
//
// One 16-byte load resolves a probe to (block, count); a voxel's points are one contiguous <= cap*32 B run.
// ---------------------------------------------------------------------------------------------------------
struct MapView {
    const int4 *slots;
    uint32_t mask;  // nslots - 1
    const double *pts;
    int cap;
    double voxel_size;
};

// Mailbox of the fused cross-GPU exchange (NCCL-LL style): rank r writes its 8 partial sums of pass `it` as sixteen 8-byte
// words {32 data bits | 32-bit tag << 32} into ll[parity][it][r] of EVERY rank's mailbox.  An aligned 8-byte store arrives
// whole, so a word whose tag matches is valid data: no fence, no separate flag.  Tags grow monotonically per registration
// and pass, so nothing is ever cleared; `parity` (registration sequence number & 1) keeps a fast rank from overwriting
// words a slow rank has not read yet.
struct P2PMailbox {
    unsigned long long ll[2][KICP_MAX_ITERATIONS][KICP_MAX_RANKS][16];
};

// Per-launch arguments of the single-pass scans (kicp_scan.cuh): one status word per tile, the ticket counter that hands the tiles
// out, and the number of the launch (never 0) that tells this launch's status words from those of earlier ones.
struct kicp_scan_args {
    unsigned long long *status;
    unsigned int *ticket;
    uint32_t launch;
};

struct RegState;  // device-side state of one registration (kicp_register.cu)

struct kicp_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    int64_t launches = 0;
    // registration options (kicp_ctx_set_option)
    int ctas_per_sm_cap = 0;         // option "ctas_per_sm": 0 = use the occupancy limit
    int persistent = 1;     // 1 = all IRLS iterations inside one cooperative launch, 0 = one launch per iteration
    int collect_stats = 0;  // option "stats": count probes / candidate points / lines on the device
    int spin_timeout_ms = 20000;  // bound of every device-side wait (upload flags, peers of the fused exchange)
    int nn_cache = 1;  // option "nn_cache"
    int frame_sync = 0;       // option "frame_sync": 1 = kicp_register_frame reads the survivor counts back mid-frame (legacy order)
    int downsample_order = 0;  // option "downsample_order": 1 = VoxelDownsample emits the robin_map's bucket order (kicp_frontend.cu)
    int correspondences = 0;   // option "correspondences": 1 = the frame calls evaluate the source at the returned pose (kicp_frontend.cu)
    // kicp_ctx_set_map_update: whether the frame calls end with the map's Update (kicp_frontend.cu)
    kicp_map_update_policy map_update = {KICP_MAP_UPDATE_ALWAYS, 0, 0.0, INFINITY};
    // kicp_ctx_set_free_space: whether the single-sensor frame calls clear free space after their Update (min_misses 0: off)
    kicp_free_space_params free_space = {0.0, 0};
    int overlap_upload = 1;
    // the registration's device state, neighbour cache, upload flags and profiling records (kicp_register_api.cu owns the type)
    struct RegScratch *reg = nullptr;
    cudaStream_t copy_stream = nullptr;   // copies that overlap the registration (the chunked frame upload, the staged clouds)
    cudaEvent_t ev_order = nullptr;       // kicp_ctx_wait_stream / kicp_stream_wait_ctx: recorded on one stream, waited on by the other
    kicp_reg_result *h_result = nullptr;  // pinned bounce buffer for synchronous calls
    // state of the single-pass scans (kicp_scan.cuh; stream-ordered, shared by the front end and the maps of this context)
    unsigned long long *d_scan_status = nullptr;
    unsigned int *d_scan_ticket = nullptr;
    uint32_t scan_tiles_cap = 0, scan_launch = 0;
    // front-end scratch (kicp_frontend.cu owns the type): frame buffers, down-sample hash, pinned staging of the clouds
    void *frontend = nullptr;
    void (*frontend_free)(kicp_ctx *) = nullptr;
    // multi-GPU
    void *nccl_comm = nullptr;
    int nranks = 1, rank = 0;
    struct P2PMailbox *p2p_local = nullptr;      // this rank's mailbox (cudaMalloc, exported through CUDA IPC)
    struct P2PMailbox *p2p_peer[KICP_MAX_RANKS] = {nullptr};  // every rank's mailbox as mapped into this process
    bool p2p_ready = false;
    unsigned long long p2p_seq = 0;              // sharded registrations issued so far (identical on all ranks)
};

struct kicp_map {
    kicp_ctx *ctx = nullptr;
    double voxel_size = 1.0, max_distance = 100.0;
    uint32_t cap = 20;
    int4 *slots = nullptr;
    uint32_t nslots = 0;
    int4 *blk = nullptr;
    double *pts = nullptr;
    int32_t *pend_head = nullptr;  // per block, -1 when idle
    uint32_t blocks_cap = 0;
    uint32_t num_blocks = 0;  // host mirror
    int64_t num_points = 0;   // host mirror
    uint32_t *d_counters = nullptr;  // [0] num_blocks [1] touched [2] overflow [3] points added [4] dead
    // staging for AddPoints
    double *d_in = nullptr, *d_xyz_t = nullptr;
    int32_t *d_next = nullptr, *d_touched = nullptr;
    double *d_dist = nullptr;  // GetClosestNeighbor of host queries: the distances (the points go to d_xyz_t)
    int64_t in_cap = 0;
    // one allocation holds every array above and below (kicp_map.cu, map_alloc_storage)
    void *slab = nullptr;
    size_t slab_bytes = 0;
    uint32_t slots_cap = 0;  // slots allocated (power of two); nslots <= slots_cap are in use
    // scratch of RemovePointsFarFromLocation: survivor flags / new ids, and the spare header+point arrays the
    // survivors are compacted into (swapped with blk/pts afterwards)
    uint32_t *d_keep = nullptr, *d_new_id = nullptr;
    int4 *blk_spare = nullptr;
    double *pts_spare = nullptr;
    // frozen prior (kicp_map_freeze): blocks [0, prior_blocks) never change and never move.  While frozen, blk_spare / pts_spare hold
    // a copy of that prefix (so that the swap after a compaction keeps it), and prior_slots (its own allocation, prior_slots_cap
    // slots) is the table as it holds the prior alone at the current nslots: an eviction restores it and re-inserts the live blocks.
    uint32_t prior_blocks = 0;
    int64_t prior_points = 0;
    int4 *prior_slots = nullptr;
    uint32_t prior_slots_cap = 0;
    // free-space clearing (kicp_map.cu, allocated by the first clearing): the statistics words and, after them, one flag word per block
    // for free_cap blocks (grown with blocks_cap)
    unsigned long long *d_free_stats = nullptr;
    uint32_t *d_free_flags = nullptr;
    uint32_t free_cap = 0;
    // occupancy evidence (kicp_map_set_occupancy; null when off): one allocation (occ_slab) of 2 * occ_cap int32, the evidence of every
    // block and the spare array a compaction writes into (swapped with it like blk / pts; while frozen it holds the prior's prefix too)
    int32_t *occ_slab = nullptr, *d_occ = nullptr, *d_occ_spare = nullptr;
    uint32_t occ_cap = 0;
    kicp_occupancy_params occ = {0, 0, 0, 0};
    // state of kicp_map_pointcloud_f32_live (kicp_map.cu), created by its first call
    struct MapLive *live = nullptr;
    // correspondence report (kicp_map.cu, created by its first use): the per-CTA partials of k_corr_eval for corr_grid CTAs, the
    // statistics k_corr_finish writes, and the inlier flags of host calls (corr_inl_cap bytes)
    double *d_corr_part = nullptr;
    kicp_corr_stats *d_corr_stats = nullptr;
    uint8_t *d_corr_inl = nullptr;
    int64_t corr_inl_cap = 0;
    int corr_grid = 0;
    // scratch of kicp_map_pose_search* (kicp_map.cu, created by its first use, grown on demand)
    struct PoseScratch *pose = nullptr;
    // scratch of kicp_map_align_planar* (kicp_align.cu, created by its first use, grown on demand)
    struct AlignScratch *align = nullptr;
    MapView view() const { return MapView{slots, nslots - 1, pts, (int)cap, voxel_size}; }
};

// A frame resident in HBM exactly as the caller holds it: float64 or float32 x,y,z fields at a byte stride
// (std::vector<Eigen::Vector3d> = {F64, 24, 0, 8, 16}; a PointCloud2 message = F32 at point_step with its field offsets,
// ros/src/kinematic_icp_ros/utils/RosUtils.cpp:30-39).  The registration kernel widens float32 while it reads.
struct kicp_scan {
    kicp_ctx *ctx = nullptr;
    void *d_data = nullptr;
    int64_t cap_bytes = 0, n = 0;
    const int *d_n = nullptr;  // optional device-resident point count (frames compacted on the device); n is then an upper bound
    int dtype = KICP_DTYPE_F64, stride = 24, ox = 0, oy = 8, oz = 16;
    const void *d_attached = nullptr;  // the caller's device memory (kicp_scan_attach_device), read in place until the next upload
    const void *data() const { return d_attached ? d_attached : d_data; }
};

// error plumbing ------------------------------------------------------------------------------------------
void kicp_set_error(const std::string &msg);
int kicp_cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define KICP_CUDA(call)                                                       \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) return kicp_cuda_fail(e__, #call, __FILE__, __LINE__); \
    } while (0)

#define KICP_CHECK_LAUNCH(ctx)                                                \
    do {                                                                      \
        (ctx)->launches++;                                                    \
        cudaError_t e__ = cudaGetLastError();                                 \
        if (e__ != cudaSuccess) return kicp_cuda_fail(e__, "kernel launch", __FILE__, __LINE__); \
    } while (0)

#define KICP_TRY(call)                 \
    do {                               \
        int s__ = (call);              \
        if (s__ != KICP_OK) return s__; \
    } while (0)

// defined in kicp_map.cu: KICP_OK when [p, p + bytes) is device (or managed) memory of the context's device and p is aligned to
// `align`; otherwise KICP_ERR_INVALID with kicp_last_error naming `what` (host memory, page-locked included, and another GPU's memory)
int kicp_check_device_range(const kicp_ctx *c, const void *p, size_t bytes, size_t align, const char *what);
// defined in kicp_map.cu: arguments of the next scan launch over `items` items on the context stream (grows the status array when
// it has to — synchronising — and numbers the launch)
int kicp_scan_next(kicp_ctx *c, int64_t items, kicp_scan_args *out);
// defined in kicp_map.cu, used by the registration entry points
int kicp_scan_reserve_bytes(kicp_scan *scan, int64_t bytes);
// dtype / point_step / field offsets as in kicp_frame_input (point_step 0 = tightly packed x,y,z); fields must be aligned
int kicp_scan_set_layout(kicp_scan *scan, int32_t dtype, int32_t point_step, int32_t ox, int32_t oy, int32_t oz);
// VoxelHashMap::Update(points, pose) with `d_xyz` already resident in HBM (packed xyz doubles): used by kicp_register_frame
int kicp_map_update_pose_packed(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7]);
// defined in kicp_align.cu: frees the map's alignment scratch (kicp_map_destroy)
void kicp_align_scratch_free(kicp_map *m);
// defined in kicp_map.cu: KICP_ERR_INVALID, with kicp_last_error "fn: why"
int kicp_invalid(const char *fn, const char *why);
// defined in kicp_frontend.cu: the checks of a device cloud in kicp_frame_input's layout (kicp_*_device) that need no device: n, data,
// dtype, point_step and the field offsets; the error text (`fn` names the call) names the condition that failed
int kicp_check_cloud_args(const kicp_frame_input *in, const char *fn);
// the same, then the device range of its records at both ends; *packed (optional): packed float64, readable in place
int kicp_check_device_cloud(kicp_ctx *c, const kicp_frame_input *in, const char *fn, bool *packed);
// defined in kicp_frontend.cu: k_ingest of such a checked cloud of n > 0 points into packed doubles at dst, on the context stream
int kicp_enqueue_widen(kicp_ctx *c, const kicp_frame_input *in, double *dst);
// the same with the point count and the pose still on the device (no read-back; kicp_map.cu).  `fs` (optional): free-space clearing of
// the frame's rays from `fs_origin` (in the cloud's frame) after the insert, its statistics copied to `h_fs` (pinned) on the stream
int kicp_map_update_pose_async(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const kicp_reg_result *d_res,
                               uint32_t *h_counters, const kicp_free_space_params *fs = nullptr, const double fs_origin[3] = nullptr,
                               kicp_free_space_stats *h_fs = nullptr);
// kicp_map_clear_free_space with `d_xyz` already resident in HBM (packed xyz doubles) and checked arguments: used by the read-back
// order of the frame calls
int kicp_map_clear_free_space_packed(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7], const double origin[3],
                                     const kicp_free_space_params *p, kicp_free_space_stats *stats);
// the checks of kicp_free_space_params (`allow_off`: min_misses 0, the frame path's "off", passes), KICP_ERR_INVALID naming the field
int kicp_check_free_space_params(const char *fn, const kicp_free_space_params *p, bool allow_off);
// the host mirrors from the counters an update copied back (`evict_only`: those of RemovePointsFarFromLocation alone)
int kicp_map_finish_update(kicp_map *m, const uint32_t *ctr, bool evict_only);
// device address of the result block the last enqueued registration on this context writes (kicp_register_api.cu)
const kicp_reg_result *kicp_device_result(kicp_ctx *c);
// defined in kicp_register_api.cu: enqueue one registration of n device-resident points on the context stream; the result
// lands in ctx->h_result (pinned) once the stream has drained
// (`d_n`, optional: device-resident point count written earlier on the same stream; n_max is then the upper bound, and the
// grid is planned for `n_hint` points, the count the producer expects, when that is smaller; 0 = no hint)
int kicp_enqueue_registration_device(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double last[7],
                                     const double odom[7], double tau, const kicp_reg_params *p, int64_t n_hint);
// defined in kicp_map.cu: the correspondence report of n_max device points (packed doubles) at `pose7` (host) or at the pose of the
// result block `d_res`, the count min(*d_n, n_max) when d_n is given; per-point outputs may be null; the statistics are copied to
// `stats` (device or page-locked host memory; may be null).  Two launches on the context stream, no host synchronisation.
int kicp_map_enqueue_correspondences(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double *pose7,
                                     const kicp_reg_result *d_res, double tau, double *d_points, double *d_dist, uint8_t *d_inlier,
                                     kicp_corr_stats *stats);
// creates / frees the registration's scratch (kicp_ctx::reg) with the context (kicp_register_api.cu)
int kicp_reg_scratch_create(kicp_ctx *c);
void kicp_reg_scratch_free(kicp_ctx *c);
// defined in kicp_comm.cu
int kicp_comm_allreduce8(kicp_ctx *ctx, double *d_buf);
