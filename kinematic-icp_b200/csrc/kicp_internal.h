// Internal definitions shared by the translation units of libkicp_b200.so.  Not installed.
#pragma once
#include <cuda_runtime.h>
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

struct kicp_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    int64_t launches = 0;
    // registration scratch
    struct RegState *d_state = nullptr;
    double *d_partials = nullptr;  // per-CTA partial sums of the registration kernel [2][grid][8]
    int pruned_ctas_per_sm = 1;      // resident CTAs per SM of k_register<false> (occupancy query)
    int persistent_ctas_per_sm = 1;  // ... of k_register<true>
    int ctas_per_sm_cap = 0;         // option "ctas_per_sm": 0 = use the occupancy limit
    int persistent = 1;     // 1 = all IRLS iterations inside one cooperative launch, 0 = one launch per iteration
    int collect_stats = 0;  // option "stats": count probes / candidate points / lines on the device
    int spin_timeout_ms = 20000;  // bound of every device-side wait (upload flags, peers of the fused exchange)
    // nearest-neighbour cache of the persistent kernel (one entry per scan point, carried from pass to pass)
    unsigned int *d_nn_g = nullptr, *d_nn_g2 = nullptr, *d_todo = nullptr;
    float *d_nn_l = nullptr, *d_nn_seed = nullptr;
    int64_t nn_cap = 0;
    int nn_cache = 1;  // option "nn_cache"
    int frame_sync = 0;       // option "frame_sync": 1 = kicp_register_frame reads the survivor counts back mid-frame (legacy order)
    int64_t reg_n_hint = 0;   // expected point count of the next registration whose exact count lives on the device (0 = none)
    kicp_scan *upload_scan = nullptr;  // staging scan used by the host-pointer entry points
    // chunked upload overlapped with the first IRLS iteration (host-pointer entry points, persistent kernel)
    cudaStream_t copy_stream = nullptr;
    uint32_t *d_chunk_flags = nullptr;   // [KICP_UPLOAD_CHUNKS] raised (to the upload sequence number) chunk by chunk
    uint32_t *h_chunk_tags = nullptr;    // pinned source of the flag copies
    uint32_t upload_seq = 0;
    int overlap_upload = 1;
    kicp_reg_result *h_result = nullptr;  // pinned bounce buffer for synchronous calls
    // profiling (kicp_ctx_profile_begin/end): event pairs per registration
    bool profiling = false;
    struct ProfReg {
        cudaEvent_t prep0, prep1;
        std::vector<cudaEvent_t> it;  // 2 per association launch
        bool persistent = false;      // one launch covers every iteration
        int32_t *d_iters;             // device word receiving the registration's iteration count
    };
    std::vector<ProfReg> prof;
    int32_t *d_prof_iters = nullptr;
    int64_t prof_cap = 0;
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

// defined in kicp_map.cu: arguments of the next scan launch over `items` items on the context stream (grows the status array when
// it has to — synchronising — and numbers the launch)
int kicp_scan_next(kicp_ctx *c, int64_t items, kicp_scan_args *out);
// defined in kicp_map.cu, used by the registration entry points
int kicp_scan_reserve_bytes(kicp_scan *scan, int64_t bytes);
// dtype / point_step / field offsets as in kicp_frame_input (point_step 0 = tightly packed x,y,z); fields must be aligned
int kicp_scan_set_layout(kicp_scan *scan, int32_t dtype, int32_t point_step, int32_t ox, int32_t oy, int32_t oz);
// VoxelHashMap::Update(points, pose) with `d_xyz` already resident in HBM (packed xyz doubles): used by kicp_register_frame
int kicp_map_update_pose_device(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7]);
// the same with the point count and the pose still on the device (no read-back; kicp_map.cu)
int kicp_map_update_pose_async(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const kicp_reg_result *d_res,
                               uint32_t *h_counters);
int kicp_map_finish_update(kicp_map *m, const uint32_t *h_counters);
// device address of the result block the last enqueued registration on this context writes (kicp_register_api.cu)
const kicp_reg_result *kicp_device_result(kicp_ctx *c);
// defined in kicp_register.cu: enqueue one registration of n device-resident points on the context stream; the result
// lands in ctx->h_result (pinned) once the stream has drained
// (`d_n`, optional: device-resident point count written earlier on the same stream; n_max is then the upper bound)
int kicp_enqueue_registration_device(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double last[7],
                                     const double odom[7], double tau, const kicp_reg_params *p);
// defined in kicp_comm.cu
int kicp_comm_allreduce8(kicp_ctx *ctx, double *d_buf);
