// kiss_icp::VoxelHashMap resident in HBM: context, storage management, AddPoints / RemovePointsFarFromLocation /
// Update / Pointcloud / GetClosestNeighbor.  (KISS-ICP v1.2.0 core/VoxelHashMap.{hpp,cpp}; reference call sites
// pipeline/KinematicICP.hpp:79,88,92, pipeline/KinematicICP.cpp:79, registration/Registration.cpp:74,157.)
//
// This translation unit is compiled with -fmad=false: every decision (voxel floor, the < map_resolution spacing
// test, the >= max_distance^2 eviction test, the nearest-neighbour argmin) is evaluated in plain IEEE double
// arithmetic in the same operation order as the reference, so the device map is bit-identical to the CPU one.
#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "kicp_device.cuh"

using namespace kicp_dev;

// ---------------------------------------------------------------------------------------------- error plumbing
static thread_local std::string g_last_error;
void kicp_set_error(const std::string &msg) { g_last_error = msg; }
int kicp_cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
    char buf[512];
    snprintf(buf, sizeof(buf), "CUDA error %d (%s) in %s at %s:%d", (int)e, cudaGetErrorString(e), what, file, line);
    g_last_error = buf;
    cudaGetLastError();  // clear the sticky-free error state
    return KICP_ERR_CUDA;
}
extern "C" const char *kicp_last_error(void) { return g_last_error.c_str(); }
extern "C" const char *kicp_status_string(int s) {
    switch (s) {
        case KICP_OK: return "ok";
        case KICP_ERR_CUDA: return "CUDA error";
        case KICP_ERR_INVALID: return "invalid argument";
        case KICP_ERR_UNSUPPORTED: return "unsupported configuration";
        case KICP_ERR_NCCL: return "NCCL error";
        case KICP_ERR_CAPACITY: return "capacity exceeded";
        case KICP_WARN_NO_CORRESPONDENCES: return "no correspondences (pose is NaN, as in the reference)";
        default: return "unknown status";
    }
}

// ---------------------------------------------------------------------------------------------------- context
extern "C" int kicp_ctx_create(int device, kicp_ctx **out) {
    if (!out) return KICP_ERR_INVALID;
    int count = 0;
    KICP_CUDA(cudaGetDeviceCount(&count));
    if (device < 0 || device >= count) {
        kicp_set_error("kicp_ctx_create: no such CUDA device (this library has no CPU fallback)");
        return KICP_ERR_CUDA;
    }
    KICP_CUDA(cudaSetDevice(device));
    kicp_ctx *c = new kicp_ctx();
    c->device = device;
    cudaDeviceProp prop;
    KICP_CUDA(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    KICP_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    KICP_CUDA(cudaMallocHost(&c->h_result, sizeof(kicp_reg_result)));
    KICP_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    KICP_CUDA(cudaMalloc(&c->d_chunk_flags, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    KICP_CUDA(cudaMemset(c->d_chunk_flags, 0, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    KICP_CUDA(cudaMallocHost(&c->h_chunk_tags, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    if (const char *e = getenv("KICP_OVERLAP_UPLOAD")) c->overlap_upload = atoi(e) ? 1 : 0;
    if (const char *e = getenv("KICP_PERSISTENT")) c->persistent = atoi(e) ? 1 : 0;
    if (const char *e = getenv("KICP_CTAS_PER_SM")) c->ctas_per_sm_cap = std::min(16, std::max(0, atoi(e)));
    if (const char *e = getenv("KICP_SPIN_TIMEOUT_MS")) c->spin_timeout_ms = std::max(1, atoi(e));
    if (const char *e = getenv("KICP_FRAME_SYNC")) c->frame_sync = atoi(e) ? 1 : 0;
    *out = c;
    return KICP_OK;
}

extern "C" int kicp_ctx_synchronize(kicp_ctx *ctx) {
    if (!ctx) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(ctx->stream));
    return KICP_OK;
}
extern "C" void *kicp_ctx_stream(kicp_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }
extern "C" int64_t kicp_ctx_launch_count(kicp_ctx *ctx) { return ctx ? ctx->launches : 0; }

extern "C" int kicp_host_alloc(uint64_t bytes, void **out) {
    if (!out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaMallocHost(out, bytes));
    return KICP_OK;
}
extern "C" int kicp_host_free(void *p) {
    KICP_CUDA(cudaFreeHost(p));
    return KICP_OK;
}

// ------------------------------------------------------------------------------------------------------ scans
int kicp_scan_reserve_bytes(kicp_scan *s, int64_t bytes) {
    if (bytes <= s->cap_bytes) return KICP_OK;
    KICP_CUDA(cudaSetDevice(s->ctx->device));
    KICP_CUDA(cudaStreamSynchronize(s->ctx->stream));
    if (s->d_data) KICP_CUDA(cudaFree(s->d_data));
    s->d_data = nullptr, s->cap_bytes = 0;
    const int64_t cap = std::max<int64_t>(bytes + bytes / 4, 32768);
    KICP_CUDA(cudaMalloc(&s->d_data, (size_t)cap));
    s->cap_bytes = cap;
    return KICP_OK;
}
int kicp_scan_set_layout(kicp_scan *s, int32_t dtype, int32_t point_step, int32_t ox, int32_t oy, int32_t oz) {
    if (dtype != KICP_DTYPE_F64 && dtype != KICP_DTYPE_F32) return KICP_ERR_INVALID;
    const int w = dtype == KICP_DTYPE_F32 ? 4 : 8;
    if (point_step == 0) point_step = 3 * w, ox = 0, oy = w, oz = 2 * w;
    // the registration kernel reads the fields with aligned loads (a PointCloud2 message keeps its fields aligned)
    if (point_step < 3 * w || point_step % w || ox < 0 || oy < 0 || oz < 0 || ox % w || oy % w || oz % w || ox + w > point_step ||
        oy + w > point_step || oz + w > point_step) {
        kicp_set_error("scan layout: point_step / field offsets must be multiples of the field width and lie inside the point");
        return KICP_ERR_INVALID;
    }
    s->dtype = dtype, s->stride = point_step, s->ox = ox, s->oy = oy, s->oz = oz;
    return KICP_OK;
}
extern "C" int kicp_scan_create(kicp_ctx *ctx, int64_t capacity, kicp_scan **out) {
    if (!ctx || !out || capacity < 0) return KICP_ERR_INVALID;
    kicp_scan *s = new kicp_scan();
    s->ctx = ctx;
    int st = kicp_scan_reserve_bytes(s, capacity * 24);
    if (st != KICP_OK) {
        delete s;
        return st;
    }
    *out = s;
    return KICP_OK;
}
extern "C" int kicp_scan_destroy(kicp_scan *s) {
    if (!s) return KICP_OK;
    cudaSetDevice(s->ctx->device);
    cudaStreamSynchronize(s->ctx->stream);
    cudaFree(s->d_data);
    delete s;
    return KICP_OK;
}
extern "C" int kicp_scan_upload_points_async(kicp_scan *s, const void *data, int64_t n, int32_t dtype, int32_t point_step,
                                             int32_t offset_x, int32_t offset_y, int32_t offset_z) {
    if (!s || n < 0 || (n > 0 && !data)) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(s->ctx->device));
    KICP_TRY(kicp_scan_set_layout(s, dtype, point_step, offset_x, offset_y, offset_z));
    KICP_TRY(kicp_scan_reserve_bytes(s, n * (int64_t)s->stride));
    if (n > 0) KICP_CUDA(cudaMemcpyAsync(s->d_data, data, (size_t)(n * s->stride), cudaMemcpyHostToDevice, s->ctx->stream));
    s->n = n, s->d_n = nullptr;
    return KICP_OK;
}
extern "C" int kicp_scan_upload_points(kicp_scan *s, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                       int32_t offset_y, int32_t offset_z) {
    KICP_TRY(kicp_scan_upload_points_async(s, data, n, dtype, point_step, offset_x, offset_y, offset_z));
    KICP_CUDA(cudaStreamSynchronize(s->ctx->stream));
    return KICP_OK;
}
extern "C" int kicp_scan_upload_async(kicp_scan *s, const double *xyz, int64_t n) {
    return kicp_scan_upload_points_async(s, xyz, n, KICP_DTYPE_F64, 0, 0, 0, 0);
}
extern "C" int kicp_scan_upload(kicp_scan *s, const double *xyz, int64_t n) {
    return kicp_scan_upload_points(s, xyz, n, KICP_DTYPE_F64, 0, 0, 0, 0);
}

extern "C" int kicp_ctx_destroy(kicp_ctx *ctx) {
    if (!ctx) return KICP_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    kicp_comm_destroy(ctx);
    if (ctx->frontend_free) ctx->frontend_free(ctx);
    if (ctx->upload_scan) kicp_scan_destroy(ctx->upload_scan);
    cudaFree(ctx->d_state);
    cudaFree(ctx->d_partials);
    cudaFree(ctx->d_nn_g);
    cudaFree(ctx->d_nn_g2);
    cudaFree(ctx->d_nn_l);
    cudaFree(ctx->d_nn_seed);
    cudaFree(ctx->d_todo);
    cudaFree(ctx->d_prof_iters);
    cudaFree(ctx->d_scan_status);
    cudaFree(ctx->d_scan_ticket);
    cudaFreeHost(ctx->h_result);
    cudaFreeHost(ctx->h_chunk_tags);
    cudaFree(ctx->d_chunk_flags);
    if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream), cudaStreamDestroy(ctx->copy_stream);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return KICP_OK;
}

#include "kicp_map_kernels.cuh"  // struct MapRW and every kernel of this file

// Arguments of the next scan launch over `items` items on the context stream.  The status array grows with the largest launch seen
// (rarely, synchronising); launches are numbered from 1, and should the 32-bit number ever wrap the array is cleared first, so that
// a word of an earlier launch can never pass for one of this launch.
int kicp_scan_next(kicp_ctx *c, int64_t items, kicp_scan_args *out) {
    if (!c || !out || items < 0 || items >= (1ll << 30)) return KICP_ERR_INVALID;
    const uint32_t tiles = (uint32_t)((items + kicp_dev::kScanTile - 1) / kicp_dev::kScanTile) + 1;
    if (tiles > c->scan_tiles_cap) {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(c->d_scan_status);
        c->d_scan_status = nullptr, c->scan_tiles_cap = 0;
        const uint32_t cap = std::max<uint32_t>(tiles + tiles / 2, 1024u);
        KICP_CUDA(cudaMalloc(&c->d_scan_status, (size_t)cap * sizeof(unsigned long long)));
        KICP_CUDA(cudaMemsetAsync(c->d_scan_status, 0, (size_t)cap * sizeof(unsigned long long), c->stream));
        c->scan_tiles_cap = cap, c->scan_launch = 0;
    }
    if (!c->d_scan_ticket) {
        KICP_CUDA(cudaMalloc(&c->d_scan_ticket, sizeof(unsigned int)));
        KICP_CUDA(cudaMemsetAsync(c->d_scan_ticket, 0, sizeof(unsigned int), c->stream));
    }
    if (++c->scan_launch == 0) {
        KICP_CUDA(cudaMemsetAsync(c->d_scan_status, 0, (size_t)c->scan_tiles_cap * sizeof(unsigned long long), c->stream));
        c->scan_launch = 1;
    }
    out->status = c->d_scan_status, out->ticket = c->d_scan_ticket, out->launch = c->scan_launch;
    return KICP_OK;
}

// out[i] = in[0] + ... + in[i-1], i < n, on the context stream (renumbering of the surviving blocks, first point of every block)
static int enqueue_exclusive_sum(kicp_ctx *c, const uint32_t *in, uint32_t *out, uint32_t n) {
    if (n == 0) return KICP_OK;
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n, &sa));
    k_exclusive_sum<<<(n + kicp_dev::kScanTile - 1) / kicp_dev::kScanTile, kicp_dev::kScanThreads, 0, c->stream>>>(in, out, n, sa);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// -------------------------------------------------------------------------------------------- host-side storage
static uint32_t next_pow2(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return (uint32_t)p;
}

// (Re)build the open-addressed table over the first `nslots` slots of the slab's table region (nslots <= slots_cap)
static int map_rebuild_table(kicp_map *m, uint32_t nslots) {
    kicp_ctx *c = m->ctx;
    if (nslots > m->slots_cap) {
        kicp_set_error("voxel map: internal error, table larger than its slab region");
        return KICP_ERR_CAPACITY;
    }
    m->nslots = nslots;
    KICP_CUDA(cudaMemsetAsync(m->slots, 0xFF, (size_t)m->nslots * sizeof(int4), c->stream));
    if (m->num_blocks) {
        k_table_rebuild<<<(m->num_blocks + 255) / 256, 256, 0, c->stream>>>(m->slots, m->nslots - 1, m->blk, m->num_blocks);
        KICP_CHECK_LAUNCH(c);
    }
    return KICP_OK;
}

// All of a map's device storage is ONE allocation (the slab), carved into the arrays below for a capacity of `ncap` voxels.
// Steady-state frames therefore never call cudaMalloc/cudaFree (a growth event costs far more than a steady-state Update);
// growth doubles the capacity and migrates the contents.
static int map_alloc_storage(kicp_map *m, uint32_t ncap) {
    kicp_ctx *c = m->ctx;
    const uint32_t slots_cap = std::max<uint32_t>(next_pow2((uint64_t)ncap * 4), 1024u);
    const size_t pts_bytes = (size_t)ncap * m->cap * KICP_PSTRIDE * sizeof(double);
    size_t off = 0;
    auto carve = [&off](size_t bytes) {
        const size_t at = off;
        off += (bytes + 255) & ~(size_t)255;
        return at;
    };
    const size_t o_blk = carve((size_t)ncap * sizeof(int4)), o_pts = carve(pts_bytes), o_head = carve((size_t)ncap * sizeof(int32_t));
    const size_t o_blk2 = carve((size_t)ncap * sizeof(int4)), o_pts2 = carve(pts_bytes);
    const size_t o_keep = carve((size_t)ncap * sizeof(uint32_t)), o_id = carve((size_t)ncap * sizeof(uint32_t));
    const size_t o_slots = carve((size_t)slots_cap * sizeof(int4));
    char *slab = nullptr;
    KICP_CUDA(cudaMalloc(&slab, off));
    int4 *nblk = reinterpret_cast<int4 *>(slab + o_blk);
    double *npts = reinterpret_cast<double *>(slab + o_pts);
    int32_t *nhead = reinterpret_cast<int32_t *>(slab + o_head);
    if (m->num_blocks) {
        KICP_CUDA(cudaMemcpyAsync(nblk, m->blk, (size_t)m->num_blocks * sizeof(int4), cudaMemcpyDeviceToDevice, c->stream));
        KICP_CUDA(cudaMemcpyAsync(npts, m->pts, (size_t)m->num_blocks * m->cap * KICP_PSTRIDE * sizeof(double), cudaMemcpyDeviceToDevice,
                                  c->stream));
    }
    k_fill_i32<<<(ncap + 255) / 256, 256, 0, c->stream>>>(nhead, -1, ncap);
    KICP_CHECK_LAUNCH(c);
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    cudaFree(m->slab);
    m->slab = slab, m->slab_bytes = off;
    m->blk = nblk, m->pts = npts, m->pend_head = nhead, m->blocks_cap = ncap;
    m->blk_spare = reinterpret_cast<int4 *>(slab + o_blk2), m->pts_spare = reinterpret_cast<double *>(slab + o_pts2);
    m->d_keep = reinterpret_cast<uint32_t *>(slab + o_keep), m->d_new_id = reinterpret_cast<uint32_t *>(slab + o_id);
    m->slots = reinterpret_cast<int4 *>(slab + o_slots), m->slots_cap = slots_cap;
    // the table moved with the slab: rebuild it at its previous size (or the minimum for a new map)
    return map_rebuild_table(m, std::max<uint32_t>(std::min(m->nslots, slots_cap), 1024u));
}

// make room for `extra` more voxels (blocks) and keep the table load factor <= 0.25
static int map_reserve(kicp_map *m, uint64_t extra) {
    const uint64_t need = (uint64_t)m->num_blocks + extra;
    if (need >= (1ull << 24)) {
        kicp_set_error("voxel map: more than 2^24 voxels");
        return KICP_ERR_CAPACITY;
    }
    if (need > m->blocks_cap) {
        const uint64_t grown = std::max<uint64_t>(std::max<uint64_t>(2ull * m->blocks_cap, need + need / 2), 4096);
        KICP_TRY(map_alloc_storage(m, (uint32_t)std::min<uint64_t>(grown, 1ull << 24)));
    }
    const uint32_t want_slots = std::max<uint32_t>(next_pow2(need * 4), 1024u);
    if (want_slots > m->nslots) KICP_TRY(map_rebuild_table(m, want_slots));
    return KICP_OK;
}

extern "C" int kicp_map_reserve(kicp_map *m, int64_t voxels) {
    if (!m || voxels < 0 || voxels >= (1ll << 24)) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    if ((uint64_t)voxels > m->blocks_cap) KICP_TRY(map_alloc_storage(m, (uint32_t)voxels));
    return KICP_OK;
}

static int map_reserve_input(kicp_map *m, int64_t n) {
    if (n <= m->in_cap) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    cudaFree(m->d_in), cudaFree(m->d_xyz_t), cudaFree(m->d_next), cudaFree(m->d_touched);
    m->d_in = m->d_xyz_t = nullptr, m->d_next = m->d_touched = nullptr;
    const int64_t cap = std::max<int64_t>(n + n / 4, 4096);
    KICP_CUDA(cudaMalloc(&m->d_in, (size_t)cap * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&m->d_xyz_t, (size_t)cap * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&m->d_next, (size_t)cap * sizeof(int32_t)));
    KICP_CUDA(cudaMalloc(&m->d_touched, (size_t)cap * sizeof(int32_t)));
    m->in_cap = cap;
    return KICP_OK;
}

extern "C" int kicp_map_create(kicp_ctx *ctx, double voxel_size, double max_distance, uint32_t max_points_per_voxel,
                               kicp_map **out) {
    if (!ctx || !out || !(voxel_size > 0.0) || max_points_per_voxel == 0) return KICP_ERR_INVALID;
    if (max_points_per_voxel > KICP_MAX_CAP) {
        kicp_set_error("max_points_per_voxel > 255 is not supported (the count shares the slot's meta word)");
        return KICP_ERR_UNSUPPORTED;
    }
    KICP_CUDA(cudaSetDevice(ctx->device));
    kicp_map *m = new kicp_map();
    m->ctx = ctx;
    m->voxel_size = voxel_size, m->max_distance = max_distance, m->cap = max_points_per_voxel;
    cudaError_t e = cudaMalloc(&m->d_counters, 8 * sizeof(uint32_t));
    if (e != cudaSuccess) {
        delete m;
        return kicp_cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
    }
    // Initial capacity: a local map is a disc of roughly pi (max_distance / voxel_size)^2 columns, a handful of voxels each.  Sized
    // generously (HBM is 180 GB; a voxel of capacity costs ~1.4 KB at 20 points) so that a drive never re-allocates;
    // KICP_MAP_VOXELS overrides, kicp_map_reserve() raises it, growth by doubling remains as the fallback.
    double guess = 8.0 * 3.141592653589793 * (max_distance / voxel_size) * (max_distance / voxel_size);
    if (const char *e = getenv("KICP_MAP_VOXELS")) guess = atof(e);
    if (!(guess >= 16384.0)) guess = 16384.0;
    if (guess > 1048576.0) guess = 1048576.0;
    int st = map_alloc_storage(m, (uint32_t)guess);
    if (st != KICP_OK) {
        kicp_map_destroy(m);
        return st;
    }
    *out = m;
    return KICP_OK;
}

extern "C" int kicp_map_destroy(kicp_map *m) {
    if (!m) return KICP_OK;
    cudaSetDevice(m->ctx->device);
    cudaStreamSynchronize(m->ctx->stream);
    cudaFree(m->slab), cudaFree(m->d_counters);
    cudaFree(m->d_in), cudaFree(m->d_xyz_t), cudaFree(m->d_next), cudaFree(m->d_touched);
    delete m;
    return KICP_OK;
}

extern "C" int kicp_map_clear(kicp_map *m) {
    if (!m) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    m->num_blocks = 0, m->num_points = 0;
    KICP_CUDA(cudaMemsetAsync(m->slots, 0xFF, (size_t)m->nslots * sizeof(int4), m->ctx->stream));
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    return KICP_OK;
}
extern "C" int kicp_map_empty(kicp_map *m, int32_t *empty) {
    if (!m || !empty) return KICP_ERR_INVALID;
    *empty = m->num_blocks == 0;
    return KICP_OK;
}
extern "C" int kicp_map_num_points(kicp_map *m, int64_t *n) {
    if (!m || !n) return KICP_ERR_INVALID;
    *n = m->num_points;
    return KICP_OK;
}
extern "C" int kicp_map_num_voxels(kicp_map *m, int64_t *n) {
    if (!m || !n) return KICP_ERR_INVALID;
    *n = m->num_blocks;
    return KICP_OK;
}

// `src_on_device`: xyz is a device pointer (packed doubles) that stays valid until the stream drains
static int map_add_points_impl(kicp_map *m, const double *xyz, int64_t n, const double *pose7, bool src_on_device = false) {
    if (!m || n < 0 || (n > 0 && !xyz)) return KICP_ERR_INVALID;
    if (n == 0) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(map_reserve_input(m, n));
    KICP_TRY(map_reserve(m, (uint64_t)n));  // worst case: every point opens a new voxel
    const double *d_src = xyz;
    if (!src_on_device) {
        KICP_CUDA(cudaMemcpyAsync(m->d_in, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        d_src = m->d_in;
    }
    uint32_t init[8] = {m->num_blocks, 0, 0, 0, 0, 0, 0, 0};
    KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    MapRW rw{m->slots, m->nslots - 1, m->blk, m->pts, m->pend_head, m->blocks_cap, (int)m->cap, m->voxel_size};
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const int threads = 256;
    k_add_find_or_create<<<(unsigned)((n + threads - 1) / threads), threads, 0, c->stream>>>(
        rw, d_src, n, pose7 ? 1 : 0, pose, m->d_xyz_t, m->d_next, m->d_counters, m->d_touched);
    KICP_CHECK_LAUNCH(c);
    // KISS AddPoints: map_resolution = sqrt(voxel_size^2 / max_points_per_voxel)
    const double map_resolution = std::sqrt(m->voxel_size * m->voxel_size / (double)m->cap);
    k_add_commit<<<(unsigned)((n + threads - 1) / threads), threads, 0, c->stream>>>(rw, m->d_xyz_t, m->d_next, m->d_counters,
                                                                                 m->d_touched, map_resolution);
    KICP_CHECK_LAUNCH(c);
    uint32_t res[8];
    KICP_CUDA(cudaMemcpyAsync(res, m->d_counters, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    if (res[2]) {
        kicp_set_error("voxel map: block storage overflow during AddPoints");
        return KICP_ERR_CAPACITY;
    }
    m->num_blocks = res[0];
    m->num_points += res[3];
    return KICP_OK;
}

extern "C" int kicp_map_add_points(kicp_map *m, const double *xyz, int64_t n) { return map_add_points_impl(m, xyz, n, nullptr); }

extern "C" int kicp_map_remove_far(kicp_map *m, const double origin[3]) {
    if (!m || !origin) return KICP_ERR_INVALID;
    if (m->num_blocks == 0) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    uint32_t *keep = m->d_keep, *new_id = m->d_new_id;
    uint32_t init[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    k_mark_far<<<(m->num_blocks + 255) / 256, 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, m->num_blocks, origin[0], origin[1],
                                                                  origin[2], m->max_distance * m->max_distance, keep,
                                                                  m->d_counters);
    KICP_CHECK_LAUNCH(c);
    uint32_t res[8];
    KICP_CUDA(cudaMemcpyAsync(res, m->d_counters, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    if (res[4] > 0) {
        // compact surviving blocks (order preserved) into the spare arrays, swap, and rebuild the table
        const uint32_t survivors = m->num_blocks - res[4];
        KICP_TRY(enqueue_exclusive_sum(c, keep, new_id, m->num_blocks));
        k_compact_blocks<<<(unsigned)(((uint64_t)m->num_blocks * 32 + 255) / 256), 256, 0, c->stream>>>(
            m->blk, m->pts, (int)m->cap, m->num_blocks, keep, new_id, m->blk_spare, m->pts_spare);
        KICP_CHECK_LAUNCH(c);
        std::swap(m->blk, m->blk_spare);
        std::swap(m->pts, m->pts_spare);
        m->num_blocks = survivors;
        m->num_points -= res[3];
        KICP_TRY(map_rebuild_table(m, m->nslots));  // stream-ordered after the compaction
    }
    return KICP_OK;
}

extern "C" int kicp_map_update(kicp_map *m, const double *xyz, int64_t n, const double origin[3]) {
    KICP_TRY(map_add_points_impl(m, xyz, n, nullptr));
    return kicp_map_remove_far(m, origin);
}
extern "C" int kicp_map_update_pose(kicp_map *m, const double *xyz, int64_t n, const double pose[7]) {
    if (!pose) return KICP_ERR_INVALID;
    KICP_TRY(map_add_points_impl(m, xyz, n, pose));
    return kicp_map_remove_far(m, pose + 4);
}
int kicp_map_update_pose_device(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7]) {
    if (!pose) return KICP_ERR_INVALID;
    KICP_TRY(map_add_points_impl(m, d_xyz, n, pose, true));
    return kicp_map_remove_far(m, pose + 4);
}

// local_map_.Update(frame, pose) (KinematicICP.cpp:79) for a frame whose point count (`d_n` <= n_max) and pose (`d_res`) are
// still being computed on the stream: everything is enqueued, nothing is read back.  The eviction always compacts (into the spare
// arrays, then the arrays swap) — a moving sensor evicts voxels on practically every frame anyway, and the host cannot know.
// The counters are copied to `h_counters` (pinned, 8 words); after the caller's end-of-frame synchronisation,
// kicp_map_finish_update() brings the host mirrors up to date.
int kicp_map_update_pose_async(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const kicp_reg_result *d_res,
                               uint32_t *h_counters) {
    if (!m || n_max <= 0 || !d_xyz || !d_n || !d_res || !h_counters) return KICP_ERR_INVALID;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(map_reserve_input(m, n_max));
    KICP_TRY(map_reserve(m, (uint64_t)n_max));  // worst case: every point opens a new voxel (grows — and synchronises — rarely)
    const uint32_t init[8] = {m->num_blocks, 0, 0, 0, 0, 0, 0, 0};
    KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    MapRW rw{m->slots, m->nslots - 1, m->blk, m->pts, m->pend_head, m->blocks_cap, (int)m->cap, m->voxel_size};
    const int threads = 256;
    const unsigned pgrid = (unsigned)((n_max + threads - 1) / threads);
    k_add_find_or_create<<<pgrid, threads, 0, c->stream>>>(rw, d_xyz, n_max, 1, Pose{0, 0, 0, 1, 0, 0, 0}, m->d_xyz_t, m->d_next, m->d_counters,
                                                        m->d_touched, d_n, d_res);
    KICP_CHECK_LAUNCH(c);
    const double map_resolution = std::sqrt(m->voxel_size * m->voxel_size / (double)m->cap);
    k_add_commit<<<pgrid, threads, 0, c->stream>>>(rw, m->d_xyz_t, m->d_next, m->d_counters, m->d_touched, map_resolution);
    KICP_CHECK_LAUNCH(c);
    // RemovePointsFarFromLocation(pose.translation()) over the blocks that exist now: at most ub
    const uint32_t ub = (uint32_t)std::min<uint64_t>((uint64_t)m->num_blocks + (uint64_t)n_max, m->blocks_cap);
    k_mark_far<<<(ub + 255) / 256, 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, ub, 0.0, 0.0, 0.0, m->max_distance * m->max_distance,
                                                     m->d_keep, m->d_counters, d_res);
    KICP_CHECK_LAUNCH(c);
    KICP_TRY(enqueue_exclusive_sum(c, m->d_keep, m->d_new_id, ub));
    k_compact_blocks<<<(unsigned)(((uint64_t)ub * 32 + 255) / 256), 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, ub, m->d_keep,
                                                                                       m->d_new_id, m->blk_spare, m->pts_spare);
    KICP_CHECK_LAUNCH(c);
    std::swap(m->blk, m->blk_spare);
    std::swap(m->pts, m->pts_spare);
    KICP_CUDA(cudaMemsetAsync(m->slots, 0xFF, (size_t)m->nslots * sizeof(int4), c->stream));
    k_table_rebuild<<<(ub + 255) / 256, 256, 0, c->stream>>>(m->slots, m->nslots - 1, m->blk, ub, m->d_counters);
    KICP_CHECK_LAUNCH(c);
    KICP_CUDA(cudaMemcpyAsync(h_counters, m->d_counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    return KICP_OK;
}
// after the stream has drained: host mirrors from the counters of kicp_map_update_pose_async
int kicp_map_finish_update(kicp_map *m, const uint32_t *h_counters) {
    if (!m || !h_counters) return KICP_ERR_INVALID;
    m->num_blocks = h_counters[0] - h_counters[4];
    m->num_points += (int64_t)h_counters[3] - (int64_t)h_counters[5];
    if (h_counters[2]) {
        kicp_set_error("voxel map: block storage overflow during AddPoints");
        return KICP_ERR_CAPACITY;
    }
    return KICP_OK;
}

// Pointcloud / export: the stored points are packed ON THE DEVICE (block order, insertion order inside a block — the order the
// host loop used to produce) and exactly num_points * 24 bytes cross PCIe, instead of the padded block array (20 slots of 32
// bytes per voxel whatever it holds).  The spare point array is the scratch: it holds nothing between two evictions.
__global__ void k_block_counts(const int4 *blk, uint32_t num_blocks, uint32_t *cnt) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < num_blocks) cnt[b] = (uint32_t)blk[b].w;
}
__global__ void k_pack_points(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, const uint32_t *first, double *out) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per block
    const int lane = threadIdx.x & 31;
    if (b >= num_blocks) return;
    const int cnt = blk[b].w;
    const double *src = pts + (size_t)b * cap * KICP_PSTRIDE;
    double *dst = out + (size_t)first[b] * 3;
    for (int i = lane; i < cnt * 3; i += 32) dst[i] = src[(i / 3) * KICP_PSTRIDE + (i % 3)];
}
// packed xyz of every stored point -> host `out_xyz` (num_points * 3 doubles); headers -> `hdr` when asked for
static int map_download_packed(kicp_map *m, double *out_xyz, std::vector<int4> *hdr) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    if (m->num_blocks == 0) return KICP_OK;
    k_block_counts<<<(m->num_blocks + 255) / 256, 256, 0, c->stream>>>(m->blk, m->num_blocks, m->d_keep);
    KICP_CHECK_LAUNCH(c);
    if (m->num_points >= (1ll << 30)) {
        kicp_set_error("voxel map: export of 2^30 points or more is not supported");
        return KICP_ERR_CAPACITY;
    }
    KICP_TRY(enqueue_exclusive_sum(c, m->d_keep, m->d_new_id, m->num_blocks));
    k_pack_points<<<(unsigned)(((uint64_t)m->num_blocks * 32 + 255) / 256), 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, m->num_blocks,
                                                                                                m->d_new_id, m->pts_spare);
    KICP_CHECK_LAUNCH(c);
    KICP_CUDA(cudaMemcpyAsync(out_xyz, m->pts_spare, (size_t)m->num_points * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (hdr) {
        hdr->resize(m->num_blocks);
        KICP_CUDA(cudaMemcpyAsync(hdr->data(), m->blk, hdr->size() * sizeof(int4), cudaMemcpyDeviceToHost, c->stream));
    }
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

extern "C" int kicp_map_pointcloud(kicp_map *m, double *out_xyz, int64_t cap, int64_t *n) {
    if (!m || !n) return KICP_ERR_INVALID;
    *n = m->num_points;
    if (m->num_points > cap) return KICP_ERR_CAPACITY;
    if (m->num_points == 0) return KICP_OK;
    if (!out_xyz) return KICP_ERR_INVALID;
    return map_download_packed(m, out_xyz, nullptr);
}

extern "C" int kicp_map_export_voxels(kicp_map *m, int32_t *keys, int32_t *counts, double *points, int64_t cap_voxels,
                                      int64_t cap_points, int64_t *num_voxels, int64_t *num_points) {
    if (!m || !num_voxels || !num_points) return KICP_ERR_INVALID;
    *num_voxels = m->num_blocks, *num_points = m->num_points;
    if ((int64_t)m->num_blocks > cap_voxels || m->num_points > cap_points) return KICP_ERR_CAPACITY;
    if (m->num_blocks == 0) return KICP_OK;
    if (!keys || !counts || !points) return KICP_ERR_INVALID;
    std::vector<int4> hdr;
    KICP_TRY(map_download_packed(m, points, &hdr));
    for (uint32_t b = 0; b < m->num_blocks; ++b) {
        keys[3 * b] = hdr[b].x, keys[3 * b + 1] = hdr[b].y, keys[3 * b + 2] = hdr[b].z;
        counts[b] = hdr[b].w;
    }
    return KICP_OK;
}

extern "C" int kicp_map_load_voxels(kicp_map *m, const int32_t *keys, const int32_t *counts, const double *points,
                                    int64_t num_voxels) {
    if (!m || num_voxels < 0 || (num_voxels > 0 && (!keys || !counts || !points))) return KICP_ERR_INVALID;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(kicp_map_clear(m));
    if (num_voxels == 0) return KICP_OK;
    std::vector<int64_t> offsets((size_t)num_voxels);
    int64_t total = 0;
    for (int64_t v = 0; v < num_voxels; ++v) {
        if (counts[v] <= 0 || counts[v] > (int32_t)m->cap) {
            kicp_set_error("kicp_map_load_voxels: voxel count outside [1, max_points_per_voxel]");
            return KICP_ERR_INVALID;
        }
        offsets[v] = total;
        total += counts[v];
    }
    KICP_TRY(map_reserve(m, (uint64_t)num_voxels));
    int32_t *d_keys = nullptr, *d_counts = nullptr;
    int64_t *d_off = nullptr;
    double *d_pts = nullptr;
    KICP_CUDA(cudaMalloc(&d_keys, (size_t)num_voxels * 3 * sizeof(int32_t)));
    KICP_CUDA(cudaMalloc(&d_counts, (size_t)num_voxels * sizeof(int32_t)));
    KICP_CUDA(cudaMalloc(&d_off, (size_t)num_voxels * sizeof(int64_t)));
    KICP_CUDA(cudaMalloc(&d_pts, (size_t)total * 3 * sizeof(double)));
    KICP_CUDA(cudaMemcpyAsync(d_keys, keys, (size_t)num_voxels * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    KICP_CUDA(cudaMemcpyAsync(d_counts, counts, (size_t)num_voxels * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    KICP_CUDA(cudaMemcpyAsync(d_off, offsets.data(), (size_t)num_voxels * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    KICP_CUDA(cudaMemcpyAsync(d_pts, points, (size_t)total * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    k_load_voxels<<<(unsigned)(((uint64_t)num_voxels * 32 + 255) / 256), 256, 0, c->stream>>>(
        m->blk, m->pts, (int)m->cap, d_keys, d_counts, d_off, d_pts, (uint32_t)num_voxels);
    KICP_CHECK_LAUNCH(c);
    m->num_blocks = (uint32_t)num_voxels;
    m->num_points = total;
    int st = map_rebuild_table(m, m->nslots);
    cudaError_t e = cudaStreamSynchronize(c->stream);
    cudaFree(d_keys), cudaFree(d_counts), cudaFree(d_off), cudaFree(d_pts);
    if (st != KICP_OK) return st;
    if (e != cudaSuccess) return kicp_cuda_fail(e, "load_voxels", __FILE__, __LINE__);
    return KICP_OK;
}

extern "C" int kicp_map_nearest(kicp_map *m, const double *queries, int64_t n, double *out_points, double *out_dist) {
    if (!m || n < 0 || (n > 0 && (!queries || !out_points || !out_dist))) return KICP_ERR_INVALID;
    if (n == 0) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    double *d_q = nullptr, *d_p = nullptr, *d_d = nullptr;
    KICP_CUDA(cudaMalloc(&d_q, (size_t)n * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&d_p, (size_t)n * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&d_d, (size_t)n * sizeof(double)));
    KICP_CUDA(cudaMemcpyAsync(d_q, queries, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    k_nearest<<<(unsigned)((n + 127) / 128), 128, 0, c->stream>>>(m->view(), d_q, n, d_p, d_d);
    KICP_CHECK_LAUNCH(c);
    KICP_CUDA(cudaMemcpyAsync(out_points, d_p, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaMemcpyAsync(out_dist, d_d, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    cudaError_t e = cudaStreamSynchronize(c->stream);
    cudaFree(d_q), cudaFree(d_p), cudaFree(d_d);
    if (e != cudaSuccess) return kicp_cuda_fail(e, "nearest", __FILE__, __LINE__);
    return KICP_OK;
}
