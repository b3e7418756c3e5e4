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
int kicp_invalid(const char *fn, const char *why) {
    kicp_set_error(std::string(fn) + ": " + why);
    return KICP_ERR_INVALID;
}
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
    KICP_CUDA(cudaEventCreateWithFlags(&c->ev_order, cudaEventDisableTiming));
    KICP_TRY(kicp_reg_scratch_create(c));
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

// Ordering with a caller's stream (0, cudaStreamLegacy and cudaStreamPerThread included): the context's event is recorded on one
// stream and waited for by the other; the host does not wait.
static int order_streams(kicp_ctx *ctx, cudaStream_t from, cudaStream_t to) {
    KICP_CUDA(cudaSetDevice(ctx->device));
    KICP_CUDA(cudaEventRecord(ctx->ev_order, from));
    KICP_CUDA(cudaStreamWaitEvent(to, ctx->ev_order, 0));
    return KICP_OK;
}
extern "C" int kicp_ctx_wait_stream(kicp_ctx *ctx, void *stream) {
    if (!ctx) return KICP_ERR_INVALID;
    return order_streams(ctx, (cudaStream_t)stream, ctx->stream);
}
extern "C" int kicp_stream_wait_ctx(kicp_ctx *ctx, void *stream) {
    if (!ctx) return KICP_ERR_INVALID;
    return order_streams(ctx, ctx->stream, (cudaStream_t)stream);
}

int kicp_check_device_range(const kicp_ctx *c, const void *p, size_t bytes, size_t align, const char *what) {
    auto fail = [what](const char *why) {
        kicp_set_error(std::string(what) + ": " + why);
        return KICP_ERR_INVALID;
    };
    if (!p) return fail("null pointer");
    if (align > 1 && reinterpret_cast<uintptr_t>(p) % align) return fail("not aligned to its element size");
    const unsigned char *ends[2] = {static_cast<const unsigned char *>(p), static_cast<const unsigned char *>(p) + (bytes ? bytes - 1 : 0)};
    for (const unsigned char *q : ends) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, q) != cudaSuccess) {
            cudaGetLastError();
            return fail("not memory the CUDA runtime knows");
        }
        if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return fail("not device memory");
        if (at.device != c->device) return fail("device memory of another GPU than the context's");
    }
    return KICP_OK;
}

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
// host `data`: copied into the scan's buffer on the context stream; `device` data: read in place by the registrations that follow
static int scan_upload(kicp_scan *s, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x, int32_t offset_y,
                       int32_t offset_z, bool device) {
    if (!s || n < 0 || (n > 0 && !data)) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(s->ctx->device));
    if (device) {
        kicp_scan l = *s;  // a failing attach leaves the scan as it was
        KICP_TRY(kicp_scan_set_layout(&l, dtype, point_step, offset_x, offset_y, offset_z));
        const int w = l.dtype == KICP_DTYPE_F32 ? 4 : 8;
        const int64_t bytes = n > 0 ? (n - 1) * l.stride + std::max(l.ox, std::max(l.oy, l.oz)) + w : 0;
        if (n > 0) KICP_TRY(kicp_check_device_range(s->ctx, data, (size_t)bytes, w, "kicp_scan_attach_device: data"));
        l.d_attached = n > 0 ? data : nullptr;
        *s = l;
    } else {
        KICP_TRY(kicp_scan_set_layout(s, dtype, point_step, offset_x, offset_y, offset_z));
        KICP_TRY(kicp_scan_reserve_bytes(s, n * (int64_t)s->stride));
        if (n > 0) KICP_CUDA(cudaMemcpyAsync(s->d_data, data, (size_t)(n * s->stride), cudaMemcpyHostToDevice, s->ctx->stream));
        s->d_attached = nullptr;
    }
    s->n = n, s->d_n = nullptr;
    return KICP_OK;
}
extern "C" int kicp_scan_upload_points_async(kicp_scan *s, const void *data, int64_t n, int32_t dtype, int32_t point_step,
                                             int32_t offset_x, int32_t offset_y, int32_t offset_z) {
    return scan_upload(s, data, n, dtype, point_step, offset_x, offset_y, offset_z, false);
}
extern "C" int kicp_scan_attach_device(kicp_scan *s, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                       int32_t offset_y, int32_t offset_z) {
    return scan_upload(s, data, n, dtype, point_step, offset_x, offset_y, offset_z, true);
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
    kicp_reg_scratch_free(ctx);
    cudaFree(ctx->d_scan_status);
    cudaFree(ctx->d_scan_ticket);
    cudaFreeHost(ctx->h_result);
    if (ctx->ev_order) cudaEventDestroy(ctx->ev_order);
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

static void map_live_free(kicp_map *m);  // state of kicp_map_pointcloud_f32_live, below
static void pose_scratch_free(kicp_map *m);  // scratch of kicp_map_pose_search*, below

// -------------------------------------------------------------------------------------------- host-side storage
static uint32_t next_pow2(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return (uint32_t)p;
}

// (Re)build the open-addressed table over the first `nslots` slots of the slab's table region (nslots <= slots_cap) from the first
// `nb` blocks.  `ctr` (the frame path): the counters of the update just enqueued, from which k_table_rebuild reads the block count;
// nb is then its upper bound.
// With a frozen prior of P blocks the table is the prior's snapshot plus blocks [P, nb): `restore` (after an eviction, same size and
// slab) copies the snapshot in, in place of the clear; otherwise (a new size or a new slab) the prior is inserted first and the
// snapshot taken from it.
static int map_rebuild_table(kicp_map *m, uint32_t nslots, uint32_t nb, const uint32_t *ctr = nullptr, bool restore = false) {
    kicp_ctx *c = m->ctx;
    if (nslots > m->slots_cap) {
        kicp_set_error("voxel map: internal error, table larger than its slab region");
        return KICP_ERR_CAPACITY;
    }
    m->nslots = nslots;
    const uint32_t P = m->prior_blocks;
    const size_t table_bytes = (size_t)m->nslots * sizeof(int4);
    if (P && restore) {
        KICP_CUDA(cudaMemcpyAsync(m->slots, m->prior_slots, table_bytes, cudaMemcpyDeviceToDevice, c->stream));
    } else {
        KICP_CUDA(cudaMemsetAsync(m->slots, 0xFF, table_bytes, c->stream));
        if (P) {
            if (m->prior_slots_cap < m->nslots) {
                KICP_CUDA(cudaStreamSynchronize(c->stream));
                cudaFree(m->prior_slots);
                m->prior_slots = nullptr, m->prior_slots_cap = 0;
                KICP_CUDA(cudaMalloc(&m->prior_slots, (size_t)m->slots_cap * sizeof(int4)));
                m->prior_slots_cap = m->slots_cap;
            }
            k_table_rebuild<<<(P + 255) / 256, 256, 0, c->stream>>>(m->slots, m->nslots - 1, m->blk, P);
            KICP_CHECK_LAUNCH(c);
            KICP_CUDA(cudaMemcpyAsync(m->prior_slots, m->slots, table_bytes, cudaMemcpyDeviceToDevice, c->stream));
        }
    }
    if (nb > P) {
        k_table_rebuild<<<(nb - P + 255) / 256, 256, 0, c->stream>>>(m->slots, m->nslots - 1, m->blk, nb, ctr, P);
        KICP_CHECK_LAUNCH(c);
    }
    return KICP_OK;
}

// the prior prefix [0, P) of the live arrays into the spare ones, which a compaction fills from block P on
static int map_mirror_prior(kicp_map *m) {
    const uint32_t P = m->prior_blocks;
    if (!P) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaMemcpyAsync(m->blk_spare, m->blk, (size_t)P * sizeof(int4), cudaMemcpyDeviceToDevice, c->stream));
    KICP_CUDA(cudaMemcpyAsync(m->pts_spare, m->pts, (size_t)P * m->cap * KICP_PSTRIDE * sizeof(double), cudaMemcpyDeviceToDevice,
                              c->stream));
    if (m->d_occ)
        KICP_CUDA(cudaMemcpyAsync(m->d_occ_spare, m->d_occ, (size_t)P * sizeof(int32_t), cudaMemcpyDeviceToDevice, c->stream));
    return KICP_OK;
}

static void map_prior_free(kicp_map *m) {
    cudaFree(m->prior_slots);
    m->prior_slots = nullptr, m->prior_slots_cap = 0;
    m->prior_blocks = 0, m->prior_points = 0;
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
    int32_t *nocc = nullptr;  // occupancy on: the evidence of [0, num_blocks) moves to a grown allocation
    if (m->occ_slab) {
        const cudaError_t e = cudaMalloc(&nocc, (size_t)2 * ncap * sizeof(int32_t));
        if (e != cudaSuccess) {
            cudaStreamSynchronize(c->stream);
            cudaFree(slab);
            return kicp_cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
        }
        if (m->num_blocks)
            KICP_CUDA(cudaMemcpyAsync(nocc, m->d_occ, (size_t)m->num_blocks * sizeof(int32_t), cudaMemcpyDeviceToDevice, c->stream));
    }
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    if (nocc) {
        cudaFree(m->occ_slab);
        m->occ_slab = m->d_occ = nocc, m->d_occ_spare = nocc + ncap, m->occ_cap = ncap;
    }
    cudaFree(m->slab);
    m->slab = slab, m->slab_bytes = off;
    m->blk = nblk, m->pts = npts, m->pend_head = nhead, m->blocks_cap = ncap;
    m->blk_spare = reinterpret_cast<int4 *>(slab + o_blk2), m->pts_spare = reinterpret_cast<double *>(slab + o_pts2);
    m->d_keep = reinterpret_cast<uint32_t *>(slab + o_keep), m->d_new_id = reinterpret_cast<uint32_t *>(slab + o_id);
    m->slots = reinterpret_cast<int4 *>(slab + o_slots), m->slots_cap = slots_cap;
    KICP_TRY(map_mirror_prior(m));  // the new spare arrays hold the frozen prefix too
    // the table moved with the slab: rebuild it at its previous size (or the minimum for a new map)
    return map_rebuild_table(m, std::max<uint32_t>(std::min(m->nslots, slots_cap), 1024u), m->num_blocks);
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
    if (want_slots > m->nslots) KICP_TRY(map_rebuild_table(m, want_slots, m->num_blocks));
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
    cudaFree(m->d_in), cudaFree(m->d_xyz_t), cudaFree(m->d_next), cudaFree(m->d_touched), cudaFree(m->d_dist);
    m->d_in = m->d_xyz_t = m->d_dist = nullptr, m->d_next = m->d_touched = nullptr;
    const int64_t cap = std::max<int64_t>(n + n / 4, 4096);
    KICP_CUDA(cudaMalloc(&m->d_in, (size_t)cap * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&m->d_xyz_t, (size_t)cap * 3 * sizeof(double)));
    KICP_CUDA(cudaMalloc(&m->d_next, (size_t)cap * sizeof(int32_t)));
    KICP_CUDA(cudaMalloc(&m->d_touched, (size_t)cap * sizeof(int32_t)));
    KICP_CUDA(cudaMalloc(&m->d_dist, (size_t)cap * sizeof(double)));
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
    cudaFree(m->slab), cudaFree(m->d_counters), cudaFree(m->d_free_stats), cudaFree(m->occ_slab);
    map_prior_free(m);
    cudaFree(m->d_in), cudaFree(m->d_xyz_t), cudaFree(m->d_next), cudaFree(m->d_touched), cudaFree(m->d_dist);
    cudaFree(m->d_corr_part), cudaFree(m->d_corr_stats), cudaFree(m->d_corr_inl);
    map_live_free(m);
    pose_scratch_free(m);
    kicp_align_scratch_free(m);
    delete m;
    return KICP_OK;
}

extern "C" int kicp_map_clear(kicp_map *m) {
    if (!m) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    m->num_blocks = 0, m->num_points = 0;
    KICP_CUDA(cudaMemsetAsync(m->slots, 0xFF, (size_t)m->nslots * sizeof(int4), m->ctx->stream));
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    map_prior_free(m);  // the prior goes with the content
    return KICP_OK;
}

extern "C" int kicp_map_freeze(kicp_map *m) {
    if (!m) return kicp_invalid("kicp_map_freeze", "null map");
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    if (m->num_blocks == 0) {  // nothing to freeze: no prior
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        map_prior_free(m);
        return KICP_OK;
    }
    // every voxel now in the table becomes prior, so the table as it stands is the prior's snapshot
    if (m->prior_slots_cap < m->slots_cap) {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(m->prior_slots);
        m->prior_slots = nullptr, m->prior_slots_cap = 0;
        KICP_CUDA(cudaMalloc(&m->prior_slots, (size_t)m->slots_cap * sizeof(int4)));
        m->prior_slots_cap = m->slots_cap;
    }
    KICP_CUDA(cudaMemcpyAsync(m->prior_slots, m->slots, (size_t)m->nslots * sizeof(int4), cudaMemcpyDeviceToDevice, c->stream));
    m->prior_blocks = m->num_blocks, m->prior_points = m->num_points;
    KICP_TRY(map_mirror_prior(m));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

extern "C" int kicp_map_thaw(kicp_map *m) {
    if (!m) return kicp_invalid("kicp_map_thaw", "null map");
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    map_prior_free(m);
    return KICP_OK;
}

extern "C" int kicp_map_prior_size(kicp_map *m, int64_t *voxels, int64_t *points) {
    static const char fn[] = "kicp_map_prior_size";
    if (!voxels) return kicp_invalid(fn, "voxels: null pointer");
    if (!points) return kicp_invalid(fn, "points: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    *voxels = m->prior_blocks, *points = m->prior_points;
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

// The host mirrors from the counter words of an update, once the stream has drained.  The kernels define the words
// (kicp_map_kernels.cuh): [0] blocks after the insert, [2] overflow, [3] points inserted, [4] blocks evicted, [5] points evicted by
// the frame path's k_mark_far.  A synchronous eviction (`evict_only`) has counters of its own, and its k_mark_far counts the points
// evicted in word 3.
int kicp_map_finish_update(kicp_map *m, const uint32_t *ctr, bool evict_only) {
    if (!m || !ctr) return KICP_ERR_INVALID;
    // cannot happen: map_reserve makes room for one new block per point before every insert
    if (ctr[2]) {
        kicp_set_error("voxel map: block storage overflow during AddPoints");
        return KICP_ERR_CAPACITY;
    }
    const int64_t added = evict_only ? 0 : ctr[3], removed = ctr[evict_only ? 3 : 5];
    m->num_blocks = (evict_only ? m->num_blocks : ctr[0]) - ctr[4];
    m->num_points += added - removed;
    return KICP_OK;
}

// AddPoints of the `n` points at `xyz` (a host array, or with `xyz_on_device` packed doubles in HBM that stay valid until the stream
// drains), enqueued on the context stream.  The points are transformed by the pose first when there is one: `pose7` from the host,
// or on the frame path the pose of `d_res`, the result block of the registration enqueued before, with the point count `d_n` (<= n)
// also read on the device.
static int map_insert(kicp_map *m, const double *xyz, bool xyz_on_device, int64_t n, const double *pose7, const int *d_n,
                      const kicp_reg_result *d_res) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(map_reserve_input(m, n));
    KICP_TRY(map_reserve(m, (uint64_t)n));  // worst case: every point opens a new voxel (grows — and synchronises — rarely)
    if (!xyz_on_device) {
        KICP_CUDA(cudaMemcpyAsync(m->d_in, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        xyz = m->d_in;
    }
    const uint32_t init[8] = {m->num_blocks, 0, 0, 0, 0, 0, 0, 0};
    KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    MapRW rw{m->slots, m->nslots - 1, m->blk, m->pts, m->pend_head, m->blocks_cap, (int)m->cap, m->voxel_size};
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const unsigned grid = (unsigned)((n + 255) / 256);
    k_add_find_or_create<<<grid, 256, 0, c->stream>>>(rw, xyz, n, pose7 || d_res ? 1 : 0, pose, m->d_xyz_t, m->d_next, m->d_counters,
                                                     m->d_touched, d_n, d_res, m->prior_blocks, m->d_occ, m->occ.initial);
    KICP_CHECK_LAUNCH(c);
    // KISS AddPoints: map_resolution = sqrt(voxel_size^2 / max_points_per_voxel)
    const double map_resolution = std::sqrt(m->voxel_size * m->voxel_size / (double)m->cap);
    k_add_commit<<<grid, 256, 0, c->stream>>>(rw, m->d_xyz_t, m->d_next, m->d_counters, m->d_touched, map_resolution);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// ---------------------------------------------------------------------------------------------------- free-space clearing
#include "kicp_free_space_kernels.cuh"  // FreeRayArgs, k_free_rays, k_mark_free

// The map's free-space words, one allocation beside the slab: kFreeStatWords statistics words, then one flag word per block of
// capacity.  Allocated on the first clearing and grown with the block capacity (the stream drained first); a map that never clears
// has none.
static int free_reserve(kicp_map *m) {
    if (m->free_cap >= m->blocks_cap) return KICP_OK;
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    cudaFree(m->d_free_stats);
    m->d_free_stats = nullptr, m->d_free_flags = nullptr, m->free_cap = 0;
    void *p = nullptr;
    KICP_CUDA(cudaMalloc(&p, kFreeStatWords * sizeof(unsigned long long) + (size_t)m->blocks_cap * sizeof(uint32_t)));
    m->d_free_stats = static_cast<unsigned long long *>(p);
    m->d_free_flags = reinterpret_cast<uint32_t *>(m->d_free_stats + kFreeStatWords);
    m->free_cap = m->blocks_cap;
    return KICP_OK;
}

// One memset (the statistics and the flags of blocks [0, nb)), then k_free_rays over the n rays of d_xyz (packed doubles) at `pose7`
// (host) or at the pose of `d_res` with the count min(*d_n, n); the grid is at most the resident one (the warps stride over the rest)
static int enqueue_free_rays(kicp_map *m, const double *d_xyz, int64_t n, const int *d_n, const double *pose7, const kicp_reg_result *d_res,
                             const double origin[3], const kicp_free_space_params &p, uint32_t nb) {
    kicp_ctx *c = m->ctx;
    KICP_TRY(free_reserve(m));
    KICP_CUDA(cudaMemsetAsync(m->d_free_stats, 0, kFreeStatWords * sizeof(unsigned long long) + (size_t)nb * sizeof(uint32_t), c->stream));
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const FreeRayArgs a{origin[0], origin[1], origin[2], p.end_margin, m->max_distance, (uint32_t)p.min_misses};
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)m->ctx->sm_count * 8));
    k_free_rays<<<grid, 256, 0, c->stream>>>(m->view(), d_xyz, n, d_n, pose, d_res, a, m->d_free_flags, m->d_free_stats);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

static int enqueue_mark_free(kicp_map *m, uint32_t nb, uint32_t min_misses, const kicp_reg_result *d_res) {
    kicp_ctx *c = m->ctx;
    const OccupancyArgs occ{m->occ.hit_gain, m->occ.miss_loss, m->occ.max_evidence};
    k_mark_free<<<(nb + 255) / 256, 256, 0, c->stream>>>(m->blk, nb, m->prior_blocks, m->d_free_flags, min_misses, m->d_keep,
                                                        m->d_counters, m->d_free_stats, d_res, m->d_occ, occ);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// RemovePointsFarFromLocation over the first `nb` blocks: k_mark_far flags the survivors, which are compacted (order kept) into the
// spare arrays; those swap with the live ones and the table is rebuilt.  Synchronous (`d_res` null): the eviction zeroes the
// counters, reads them back after k_mark_far and compacts only when a voxel died.  Frame path: the origin and the registration's
// status are read from `d_res` on the device (`origin` is unused) and the block count from the insert's counters (nb is its upper
// bound).  Nothing is read back and the compaction always runs — a moving sensor evicts voxels on practically every frame anyway,
// and the host cannot know.
// With a frozen prior of P blocks every step runs over the suffix [P, nb) only: the prior never dies, the spare arrays already hold
// its copy at [0, P), and the table is restored from the prior's snapshot before the live blocks are re-inserted.  Each step is still
// one launch.
// The survivors of d_keep over [P, nb) compacted in order into the spare arrays, which swap with the live ones; the host mirrors from
// `res` (synchronous: the counters read back) and the table restored after the compaction
static int map_compact(kicp_map *m, const kicp_reg_result *d_res, uint32_t nb, const uint32_t *res) {
    kicp_ctx *c = m->ctx;
    const uint32_t P = m->prior_blocks, nl = nb - P;
    KICP_TRY(enqueue_exclusive_sum(c, m->d_keep + P, m->d_new_id + P, nl));
    k_compact_blocks<<<(unsigned)(((uint64_t)nl * 32 + 255) / 256), 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, nb, m->d_keep,
                                                                                       m->d_new_id, m->blk_spare, m->pts_spare, P, m->d_occ,
                                                                                       m->d_occ_spare);
    KICP_CHECK_LAUNCH(c);
    std::swap(m->blk, m->blk_spare);
    std::swap(m->pts, m->pts_spare);
    std::swap(m->d_occ, m->d_occ_spare);
    if (!d_res) KICP_TRY(kicp_map_finish_update(m, res, true));
    return map_rebuild_table(m, m->nslots, d_res ? nb : m->num_blocks, d_res ? m->d_counters : nullptr, true);
}
// `free_min` (frame path with free-space clearing, > 0): k_mark_free runs after k_mark_far over the flags k_free_rays left
static int map_evict(kicp_map *m, const double origin[3], const kicp_reg_result *d_res, uint32_t nb, uint32_t free_min = 0) {
    kicp_ctx *c = m->ctx;
    const uint32_t P = m->prior_blocks;
    if (nb <= P) return KICP_OK;  // (synchronous only: the frame path's bound exceeds the block count) nothing can die
    const uint32_t nl = nb - P;
    const uint32_t init[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (!d_res) KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    k_mark_far<<<(nl + 255) / 256, 256, 0, c->stream>>>(m->blk, m->pts, (int)m->cap, nb, origin[0], origin[1], origin[2],
                                                       m->max_distance * m->max_distance, m->d_keep, m->d_counters, d_res, P);
    KICP_CHECK_LAUNCH(c);
    if (free_min) KICP_TRY(enqueue_mark_free(m, nb, free_min, d_res));
    uint32_t res[8];
    if (!d_res) {
        KICP_CUDA(cudaMemcpyAsync(res, m->d_counters, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        if (res[4] == 0) return KICP_OK;
    }
    return map_compact(m, d_res, nb, res);
}

// AddPoints with the count and the pose on the host: one synchronisation, after which the host mirrors are current
static int map_add_points_impl(kicp_map *m, const double *xyz, int64_t n, const double *pose7, bool xyz_on_device = false) {
    if (!m || n < 0 || (n > 0 && !xyz)) return KICP_ERR_INVALID;
    if (n == 0) return KICP_OK;
    KICP_TRY(map_insert(m, xyz, xyz_on_device, n, pose7, nullptr, nullptr));
    uint32_t res[8];
    KICP_CUDA(cudaMemcpyAsync(res, m->d_counters, sizeof(res), cudaMemcpyDeviceToHost, m->ctx->stream));
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    return kicp_map_finish_update(m, res, false);
}

extern "C" int kicp_map_add_points(kicp_map *m, const double *xyz, int64_t n) { return map_add_points_impl(m, xyz, n, nullptr); }

extern "C" int kicp_map_remove_far(kicp_map *m, const double origin[3]) {
    if (!m || !origin) return KICP_ERR_INVALID;
    if (m->num_blocks == 0) return KICP_OK;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    return map_evict(m, origin, nullptr, m->num_blocks);
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
int kicp_map_update_pose_packed(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7]) {
    if (!pose) return KICP_ERR_INVALID;
    KICP_TRY(map_add_points_impl(m, d_xyz, n, pose, true));
    return kicp_map_remove_far(m, pose + 4);
}

// The points of a map call from a device cloud (kicp_map_*_device): read in place when they are packed doubles, else widened by
// k_ingest into the map's input buffer.  `in` has passed kicp_check_device_cloud.
static int map_device_points(kicp_map *m, const kicp_frame_input &in, bool packed, const double **xyz) {
    *xyz = static_cast<const double *>(in.data);
    if (packed || in.n == 0) return KICP_OK;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    KICP_TRY(map_reserve_input(m, in.n));
    KICP_TRY(kicp_enqueue_widen(m->ctx, &in, m->d_in));
    *xyz = m->d_in;
    return KICP_OK;
}

// AddPoints (pose7 null) or the insert half of Update(points, pose) from a device cloud: one synchronisation, like the host variants
static int map_add_points_device(kicp_map *m, const kicp_frame_input &in, const double *pose7, const char *fn) {
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    if (!m) return kicp_invalid(fn, "null map");
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    const double *xyz = nullptr;
    KICP_TRY(map_device_points(m, in, packed, &xyz));
    return map_add_points_impl(m, xyz, in.n, pose7, true);
}
extern "C" int kicp_map_add_points_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                          int32_t offset_y, int32_t offset_z) {
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    return map_add_points_device(m, in, nullptr, "kicp_map_add_points_device");
}
extern "C" int kicp_map_update_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                      int32_t offset_y, int32_t offset_z, const double origin[3]) {
    static const char fn[] = "kicp_map_update_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    if (!origin) return kicp_invalid(fn, "origin: null pointer");
    KICP_TRY(map_add_points_device(m, in, nullptr, fn));
    return kicp_map_remove_far(m, origin);
}
extern "C" int kicp_map_update_pose_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                           int32_t offset_y, int32_t offset_z, const double pose[7]) {
    static const char fn[] = "kicp_map_update_pose_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    if (!pose) return kicp_invalid(fn, "pose: null pointer");
    KICP_TRY(map_add_points_device(m, in, pose, fn));
    return kicp_map_remove_far(m, pose + 4);
}

// local_map_.Update(frame, pose) (KinematicICP.cpp:79) for a frame whose point count (`d_n` <= n_max) and pose (`d_res`) are
// still being computed on the stream: everything is enqueued, nothing is read back.  The counters are copied to `h_counters`
// (pinned, 8 words); after the caller's end-of-frame synchronisation, kicp_map_finish_update() brings the host mirrors up to date.
int kicp_map_update_pose_async(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const kicp_reg_result *d_res,
                               uint32_t *h_counters, const kicp_free_space_params *fs, const double fs_origin[3],
                               kicp_free_space_stats *h_fs) {
    if (!m || n_max <= 0 || !d_xyz || !d_n || !d_res || !h_counters || (fs && (!fs_origin || !h_fs))) return KICP_ERR_INVALID;
    KICP_TRY(map_insert(m, d_xyz, true, n_max, nullptr, d_n, d_res));
    // RemovePointsFarFromLocation(pose.translation()) over the blocks that exist now: at most ub
    const uint32_t ub = (uint32_t)std::min<uint64_t>((uint64_t)m->num_blocks + (uint64_t)n_max, m->blocks_cap);
    // free-space clearing: the frame's rays against the map after the insert, decided after the eviction
    if (fs) KICP_TRY(enqueue_free_rays(m, d_xyz, n_max, d_n, nullptr, d_res, fs_origin, *fs, ub));
    const double unused[3] = {0.0, 0.0, 0.0};
    KICP_TRY(map_evict(m, unused, d_res, ub, fs ? (uint32_t)fs->min_misses : 0u));
    KICP_CUDA(cudaMemcpyAsync(h_counters, m->d_counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, m->ctx->stream));
    static_assert(sizeof(kicp_free_space_stats) <= kFreeStatWords * sizeof(unsigned long long), "statistics words");
    if (fs) KICP_CUDA(cudaMemcpyAsync(h_fs, m->d_free_stats, sizeof(kicp_free_space_stats), cudaMemcpyDeviceToHost, m->ctx->stream));
    return KICP_OK;
}

// Free-space clearing of the n rays of d_xyz (packed doubles in HBM, valid until the call returns) at a host pose, synchronously: the
// flags, k_free_rays and k_mark_free, ONE read-back of the counters and the statistics, and (when a live voxel was cleared) the
// eviction's compaction and table restore.  The host mirrors are current when it returns.
int kicp_map_clear_free_space_packed(kicp_map *m, const double *d_xyz, int64_t n, const double pose[7], const double origin[3],
                                     const kicp_free_space_params *p, kicp_free_space_stats *stats) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    kicp_free_space_stats st{};
    if (n > 0) {
        const uint32_t nb = m->num_blocks;
        const uint32_t init[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        KICP_CUDA(cudaMemcpyAsync(m->d_counters, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
        KICP_TRY(enqueue_free_rays(m, d_xyz, n, nullptr, pose, nullptr, origin, *p, nb));
        if (nb) KICP_TRY(enqueue_mark_free(m, nb, (uint32_t)p->min_misses, nullptr));
        uint32_t res[8];
        KICP_CUDA(cudaMemcpyAsync(res, m->d_counters, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaMemcpyAsync(&st, m->d_free_stats, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        if (res[4]) KICP_TRY(map_compact(m, nullptr, nb, res));
    }
    if (stats) *stats = st;
    return KICP_OK;
}

// the checks of the clearing calls after their cloud's: pose, origin and parameters, the map last
static int free_space_args(kicp_map *m, const char *fn, const double *pose, const double *origin, const kicp_free_space_params *p) {
    if (!pose) return kicp_invalid(fn, "pose: null pointer");
    if (!origin) return kicp_invalid(fn, "sensor_origin: null pointer");
    if (!p) return kicp_invalid(fn, "params: null pointer");
    for (int k = 0; k < 7; ++k)
        if (!std::isfinite(pose[k])) return kicp_invalid(fn, "pose: not finite");
    for (int k = 0; k < 3; ++k)
        if (!std::isfinite(origin[k])) return kicp_invalid(fn, "sensor_origin: not finite");
    KICP_TRY(kicp_check_free_space_params(fn, p, false));
    if (!m) return kicp_invalid(fn, "null map");
    return KICP_OK;
}
int kicp_check_free_space_params(const char *fn, const kicp_free_space_params *p, bool allow_off) {
    if (!(p->end_margin >= 0.0) || std::isinf(p->end_margin)) return kicp_invalid(fn, "params->end_margin: NaN, negative or infinite");
    if (p->min_misses < (allow_off ? 0 : 1)) return kicp_invalid(fn, allow_off ? "params->min_misses: negative" : "params->min_misses: < 1");
    return KICP_OK;
}

extern "C" int kicp_map_clear_free_space(kicp_map *m, const double *xyz, int64_t n, const double pose[7], const double sensor_origin[3],
                                         const kicp_free_space_params *params, kicp_free_space_stats *stats) {
    static const char fn[] = "kicp_map_clear_free_space";
    if (n < 0) return kicp_invalid(fn, "n < 0");
    if (n >= (1ll << 40)) return kicp_invalid(fn, "n: 2^40 points or more");
    if (n > 0 && !xyz) return kicp_invalid(fn, "xyz: null pointer");
    KICP_TRY(free_space_args(m, fn, pose, sensor_origin, params));
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    if (n > 0) {
        KICP_TRY(map_reserve_input(m, n));
        KICP_CUDA(cudaMemcpyAsync(m->d_in, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, m->ctx->stream));
    }
    return kicp_map_clear_free_space_packed(m, m->d_in, n, pose, sensor_origin, params, stats);
}

extern "C" int kicp_map_clear_free_space_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                                int32_t offset_y, int32_t offset_z, const double pose[7], const double sensor_origin[3],
                                                const kicp_free_space_params *params, kicp_free_space_stats *stats) {
    static const char fn[] = "kicp_map_clear_free_space_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    KICP_TRY(free_space_args(m, fn, pose, sensor_origin, params));
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    const double *xyz = nullptr;
    KICP_TRY(map_device_points(m, in, packed, &xyz));
    return kicp_map_clear_free_space_packed(m, xyz, n, pose, sensor_origin, params, stats);
}

// ---------------------------------------------------------------------------------------------------- occupancy evidence
// The setting of the map, checked field by field (the map last); a set call (re)allocates the evidence and its spare array for the
// block capacity and fills both with `initial` (the spare's copy of a frozen prefix included); NULL frees them.
extern "C" int kicp_map_set_occupancy(kicp_map *m, const kicp_occupancy_params *p) {
    static const char fn[] = "kicp_map_set_occupancy";
    constexpr int32_t kMax = 1 << 24;
    if (p) {
        if (p->max_evidence < 1 || p->max_evidence > kMax) return kicp_invalid(fn, "params->max_evidence: outside [1, 2^24]");
        if (p->initial < 1 || p->initial > p->max_evidence) return kicp_invalid(fn, "params->initial: outside [1, max_evidence]");
        if (p->hit_gain < 0 || p->hit_gain > kMax) return kicp_invalid(fn, "params->hit_gain: outside [0, 2^24]");
        if (p->miss_loss < 1 || p->miss_loss > kMax) return kicp_invalid(fn, "params->miss_loss: outside [1, 2^24]");
    }
    if (!m) return kicp_invalid(fn, "null map");
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    if (!p || m->occ_cap < m->blocks_cap) {
        cudaFree(m->occ_slab);
        m->occ_slab = m->d_occ = m->d_occ_spare = nullptr, m->occ_cap = 0, m->occ = kicp_occupancy_params{0, 0, 0, 0};
        if (!p) return KICP_OK;
        KICP_CUDA(cudaMalloc(&m->occ_slab, (size_t)2 * m->blocks_cap * sizeof(int32_t)));
        m->occ_cap = m->blocks_cap;
    }
    m->d_occ = m->occ_slab, m->d_occ_spare = m->occ_slab + m->occ_cap;
    k_fill_i32<<<(2 * m->occ_cap + 255) / 256, 256, 0, c->stream>>>(m->occ_slab, p->initial, 2 * m->occ_cap);
    KICP_CHECK_LAUNCH(c);
    m->occ = *p;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

extern "C" int kicp_map_export_occupancy(kicp_map *m, int32_t *evidence, int64_t cap, int64_t *n) {
    static const char fn[] = "kicp_map_export_occupancy";
    if (!n) return kicp_invalid(fn, "n: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    if (!m->d_occ) return kicp_invalid(fn, "occupancy is off (kicp_map_set_occupancy)");
    *n = m->num_blocks;
    if (cap < *n) return KICP_ERR_CAPACITY;
    if (*n == 0) return KICP_OK;
    if (!evidence) return kicp_invalid(fn, "evidence: null pointer");
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    KICP_CUDA(cudaMemcpyAsync(evidence, m->d_occ, (size_t)*n * sizeof(int32_t), cudaMemcpyDeviceToHost, m->ctx->stream));
    KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
    return KICP_OK;
}

// Pointcloud / export: the stored points are packed ON THE DEVICE (k_block_counts + k_exclusive_sum + k_pack_points, block order,
// insertion order inside a block — the order the host loop used to produce) and exactly num_points * sizeof(T) * 3 bytes cross PCIe,
// instead of the padded block array (20 slots of 32 bytes per voxel whatever it holds).  The spare point array is the scratch: it
// holds nothing between two evictions but the mirrored prior prefix [0, P), so the packing starts after it (or, when the rest of the
// spare is too small for the packed cloud, goes to a buffer of this call).
// One layer (KICP_MAP_LAYER_*) is one range of blocks: ALL [0, nb), PRIOR [0, P), LIVE [P, nb).
struct LayerRange {
    uint32_t b0, nb;
    int64_t points;
};
static LayerRange map_layer(const kicp_map *m, int layer) {
    const uint32_t P = m->prior_blocks;
    if (layer == KICP_MAP_LAYER_PRIOR) return LayerRange{0, P, m->prior_points};
    if (layer == KICP_MAP_LAYER_LIVE) return LayerRange{P, m->num_blocks - P, m->num_points - m->prior_points};
    return LayerRange{0, m->num_blocks, m->num_points};
}
// packed xyz of the layer's stored points -> host `out_xyz` (points * 3 doubles, or float32 records for T = float); headers -> `hdr`
// when asked for.  A `device` out_xyz is packed into directly, on the context stream, without a copy or a host synchronisation.
template <class T>
static int map_download_packed(kicp_map *m, T *out_xyz, std::vector<int4> *hdr, bool device = false, int layer = KICP_MAP_LAYER_ALL) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    const LayerRange L = map_layer(m, layer);
    if (L.nb == 0) return KICP_OK;
    const int4 *blk = m->blk + L.b0;
    const double *pts = m->pts + (size_t)L.b0 * m->cap * KICP_PSTRIDE;
    k_block_counts<<<(L.nb + 255) / 256, 256, 0, c->stream>>>(blk, L.nb, m->d_keep);
    KICP_CHECK_LAUNCH(c);
    if (L.points >= (1ll << 30)) {
        kicp_set_error("voxel map: export of 2^30 points or more is not supported");
        return KICP_ERR_CAPACITY;
    }
    KICP_TRY(enqueue_exclusive_sum(c, m->d_keep, m->d_new_id, L.nb));
    const size_t spare_off = (size_t)m->prior_blocks * m->cap * KICP_PSTRIDE;
    const size_t spare_room = ((size_t)m->blocks_cap * m->cap * KICP_PSTRIDE - spare_off) * sizeof(double);
    const size_t packed_bytes = (size_t)L.points * 3 * sizeof(T);
    T *scratch = nullptr;
    if (!device && packed_bytes > spare_room) KICP_CUDA(cudaMalloc(&scratch, packed_bytes));
    T *packed = device ? out_xyz : scratch ? scratch : reinterpret_cast<T *>(m->pts_spare + spare_off);
    k_pack_points<T><<<(unsigned)(((uint64_t)L.nb * 32 + 255) / 256), 256, 0, c->stream>>>(blk, pts, (int)m->cap, L.nb, m->d_new_id,
                                                                                          packed);
    c->launches++;  // KICP_CHECK_LAUNCH, with the scratch freed on every path
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && !device) {
        e = cudaMemcpyAsync(out_xyz, packed, packed_bytes, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess && hdr) {
            hdr->resize(L.nb);
            e = cudaMemcpyAsync(hdr->data(), blk, hdr->size() * sizeof(int4), cudaMemcpyDeviceToHost, c->stream);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    }
    cudaFree(scratch);
    if (e != cudaSuccess) return kicp_cuda_fail(e, "map_download_packed", __FILE__, __LINE__);
    return KICP_OK;
}

template <class T>
static int map_pointcloud(kicp_map *m, T *out_xyz, int64_t cap, int64_t *n, bool device = false, int layer = KICP_MAP_LAYER_ALL,
                          const char *fn = "kicp_map_pointcloud_device_async") {
    if (!m || !n || (device && !out_xyz)) return KICP_ERR_INVALID;
    const int64_t points = map_layer(m, layer).points;
    *n = points;
    if (device)
        KICP_TRY(kicp_check_device_range(m->ctx, out_xyz, (size_t)std::max<int64_t>(1, std::min(cap, points)) * 3 * sizeof(T),
                                         sizeof(T), (std::string(fn) + ": out").c_str()));
    if (points > cap) return KICP_ERR_CAPACITY;
    if (points == 0) return KICP_OK;
    if (!out_xyz) return KICP_ERR_INVALID;
    return map_download_packed(m, out_xyz, nullptr, device, layer);
}

extern "C" int kicp_map_pointcloud(kicp_map *m, double *out_xyz, int64_t cap, int64_t *n) { return map_pointcloud(m, out_xyz, cap, n); }

// Pointcloud() as the float32 records EigenToPointCloud2 builds from it (RosUtils.cpp:41-63): the same order, half the bytes, and
// the narrowing done on the device by the reference's x86-64 rule (to_f32_x86)
extern "C" int kicp_map_pointcloud_f32(kicp_map *m, float *out_xyz, int64_t cap, int64_t *n) { return map_pointcloud(m, out_xyz, cap, n); }

// Pointcloud() (F64) or kicp_map_pointcloud_f32's records (F32) packed by k_pack_points straight into the caller's device memory
extern "C" int kicp_map_pointcloud_device_async(kicp_map *m, void *out, int32_t dtype, int64_t cap, int64_t *n) {
    if (dtype == KICP_DTYPE_F64) return map_pointcloud(m, static_cast<double *>(out), cap, n, true);
    if (dtype == KICP_DTYPE_F32) return map_pointcloud(m, static_cast<float *>(out), cap, n, true);
    return KICP_ERR_INVALID;
}

// one layer of the map (KICP_MAP_LAYER_*), by the rules of the whole-map calls above; the arguments are checked before the map
static int map_pointcloud_layer(kicp_map *m, int32_t layer, int32_t dtype, void *out, int64_t cap, int64_t *n, bool device, const char *fn) {
    if (layer != KICP_MAP_LAYER_ALL && layer != KICP_MAP_LAYER_PRIOR && layer != KICP_MAP_LAYER_LIVE)
        return kicp_invalid(fn, "layer: not KICP_MAP_LAYER_ALL, KICP_MAP_LAYER_PRIOR or KICP_MAP_LAYER_LIVE");
    if (dtype != KICP_DTYPE_F64 && dtype != KICP_DTYPE_F32) return kicp_invalid(fn, "dtype: not KICP_DTYPE_F64 or KICP_DTYPE_F32");
    if (!n) return kicp_invalid(fn, "n: null pointer");
    if (device && !out) return kicp_invalid(fn, "out: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    const int64_t points = map_layer(m, layer).points;
    if (!device && !out && points > 0 && cap >= points) return kicp_invalid(fn, "out: null pointer");
    if (dtype == KICP_DTYPE_F64) return map_pointcloud(m, static_cast<double *>(out), cap, n, device, layer, fn);
    return map_pointcloud(m, static_cast<float *>(out), cap, n, device, layer, fn);
}
extern "C" int kicp_map_pointcloud_layer(kicp_map *m, int32_t layer, int32_t dtype, void *out, int64_t cap, int64_t *n) {
    return map_pointcloud_layer(m, layer, dtype, out, cap, n, false, "kicp_map_pointcloud_layer");
}
extern "C" int kicp_map_pointcloud_layer_device_async(kicp_map *m, int32_t layer, int32_t dtype, void *out, int64_t cap, int64_t *n) {
    return map_pointcloud_layer(m, layer, dtype, out, cap, n, true, "kicp_map_pointcloud_layer_device_async");
}

// ------------------------------------------------------------------------------------------- live local-map cloud
#include "kicp_map_live_kernels.cuh"  // struct LiveArgs and the k_live_* kernels

// State of kicp_map_pointcloud_f32_live.  The published records, the published voxels and their slot positions persist from call to
// call; the other device arrays are scratch of one call.  Position arrays hold rec_cap positions, voxel arrays vox_cap voxels (times
// max_points_per_voxel for the slot positions); both grow, keeping what the next call reads, and never shrink.
struct MapLive {
    float *h_rec = nullptr;  // the published records, page-locked: the buffer the caller reads
    int64_t h_cap = 0;       // records it holds
    int64_t n = 0;           // records published by the previous call
    uint32_t num_pub = 0;    // voxels published by the previous call
    int64_t rec_cap = 0, vox_cap = 0;
    float *rec = nullptr;  // device mirror of h_rec
    uint32_t *owner = nullptr, *hole = nullptr, *rank = nullptr, *hole_list = nullptr;
    int4 *pub = nullptr;
    uint32_t *pos_old = nullptr, *pos_new = nullptr, *new_cnt = nullptr, *new_base = nullptr;
    int32_t *match = nullptr;
    uint32_t *d_ctr = nullptr, *h_ctr = nullptr;  // [0] removed [1] rewritten [2] moved
};

static void map_live_free(kicp_map *m) {
    MapLive *L = m->live;
    if (!L) return;
    cudaFreeHost(L->h_rec), cudaFreeHost(L->h_ctr);
    cudaFree(L->rec), cudaFree(L->owner), cudaFree(L->hole), cudaFree(L->rank), cudaFree(L->hole_list);
    cudaFree(L->pub), cudaFree(L->pos_old), cudaFree(L->pos_new), cudaFree(L->new_cnt), cudaFree(L->new_base), cudaFree(L->match);
    cudaFree(L->d_ctr);
    delete L;
    m->live = nullptr;
}

// replace p by an allocation of `bytes` that starts with p's first `keep` bytes (the stream has drained)
template <class T>
static int live_realloc(T *&p, size_t bytes, size_t keep) {
    void *q = nullptr;
    KICP_CUDA(cudaMalloc(&q, bytes));
    if (keep) {
        cudaError_t e = cudaMemcpy(q, p, keep, cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) {
            cudaFree(q);
            return kicp_cuda_fail(e, "cudaMemcpy", __FILE__, __LINE__);
        }
    }
    cudaFree(p);
    p = static_cast<T *>(q);
    return KICP_OK;
}

static int live_reserve(kicp_map *m, MapLive &L, int64_t recs, int64_t voxels) {
    const size_t u = sizeof(uint32_t);
    if (recs > L.rec_cap) {
        KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
        const size_t cap = (size_t)std::max<int64_t>(recs + recs / 4, 4096);
        KICP_TRY(live_realloc(L.rec, cap * 3 * sizeof(float), (size_t)L.n * 3 * sizeof(float)));
        KICP_TRY(live_realloc(L.owner, cap * u, 0));
        KICP_TRY(live_realloc(L.hole, cap * u, 0));
        KICP_TRY(live_realloc(L.rank, cap * u, 0));
        KICP_TRY(live_realloc(L.hole_list, cap * u, 0));
        L.rec_cap = (int64_t)cap;
    }
    if (voxels > L.vox_cap) {
        KICP_CUDA(cudaStreamSynchronize(m->ctx->stream));
        const size_t cap = (size_t)std::max<int64_t>(voxels + voxels / 4, 1024);
        KICP_TRY(live_realloc(L.pub, cap * sizeof(int4), (size_t)L.num_pub * sizeof(int4)));
        KICP_TRY(live_realloc(L.pos_old, cap * m->cap * u, (size_t)L.num_pub * m->cap * u));
        KICP_TRY(live_realloc(L.pos_new, cap * m->cap * u, 0));
        KICP_TRY(live_realloc(L.new_cnt, cap * u, 0));
        KICP_TRY(live_realloc(L.new_base, cap * u, 0));
        KICP_TRY(live_realloc(L.match, cap * sizeof(int32_t), 0));
        L.vox_cap = (int64_t)cap;
    }
    return KICP_OK;
}

// One call of kicp_map_pointcloud_f32_live: the launch sequence of kicp_map_live_kernels.cuh, then ONE synchronisation.  `grown`:
// the new host buffer when the map outgrew the old one (the kernels then write the mirror only, and the mirror is copied whole).
static int live_update(kicp_map *m, MapLive &L, float *grown, kicp_map_live_stats *st) {
    kicp_ctx *c = m->ctx;
    const int64_t n_old = L.n, n_new = m->num_points;
    const uint32_t nb = m->num_blocks, npub = L.num_pub;
    const int cap = (int)m->cap;
    KICP_TRY(live_reserve(m, L, std::max(n_old, n_new), std::max<int64_t>(nb, npub)));
    const LiveArgs a{L.rec, grown ? nullptr : L.h_rec, L.owner, L.pub, L.pos_old, L.pos_new, L.match, L.new_cnt, L.new_base,
                     L.hole, L.rank, L.hole_list, L.d_ctr, n_old, n_new};
    KICP_CUDA(cudaMemsetAsync(L.d_ctr, 0, 4 * sizeof(uint32_t), c->stream));
    if (nb) {
        k_live_init<<<(nb + 255) / 256, 256, 0, c->stream>>>(m->blk, nb, a);
        KICP_CHECK_LAUNCH(c);
    }
    if (npub) {
        k_live_match<<<(unsigned)(((uint64_t)npub * 32 + 255) / 256), 256, 0, c->stream>>>(m->view(), m->blk, npub, a);
        KICP_CHECK_LAUNCH(c);
    }
    KICP_TRY(enqueue_exclusive_sum(c, L.new_cnt, L.new_base, nb));
    KICP_TRY(enqueue_exclusive_sum(c, L.hole, L.rank, (uint32_t)n_old));
    if (n_old) {
        k_live_holes<<<(unsigned)((n_old + 255) / 256), 256, 0, c->stream>>>(a);
        KICP_CHECK_LAUNCH(c);
    }
    if (nb) {
        k_live_add<<<(unsigned)(((uint64_t)nb * 32 + 255) / 256), 256, 0, c->stream>>>(m->blk, m->pts, cap, nb, a);
        KICP_CHECK_LAUNCH(c);
    }
    if (n_old > n_new) {
        k_live_move<<<(unsigned)((n_old - n_new + 255) / 256), 256, 0, c->stream>>>(m->pts, cap, a);
        KICP_CHECK_LAUNCH(c);
    }
    if (nb) KICP_CUDA(cudaMemcpyAsync(L.pub, m->blk, (size_t)nb * sizeof(int4), cudaMemcpyDeviceToDevice, c->stream));
    if (grown && n_new) KICP_CUDA(cudaMemcpyAsync(grown, L.rec, (size_t)n_new * 3 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaMemcpyAsync(L.h_ctr, L.d_ctr, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    std::swap(L.pos_old, L.pos_new);
    L.num_pub = nb, L.n = n_new;
    st->removed = L.h_ctr[0], st->rewritten = L.h_ctr[1], st->moved = L.h_ctr[2];
    st->added = n_new - n_old + st->removed;
    st->written = grown ? n_new : st->added + st->moved + st->rewritten;
    return KICP_OK;
}

extern "C" int kicp_map_pointcloud_f32_live(kicp_map *m, const float **records, int64_t *n, kicp_map_live_stats *stats) {
    if (!m || !records || !n) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    if (m->num_points >= (1ll << 30)) {
        kicp_set_error("voxel map: a live cloud of 2^30 points or more is not supported");
        return KICP_ERR_CAPACITY;
    }
    if (!m->live) {
        MapLive *L = new MapLive();
        m->live = L;
        KICP_CUDA(cudaMallocHost(&L->h_ctr, 4 * sizeof(uint32_t)));
        KICP_CUDA(cudaMalloc(&L->d_ctr, 4 * sizeof(uint32_t)));
    }
    MapLive &L = *m->live;
    float *grown = nullptr;
    int64_t grown_cap = 0;
    if (!L.h_rec || m->num_points > L.h_cap) {
        grown_cap = std::max<int64_t>(m->num_points + m->num_points / 4, 4096);
        KICP_CUDA(cudaMallocHost(&grown, (size_t)grown_cap * 3 * sizeof(float)));
    }
    kicp_map_live_stats st{};
    const int s = live_update(m, L, grown, &st);
    if (s != KICP_OK) {
        // the device state may be half updated: publish everything anew next time (the buffer itself stays valid)
        cudaStreamSynchronize(m->ctx->stream);
        cudaFreeHost(grown);
        L.n = 0, L.num_pub = 0;
        return s;
    }
    if (grown) {
        cudaFreeHost(L.h_rec);
        L.h_rec = grown, L.h_cap = grown_cap;
    }
    *records = L.h_rec;
    *n = L.n;
    if (stats) *stats = st;
    return KICP_OK;
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
    if (m->d_occ) {  // occupancy on: every loaded voxel starts at `initial`
        k_fill_i32<<<(unsigned)((num_voxels + 255) / 256), 256, 0, c->stream>>>(m->d_occ, m->occ.initial, (uint32_t)num_voxels);
        KICP_CHECK_LAUNCH(c);
    }
    m->num_blocks = (uint32_t)num_voxels;
    m->num_points = total;
    int st = map_rebuild_table(m, m->nslots, m->num_blocks);
    cudaError_t e = cudaStreamSynchronize(c->stream);
    cudaFree(d_keys), cudaFree(d_counts), cudaFree(d_off), cudaFree(d_pts);
    if (st != KICP_OK) return st;
    if (e != cudaSuccess) return kicp_cuda_fail(e, "load_voxels", __FILE__, __LINE__);
    return KICP_OK;
}

// GetClosestNeighbor of n > 0 queries at d_q (packed doubles in HBM) into d_points / d_dist, enqueued on the context stream: a warp per
// query, four per CTA (at its 54 registers a thread, nine CTAs of 128 threads fit on an SM against four of 256), the grid capped
// (k_nearest strides over the queries beyond it)
static int enqueue_nearest(kicp_map *m, const double *d_q, int64_t n, double *d_points, double *d_dist) {
    kicp_ctx *c = m->ctx;
    const unsigned grid = (unsigned)std::min<int64_t>((n + 3) / 4, 1 << 20);
    k_nearest<<<grid, 128, 0, c->stream>>>(m->view(), d_q, n, d_points, d_dist);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// host queries: copied into the map's input buffer, the results into its own buffers, which grow and are kept from call to call
extern "C" int kicp_map_nearest(kicp_map *m, const double *queries, int64_t n, double *out_points, double *out_dist) {
    if (!m || n < 0 || (n > 0 && (!queries || !out_points || !out_dist))) return KICP_ERR_INVALID;
    if (n == 0) return KICP_OK;
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(map_reserve_input(m, n));
    KICP_CUDA(cudaMemcpyAsync(m->d_in, queries, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    KICP_TRY(enqueue_nearest(m, m->d_in, n, m->d_xyz_t, m->d_dist));
    KICP_CUDA(cudaMemcpyAsync(out_points, m->d_xyz_t, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaMemcpyAsync(out_dist, m->d_dist, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

// device queries: read in place (packed doubles) or widened into the map's input buffer; the results go straight to the caller's
// device memory, and nothing waits for them
extern "C" int kicp_map_nearest_device_async(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                             int32_t offset_y, int32_t offset_z, double *out_points, double *out_dist) {
    static const char fn[] = "kicp_map_nearest_device_async";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    if (n > 0 && !out_points) return kicp_invalid(fn, "out_points: null pointer");
    if (n > 0 && !out_dist) return kicp_invalid(fn, "out_dist: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    if (n == 0) return KICP_OK;
    KICP_TRY(kicp_check_device_range(m->ctx, out_points, (size_t)n * 3 * sizeof(double), sizeof(double),
                                     (std::string(fn) + ": out_points").c_str()));
    KICP_TRY(kicp_check_device_range(m->ctx, out_dist, (size_t)n * sizeof(double), sizeof(double), (std::string(fn) + ": out_dist").c_str()));
    const double *q = nullptr;
    KICP_TRY(map_device_points(m, in, packed, &q));
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    return enqueue_nearest(m, q, n, out_points, out_dist);
}

// ---------------------------------------------------------------------------------------------------------- correspondences
#include "kicp_corr_kernels.cuh"  // k_corr_eval, k_corr_finish

// KICP_OK when `stats` is device memory of the context's device or page-locked host memory (what a copy on the stream can write
// without waiting); otherwise KICP_ERR_INVALID naming it
static int check_stats_memory(const kicp_ctx *c, const void *p, const char *what) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return kicp_invalid(what, "not memory the CUDA runtime knows");
    }
    if (at.type == cudaMemoryTypeHost) return KICP_OK;
    if (reinterpret_cast<uintptr_t>(p) % alignof(kicp_corr_stats)) return kicp_invalid(what, "not aligned to 8 bytes");
    return kicp_check_device_range(c, p, sizeof(kicp_corr_stats), alignof(kicp_corr_stats), what);
}

// k_corr_eval's grid: as many 256-thread CTAs as are resident at once (the warps stride over the points beyond them), fewer for a
// small n; the partials are allocated for the resident grid on first use
static int corr_reserve(kicp_map *m) {
    if (m->d_corr_part) return KICP_OK;
    int per_sm = 0;
    KICP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_corr_eval, kCorrThreads, 0));
    const int grid = std::max(1, per_sm) * m->ctx->sm_count;
    KICP_CUDA(cudaMalloc(&m->d_corr_part, (size_t)grid * kCorrStride * sizeof(double)));
    KICP_CUDA(cudaMalloc(&m->d_corr_stats, sizeof(kicp_corr_stats)));
    m->corr_grid = grid;
    return KICP_OK;
}

int kicp_map_enqueue_correspondences(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double *pose7,
                                     const kicp_reg_result *d_res, double tau, double *d_points, double *d_dist, uint8_t *d_inlier,
                                     kicp_corr_stats *stats) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(corr_reserve(m));
    const int per_cta = kCorrThreads / 32;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_max + per_cta - 1) / per_cta, m->corr_grid));
    Pose pose{0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    k_corr_eval<<<grid, kCorrThreads, 0, c->stream>>>(m->view(), d_xyz, n_max, d_n, pose, d_res, tau, d_points, d_dist, d_inlier,
                                                      m->d_corr_part);
    KICP_CHECK_LAUNCH(c);
    k_corr_finish<<<1, 32, 0, c->stream>>>(m->d_corr_part, grid, n_max, d_n, m->d_corr_stats);
    KICP_CHECK_LAUNCH(c);
    if (stats) KICP_CUDA(cudaMemcpyAsync(stats, m->d_corr_stats, sizeof(kicp_corr_stats), cudaMemcpyDefault, c->stream));
    return KICP_OK;
}

// host points: copied into the map's input buffer, the per-point results into its own buffers (kicp_map_nearest's), then to the host
extern "C" int kicp_map_correspondences(kicp_map *m, const double *xyz, int64_t n, const double pose[7], double tau, double *out_points,
                                        double *out_dist, uint8_t *out_inlier, kicp_corr_stats *stats) {
    static const char fn[] = "kicp_map_correspondences";
    if (n < 0) return kicp_invalid(fn, "n < 0");
    if (n > 0 && !xyz) return kicp_invalid(fn, "xyz: null pointer");
    if (!pose) return kicp_invalid(fn, "pose: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(map_reserve_input(m, std::max<int64_t>(n, 1)));
    if (out_inlier && n > m->corr_inl_cap) {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(m->d_corr_inl);
        m->d_corr_inl = nullptr, m->corr_inl_cap = 0;
        const int64_t cap = std::max<int64_t>(n + n / 4, 4096);
        KICP_CUDA(cudaMalloc(&m->d_corr_inl, (size_t)cap));
        m->corr_inl_cap = cap;
    }
    if (n) KICP_CUDA(cudaMemcpyAsync(m->d_in, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    KICP_TRY(kicp_map_enqueue_correspondences(m, m->d_in, n, nullptr, pose, nullptr, tau, out_points ? m->d_xyz_t : nullptr,
                                              out_dist ? m->d_dist : nullptr, out_inlier ? m->d_corr_inl : nullptr, nullptr));
    if (out_points && n) KICP_CUDA(cudaMemcpyAsync(out_points, m->d_xyz_t, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (out_dist && n) KICP_CUDA(cudaMemcpyAsync(out_dist, m->d_dist, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (out_inlier && n) KICP_CUDA(cudaMemcpyAsync(out_inlier, m->d_corr_inl, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    if (stats) KICP_CUDA(cudaMemcpyAsync(stats, m->d_corr_stats, sizeof(kicp_corr_stats), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

// device points: read in place (packed doubles) or widened into the map's input buffer; the results go straight to the caller's
// memory, and nothing waits for them
extern "C" int kicp_map_correspondences_device_async(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step,
                                                     int32_t offset_x, int32_t offset_y, int32_t offset_z, const double pose[7], double tau,
                                                     double *out_points, double *out_dist, uint8_t *out_inlier, kicp_corr_stats *stats) {
    static const char fn[] = "kicp_map_correspondences_device_async";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));
    if (!pose) return kicp_invalid(fn, "pose: null pointer");
    if (!m) return kicp_invalid(fn, "null map");
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    const std::string f(fn);
    if (n > 0 && out_points)
        KICP_TRY(kicp_check_device_range(m->ctx, out_points, (size_t)n * 3 * sizeof(double), sizeof(double), (f + ": out_points").c_str()));
    if (n > 0 && out_dist)
        KICP_TRY(kicp_check_device_range(m->ctx, out_dist, (size_t)n * sizeof(double), sizeof(double), (f + ": out_dist").c_str()));
    if (n > 0 && out_inlier) KICP_TRY(kicp_check_device_range(m->ctx, out_inlier, (size_t)n, 1, (f + ": out_inlier").c_str()));
    if (stats) KICP_TRY(check_stats_memory(m->ctx, stats, (f + ": stats").c_str()));
    const double *q = nullptr;
    KICP_TRY(map_device_points(m, in, packed, &q));
    return kicp_map_enqueue_correspondences(m, q, n, nullptr, pose, nullptr, tau, out_points, out_dist, out_inlier, stats);
}

// ---------------------------------------------------------------------------------------------------------- pose search
#include "kicp_pose_search_kernels.cuh"  // k_pose_score, k_pose_select; the host logic of kicp_pose_search.h

// Device buffers of kicp_map_pose_search*, grown on demand and kept: the widened points, a level's tables, the scores and two entry
// lists for k_pose_select's passes.  A repeated call of the same size allocates nothing.
struct PoseScratch {
    double *pts = nullptr, *rot = nullptr, *trans = nullptr, *sum = nullptr;
    int32_t *pair_t = nullptr, *lat = nullptr, *tiles = nullptr;
    int64_t *cnt = nullptr;
    PsEntry *ent[2] = {nullptr, nullptr};
    size_t pts_cap = 0, rot_cap = 0, trans_cap = 0, pair_cap = 0, lat_cap = 0, tiles_cap = 0, hyp_cap = 0, sum_cap = 0, ent_cap = 0;
    int score_grid = 0;
    PsTables tables;
    std::vector<PsEntry> best;
};

static void pose_scratch_free(kicp_map *m) {
    PoseScratch *S = m->pose;
    if (!S) return;
    cudaFree(S->pts), cudaFree(S->rot), cudaFree(S->trans), cudaFree(S->sum), cudaFree(S->pair_t), cudaFree(S->lat), cudaFree(S->tiles);
    cudaFree(S->cnt), cudaFree(S->ent[0]), cudaFree(S->ent[1]);
    delete S;
    m->pose = nullptr;
}

// `p` holds at least `need` elements (growth by 1.25x; the stream is drained before a buffer it may use is freed)
template <class T>
static int ps_grow(kicp_ctx *c, T *&p, size_t &cap, size_t need) {
    if (need <= cap) return KICP_OK;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    cudaFree(p);
    p = nullptr, cap = 0;
    const size_t n = std::max<size_t>(need + need / 4, 64);
    KICP_CUDA(cudaMalloc(&p, n * sizeof(T)));
    cap = n;
    return KICP_OK;
}

template <class T>
static int ps_upload(kicp_ctx *c, T *&d, size_t &cap, const std::vector<T> &h) {
    KICP_TRY(ps_grow(c, d, cap, h.size()));
    if (!h.empty()) KICP_CUDA(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, c->stream));
    return KICP_OK;
}

// Scores `n_hyp` hypotheses of the tables on the device and returns the best `keep` of them (one synchronisation)
static int ps_score_level(kicp_map *m, const double *d_pts, int64_t n, const PsPlan &P, bool level0, int64_t n_hyp,
                          std::vector<PsEntry> &best) {
    kicp_ctx *c = m->ctx;
    PoseScratch &S = *m->pose;
    KICP_TRY(ps_upload(c, S.rot, S.rot_cap, S.tables.rot));
    KICP_TRY(ps_upload(c, S.trans, S.trans_cap, S.tables.trans));
    int64_t n_tiles = 0;
    if (level0) {
        n_tiles = P.nr0 * ((P.nt0 + kPsTile - 1) / kPsTile);
    } else {
        KICP_TRY(ps_upload(c, S.pair_t, S.pair_cap, S.tables.pair_t));
        KICP_TRY(ps_upload(c, S.lat, S.lat_cap, S.tables.lat));
        KICP_TRY(ps_upload(c, S.tiles, S.tiles_cap, S.tables.tiles));
        n_tiles = (int64_t)S.tables.tiles.size() / 3;
    }
    const int per_cta = kPsThreads * kPsSelectItems;
    const int64_t parts = (n_hyp + per_cta - 1) / per_cta;
    KICP_TRY(ps_grow(c, S.cnt, S.hyp_cap, (size_t)n_hyp));
    KICP_TRY(ps_grow(c, S.sum, S.sum_cap, (size_t)n_hyp));
    const size_t ent_need = (size_t)parts * P.keep;
    if (ent_need > S.ent_cap) {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(S.ent[0]), cudaFree(S.ent[1]);
        S.ent[0] = S.ent[1] = nullptr, S.ent_cap = 0;
        const size_t e = ent_need + ent_need / 4;
        KICP_CUDA(cudaMalloc(&S.ent[0], e * sizeof(PsEntry)));
        KICP_CUDA(cudaMalloc(&S.ent[1], e * sizeof(PsEntry)));
        S.ent_cap = e;
    }
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(n_tiles, S.score_grid));
    k_pose_score<<<grid, kPsThreads, 0, c->stream>>>(m->view(), d_pts, n, S.rot, S.trans, level0 ? (int32_t)P.nt0 : 0,
                                                     level0 ? nullptr : S.pair_t, level0 ? nullptr : S.tiles, n_tiles, P.tau, S.cnt, S.sum);
    KICP_CHECK_LAUNCH(c);
    k_pose_select<<<(unsigned)parts, kPsThreads, 0, c->stream>>>(S.cnt, S.sum, level0 ? nullptr : S.lat, P.g, nullptr, n_hyp, per_cta,
                                                                  P.keep, S.ent[0]);
    KICP_CHECK_LAUNCH(c);
    int cur = 0;
    for (int64_t items = parts * P.keep; items > P.keep; items = ((items + per_cta - 1) / per_cta) * P.keep) {  // lists of lists
        const unsigned g = (unsigned)((items + per_cta - 1) / per_cta);
        k_pose_select<<<g, kPsThreads, 0, c->stream>>>(nullptr, nullptr, nullptr, P.g, S.ent[cur], items, per_cta, P.keep, S.ent[cur ^ 1]);
        KICP_CHECK_LAUNCH(c);
        cur ^= 1;
    }
    best.resize(P.keep);
    KICP_CUDA(cudaMemcpyAsync(best.data(), S.ent[cur], P.keep * sizeof(PsEntry), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

// The level loop over device points d_pts (packed doubles); validated arguments
static int ps_search(kicp_map *m, const double *d_pts, int64_t n, const double prior[7], const PsPlan &P, kicp_pose_hypothesis *out,
                     int32_t *n_out, int64_t *n_scored) {
    PoseScratch &S = *m->pose;
    ps_tables0(P, prior, S.tables);
    std::vector<PsKept> kept;
    KICP_TRY(ps_score_level(m, d_pts, n, P, true, P.n0, S.best));
    ps_merge(kept, S.best, 0, P.keep);
    PsScored scored{&P, {}, P.n0};
    for (int level = 1; level < P.levels; ++level) {
        std::vector<PsEntry> parents;
        for (const PsKept &k : kept) parents.push_back(k.e);
        const std::vector<std::array<int32_t, 3>> kids = ps_children(P, level, parents, scored);
        if (kids.empty()) continue;
        ps_tables(P, prior, kids, S.tables);
        KICP_TRY(ps_score_level(m, d_pts, n, P, false, (int64_t)kids.size(), S.best));
        ps_merge(kept, S.best, level, P.keep);
    }
    for (size_t i = 0; i < kept.size(); ++i) ps_output(P, prior, kept[i], n, &out[i]);
    *n_out = (int32_t)kept.size();
    if (n_scored) *n_scored = scored.count;
    return KICP_OK;
}

// the checks shared by both entry points, before any device work (the map last, so that every argument check is reachable without
// one); creates the scratch
static int ps_prepare(kicp_map *m, const char *fn, const double *prior, const kicp_pose_search_params *params, kicp_pose_hypothesis *out,
                      int32_t cap, int32_t *n_out, PsPlan *P) {
    if (!prior) return kicp_invalid(fn, "prior: null pointer");
    if (!params) return kicp_invalid(fn, "params: null pointer");
    if (!out) return kicp_invalid(fn, "out: null pointer");
    if (!n_out) return kicp_invalid(fn, "n_out: null pointer");
    for (int k = 0; k < 7; ++k)
        if (!std::isfinite(prior[k])) return kicp_invalid(fn, "prior: not finite");
    const std::string why = ps_plan(params, cap, P);
    if (!why.empty()) return kicp_invalid(fn, why.c_str());
    if (!m) return kicp_invalid(fn, "null map");
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    if (!m->pose) {  // the scratch is attached only once its grid is known, so a failed occupancy query is reported every call
        int per_sm = 0;
        KICP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pose_score, kPsThreads, 0));
        if (per_sm < 1) return kicp_invalid(fn, "k_pose_score cannot be resident on this device");
        m->pose = new PoseScratch();
        m->pose->score_grid = per_sm * m->ctx->sm_count;
    }
    return KICP_OK;
}

extern "C" int kicp_map_pose_search(kicp_map *m, const double *xyz, int64_t n, const double prior[7], const kicp_pose_search_params *params,
                                    kicp_pose_hypothesis *out, int32_t cap, int32_t *n_out, int64_t *n_scored) {
    static const char fn[] = "kicp_map_pose_search";
    if (n < 0) return kicp_invalid(fn, "n < 0");
    if (n >= kPsMaxPoints) return kicp_invalid(fn, "n: 2^40 points or more");
    if (n > 0 && !xyz) return kicp_invalid(fn, "xyz: null pointer");
    PsPlan P;
    KICP_TRY(ps_prepare(m, fn, prior, params, out, cap, n_out, &P));
    kicp_ctx *c = m->ctx;
    PoseScratch &S = *m->pose;
    KICP_TRY(ps_grow(c, S.pts, S.pts_cap, (size_t)std::max<int64_t>(n, 1) * 3));
    if (n) KICP_CUDA(cudaMemcpyAsync(S.pts, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    return ps_search(m, S.pts, n, prior, P, out, n_out, n_scored);
}

extern "C" int kicp_map_pose_search_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                           int32_t offset_y, int32_t offset_z, const double prior[7], const kicp_pose_search_params *params,
                                           kicp_pose_hypothesis *out, int32_t cap, int32_t *n_out, int64_t *n_scored) {
    static const char fn[] = "kicp_map_pose_search_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));  // also n < 2^30, well inside kPsMaxPoints
    PsPlan P;
    KICP_TRY(ps_prepare(m, fn, prior, params, out, cap, n_out, &P));
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    kicp_ctx *c = m->ctx;
    PoseScratch &S = *m->pose;
    const double *q = static_cast<const double *>(data);
    if (!packed && n > 0) {  // widened once into the search's own buffer (the map's input buffer is left alone)
        KICP_TRY(ps_grow(c, S.pts, S.pts_cap, (size_t)n * 3));
        KICP_TRY(kicp_enqueue_widen(c, &in, S.pts));
        q = S.pts;
    }
    return ps_search(m, q, n, prior, P, out, n_out, n_scored);
}
