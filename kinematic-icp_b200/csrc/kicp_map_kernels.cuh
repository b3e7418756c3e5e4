// Kernels of the device-resident kiss_icp::VoxelHashMap (included by kicp_map.cu, which is compiled with -fmad=false: every decision
// — voxel floor, the < map_resolution spacing test, the >= max_distance^2 eviction test, the nearest-neighbour argmin — is evaluated
// in plain IEEE double arithmetic in the reference's operation order).  A header of its own so that tests/emu can compile the kernels
// for the host against the SIMT emulator without the CUDA-runtime orchestration of kicp_map.cu.
#pragma once
#include <cfloat>

#include "kicp_device.cuh"
#include "kicp_nearest.cuh"  // warp_closest_neighbor
#include "kicp_scan.cuh"

using namespace kicp_dev;

// -------------------------------------------------------------------------------------------------- map kernels
// out[i] = in[0] + ... + in[i-1] for i < n (uint32, total < 2^30); grid = ceil(n / kScanTile) CTAs of kScanThreads threads
__global__ void __launch_bounds__(kScanThreads) k_exclusive_sum(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint32_t n,
                                                                kicp_scan_args a) {
    __shared__ uint32_t s_warp[kScanWarps + 1];
    const uint32_t tile = scan_take_tile(a, &s_warp[kScanWarps]);
    const int64_t i0 = scan_first_item(tile);
    uint32_t v[kScanItems], excl[kScanItems];
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int64_t i = i0 + 32 * k;
        v[k] = i < (int64_t)n ? in[i] : 0u;
    }
    const uint32_t warp_total = scan_warp_values(v, excl);
    uint32_t inclusive;
    const uint32_t base = scan_offset(a, tile, warp_total, s_warp, inclusive);
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int64_t i = i0 + 32 * k;
        if (i < (int64_t)n) out[i] = base + excl[k];
    }
}

struct MapRW {
    int4 *slots;
    uint32_t mask;
    int4 *blk;
    double *pts;
    int32_t *pend_head;
    uint32_t blocks_cap;
    int cap;
    double voxel_size;
};

// Insert a key known to be absent (rebuild / bulk load): claim the first empty slot of the probe chain.
__device__ __forceinline__ void table_insert_unique(int4 *slots, uint32_t mask, int kx, int ky, int kz, uint32_t meta) {
    uint32_t h = voxel_hash(kx, ky, kz) & mask;
    while (true) {
        const uint32_t old = atomicCAS((unsigned int *)&slots[h].w, KICP_SLOT_EMPTY, meta);
        if (old == KICP_SLOT_EMPTY) {
            slots[h].x = kx, slots[h].y = ky, slots[h].z = kz;
            return;
        }
        h = (h + 1) & mask;
    }
}

// `ctr` (optional): the block count lives on the device — blocks after the last AddPoints minus the ones just evicted.
// `first`: only blocks [first, num_blocks) are inserted (a frozen prior prefix [0, first) is already in the table, restored from its
// snapshot)
__global__ void k_table_rebuild(int4 *slots, uint32_t mask_in, const int4 *blk, uint32_t num_blocks, const uint32_t *ctr = nullptr,
                                uint32_t first = 0) {
    __shared__ uint32_t s_mask[32];
    const uint32_t mask = lane_private(mask_in, s_mask);  // divergence safety, see kicp_device.cuh
    const uint32_t b = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (ctr) num_blocks = min(num_blocks, ctr[0] - ctr[4]);
    if (b >= num_blocks) return;
    const int4 h = blk[b];
    table_insert_unique(slots, mask, h.x, h.y, h.z, (b << 8) | (uint32_t)h.w);
}

// AddPoints, phase 1: per input point, (optionally) transform by the pose, find or create its voxel, and push the
// point's index on that voxel's pending list.
// Asynchronous frames (kicp_register_frame): the point count (`d_n`, n is then its upper bound) and the pose (`d_res`, the result
// block of the registration that precedes this launch on the stream) are read from device memory; a registration that did not
// end with KICP_OK (NaN pose) leaves the map untouched.
// `prior_blocks`: blocks [0, prior_blocks) are a frozen prior (kicp_map_freeze); a point whose voxel is one of them is dropped.
// `evidence` (occupancy on, kicp_map_set_occupancy): a block this launch creates starts at `initial`.
__global__ void k_add_find_or_create(MapRW m, const double *__restrict__ xyz, int64_t n, int has_pose, Pose pose,
                                     double *__restrict__ xyz_t, int32_t *__restrict__ pend_next, uint32_t *counters,
                                     int32_t *__restrict__ touched, const int *d_n = nullptr, const kicp_reg_result *d_res = nullptr,
                                     uint32_t prior_blocks = 0, int32_t *evidence = nullptr, int32_t initial = 0) {
    __shared__ uint32_t s_mask[32];
    const uint32_t tmask = lane_private(m.mask, s_mask);  // divergence safety, see kicp_device.cuh
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (d_n) n = min((int64_t)*d_n, n);
    if (d_res) {
        if (d_res->status != KICP_OK) return;
        pose = Pose{d_res->pose[0], d_res->pose[1], d_res->pose[2], d_res->pose[3], d_res->pose[4], d_res->pose[5], d_res->pose[6]};
    }
    if (i >= n) return;
    double px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    if (has_pose) {
        double ox, oy, oz;
        pose_apply(pose, px, py, pz, ox, oy, oz);
        px = ox, py = oy, pz = oz;
    }
    xyz_t[3 * i] = px, xyz_t[3 * i + 1] = py, xyz_t[3 * i + 2] = pz;
    const int kx = voxel_coord(px, m.voxel_size), ky = voxel_coord(py, m.voxel_size), kz = voxel_coord(pz, m.voxel_size);
    uint32_t h = voxel_hash(kx, ky, kz) & tmask;
    uint32_t block = 0xFFFFFFFFu;
    volatile int4 *vs = m.slots;
    while (true) {
        uint32_t meta = (uint32_t)vs[h].w;
        if (meta == KICP_SLOT_EMPTY) {
            const uint32_t old = atomicCAS((unsigned int *)&m.slots[h].w, KICP_SLOT_EMPTY, KICP_SLOT_LOCKED);
            if (old == KICP_SLOT_EMPTY) {  // we create the voxel
                const uint32_t b = atomicAdd(&counters[0], 1u);
                if (b >= m.blocks_cap) {   // cannot happen: the host reserves num_blocks + n before the launch
                    atomicExch(&counters[2], 1u);
                    return;
                }
                vs[h].x = kx, vs[h].y = ky, vs[h].z = kz;
                m.blk[b] = make_int4(kx, ky, kz, 0);
                if (evidence) evidence[b] = initial;
                __threadfence();
                atomicExch((unsigned int *)&m.slots[h].w, b << 8);
                block = b;
                break;
            }
            meta = old;
        }
        if (meta == KICP_SLOT_LOCKED) continue;  // another thread is publishing this slot: re-read it
        __threadfence();
        if (vs[h].x == kx && vs[h].y == ky && vs[h].z == kz) {
            block = meta >> 8;
            break;
        }
        h = (h + 1) & tmask;
    }
    if (block < prior_blocks) return;  // a frozen prior voxel: read-only
    const int32_t prev = atomicExch(&m.pend_head[block], (int32_t)i);
    pend_next[i] = prev;
    if (prev == -1) touched[atomicAdd(&counters[1], 1u)] = (int32_t)block;
}

// AddPoints, phase 2: one thread per touched voxel replays ITS pending points in input order against the voxel's
// current content — exactly the reference's greedy rule, which never looks outside the point's own voxel:
//   skip if the voxel is full, or if any stored point is closer than map_resolution; else append.
__global__ void k_add_commit(MapRW m, const double *__restrict__ xyz_t, const int32_t *__restrict__ pend_next,
                             uint32_t *counters, const int32_t *__restrict__ touched, double map_resolution) {
    __shared__ uint32_t s_mask[32];
    __shared__ const double *s_xyz[32];
    __shared__ double *s_pts[32];
    __shared__ double s_res[32];
    // divergence safety, see kicp_device.cuh (sm_90a keeps the two point arrays and map_resolution in uniform registers inside
    // the replay loop otherwise)
    const uint32_t tmask = lane_private(m.mask, s_mask);
    xyz_t = lane_private(xyz_t, s_xyz);
    m.pts = lane_private(m.pts, s_pts);
    map_resolution = lane_private(map_resolution, s_res);
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= counters[1]) return;
    const uint32_t b = (uint32_t)touched[t];
    const int4 hdr = m.blk[b];
    int cnt = hdr.w;
    const int cnt0 = cnt;
    double *vp = m.pts + (size_t)b * m.cap * KICP_PSTRIDE;
    const int32_t head = m.pend_head[b];
    // the pending list is in arrival order (a stack of atomic pushes); the reference replays input order.  Short lists — the rule
    // in a pipeline, where the 0.5-voxel down-sample leaves at most 8 points per map voxel — are sorted in a local array; a longer
    // one (a dense raw cloud through kicp_map_add_points) falls back to repeated selection of the next index.
    constexpr int KMAX = 48;
    int32_t idx[KMAX];
    int k = 0;
    bool longlist = false;
    for (int32_t i = head; i != -1; i = pend_next[i]) {
        if (k == KMAX) {
            longlist = true;
            break;
        }
        int j = k++;
        for (; j > 0 && idx[j - 1] > i; --j) idx[j] = idx[j - 1];  // insertion sort, ascending
        idx[j] = i;
    }
    int32_t last = -1;
    int next_sorted = 0;
    while (cnt < m.cap) {
        int32_t best = 0x7FFFFFFF;
        if (!longlist) {
            if (next_sorted == k) break;
            best = idx[next_sorted++];
        } else {
            for (int32_t i = head; i != -1; i = pend_next[i])
                if (i > last && i < best) best = i;
            if (best == 0x7FFFFFFF) break;
        }
        last = best;
        const double px = xyz_t[3 * (size_t)best], py = xyz_t[3 * (size_t)best + 1], pz = xyz_t[3 * (size_t)best + 2];
        bool too_close = false;
        for (int j = 0; j < cnt; ++j) {
            const double dx = vp[KICP_PSTRIDE * j] - px, dy = vp[KICP_PSTRIDE * j + 1] - py, dz = vp[KICP_PSTRIDE * j + 2] - pz;
            if (sqrt(dx * dx + dy * dy + dz * dz) < map_resolution) {
                too_close = true;
                break;
            }
        }
        if (too_close) continue;
        vp[KICP_PSTRIDE * cnt] = px, vp[KICP_PSTRIDE * cnt + 1] = py, vp[KICP_PSTRIDE * cnt + 2] = pz, vp[KICP_PSTRIDE * cnt + 3] = 0.0;
        ++cnt;
    }
    m.pend_head[b] = -1;
    if (cnt != cnt0) {
        m.blk[b].w = cnt;
        atomicAdd(&counters[3], (uint32_t)(cnt - cnt0));
        uint32_t h = voxel_hash(hdr.x, hdr.y, hdr.z) & tmask;
        while (true) {
            const int4 s = m.slots[h];
            if (s.x == hdr.x && s.y == hdr.y && s.z == hdr.z && (uint32_t)s.w != KICP_SLOT_EMPTY) {
                m.slots[h].w = (int)((b << 8) | (uint32_t)cnt);
                break;
            }
            h = (h + 1) & tmask;
        }
    }
}

// RemovePointsFarFromLocation: a voxel dies when its FIRST point is >= max_distance from the origin.
// `d_res` (asynchronous frames): the block count is counters[0] (num_blocks is its upper bound: the flags beyond it are
// cleared for the scan that follows), the origin is the translation of the registration result, removed points are counted in
// counters[5], and nothing dies after a registration that did not end with KICP_OK.
// `first`: only blocks [first, num_blocks) are judged (and flagged); a frozen prior prefix [0, first) never dies.
__global__ void k_mark_far(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, double ox, double oy, double oz,
                           double max_distance2, uint32_t *keep, uint32_t *counters, const kicp_reg_result *d_res = nullptr,
                           uint32_t first = 0) {
    const uint32_t b = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= num_blocks) return;
    bool alive_only = false;
    if (d_res) {
        if (b >= counters[0]) {
            keep[b] = 0u;
            return;
        }
        ox = d_res->pose[4], oy = d_res->pose[5], oz = d_res->pose[6];
        alive_only = d_res->status != KICP_OK;
    }
    const double *p = pts + (size_t)b * cap * KICP_PSTRIDE;
    const double dx = p[0] - ox, dy = p[1] - oy, dz = p[2] - oz;
    const bool dead = !alive_only && (dx * dx + dy * dy + dz * dz) >= max_distance2;
    keep[b] = dead ? 0u : 1u;
    if (dead) {
        atomicAdd(&counters[4], 1u);
        atomicAdd(&counters[d_res ? 5 : 3], (uint32_t)blk[b].w);  // points removed
    }
}

// `first`: only blocks [first, num_blocks) move; new_id[b] counts the survivors in [first, b), so block b lands at first + new_id[b]
// (the prefix [0, first) is a frozen prior, which the spare arrays already hold).  `ev` / `ev_out` (occupancy on): the blocks'
// evidence moves with them.
__global__ void k_compact_blocks(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, const uint32_t *keep,
                                 const uint32_t *new_id, int4 *blk_out, double *pts_out, uint32_t first = 0, const int32_t *ev = nullptr,
                                 int32_t *ev_out = nullptr) {
    // one warp per block: header by lane 0, points copied cooperatively (blocks beyond the live count carry keep = 0)
    const uint32_t b = first + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= num_blocks || !keep[b]) return;
    const uint32_t nb = first + new_id[b];
    const int4 h = blk[b];
    if (lane == 0) {
        blk_out[nb] = h;
        if (ev_out) ev_out[nb] = ev[b];
    }
    const double *src = pts + (size_t)b * cap * KICP_PSTRIDE;
    double *dst = pts_out + (size_t)nb * cap * KICP_PSTRIDE;
    for (int i = lane; i < h.w * KICP_PSTRIDE; i += 32) dst[i] = src[i];
}

// Pointcloud / export (map_download_packed): every block's point count, whose exclusive sum is the first packed index of its points
__global__ void k_block_counts(const int4 *blk, uint32_t num_blocks, uint32_t *cnt) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < num_blocks) cnt[b] = (uint32_t)blk[b].w;
}
// the stored points packed as xyz triples from `first[b]` on, one warp per block: doubles as stored (T = double), or the float32
// records EigenToPointCloud2 writes (T = float, each coordinate narrowed by to_f32_x86)
__device__ __forceinline__ void pack_store(double *dst, double v) { *dst = v; }
__device__ __forceinline__ void pack_store(float *dst, double v) { *dst = to_f32_x86(v); }
template <class T>
__global__ void k_pack_points(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, const uint32_t *first, T *out) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per block
    const int lane = threadIdx.x & 31;
    if (b >= num_blocks) return;
    const int cnt = blk[b].w;
    const double *src = pts + (size_t)b * cap * KICP_PSTRIDE;
    T *dst = out + (size_t)first[b] * 3;
    for (int i = lane; i < cnt * 3; i += 32) pack_store(dst + i, src[(i / 3) * KICP_PSTRIDE + (i % 3)]);
}

__global__ void k_fill_i32(int32_t *p, int32_t v, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// bulk load: voxel v becomes block v
__global__ void k_load_voxels(int4 *blk, double *pts, int cap, const int32_t *keys, const int32_t *counts,
                              const int64_t *offsets, const double *points, uint32_t num_voxels) {
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (v >= num_voxels) return;
    const int c = counts[v];
    if (lane == 0) blk[v] = make_int4(keys[3 * v], keys[3 * v + 1], keys[3 * v + 2], c);
    const double *src = points + offsets[v] * 3;
    double *dst = pts + (size_t)v * cap * KICP_PSTRIDE;
    for (int i = lane; i < c * KICP_PSTRIDE; i += 32) dst[i] = (i & 3) == 3 ? 0.0 : src[(i >> 2) * 3 + (i & 3)];
}

// GetClosestNeighbor for a batch of queries, one WARP each (warp_closest_neighbor), queries grid-strided by warp, so every launch shape
// is correct.
__global__ void __launch_bounds__(256) k_nearest(MapView m, const double *__restrict__ q, int64_t n, double *__restrict__ out_pts,
                                                 double *__restrict__ out_dist) {
    __shared__ MapView s_map[32];
    const MapRegs mr = map_regs(m, s_map);  // per-thread copy of the map view (divergence safety, kicp_device.cuh)
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
        warp_closest_neighbor(mr, m.voxel_size, lane, qx, qy, qz, [&](double x, double y, double z, double d) {
            out_pts[3 * i] = x, out_pts[3 * i + 1] = y, out_pts[3 * i + 2] = z;
            out_dist[i] = d;
        }, [&]() { out_pts[3 * i] = out_pts[3 * i + 1] = out_pts[3 * i + 2] = 0.0, out_dist[i] = DBL_MAX; });
    }
}
