// Kernels of the device-resident kiss_icp::VoxelHashMap (included by kicp_map.cu, which is compiled with -fmad=false: every decision
// — voxel floor, the < map_resolution spacing test, the >= max_distance^2 eviction test, the nearest-neighbour argmin — is evaluated
// in plain IEEE double arithmetic in the reference's operation order).  A header of its own so that tests/emu can compile the kernels
// for the host against the SIMT emulator without the CUDA-runtime orchestration of kicp_map.cu.
#pragma once
#include <cfloat>

#include "kicp_device.cuh"
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

// `ctr` (optional): the block count lives on the device — blocks after the last AddPoints minus the ones just evicted
__global__ void k_table_rebuild(int4 *slots, uint32_t mask_in, const int4 *blk, uint32_t num_blocks, const uint32_t *ctr = nullptr) {
    __shared__ uint32_t s_mask[32];
    const uint32_t mask = lane_private(mask_in, s_mask);  // divergence safety, see kicp_device.cuh
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
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
__global__ void k_add_find_or_create(MapRW m, const double *__restrict__ xyz, int64_t n, int has_pose, Pose pose,
                                     double *__restrict__ xyz_t, int32_t *__restrict__ pend_next, uint32_t *counters,
                                     int32_t *__restrict__ touched, const int *d_n = nullptr, const kicp_reg_result *d_res = nullptr) {
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
__global__ void k_mark_far(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, double ox, double oy, double oz,
                           double max_distance2, uint32_t *keep, uint32_t *counters, const kicp_reg_result *d_res = nullptr) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
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

__global__ void k_compact_blocks(const int4 *blk, const double *pts, int cap, uint32_t num_blocks, const uint32_t *keep,
                                 const uint32_t *new_id, int4 *blk_out, double *pts_out) {
    // one warp per block: header by lane 0, points copied cooperatively (blocks beyond the live count carry keep = 0)
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= num_blocks || !keep[b]) return;
    const uint32_t nb = new_id[b];
    const int4 h = blk[b];
    if (lane == 0) blk_out[nb] = h;
    const double *src = pts + (size_t)b * cap * KICP_PSTRIDE;
    double *dst = pts_out + (size_t)nb * cap * KICP_PSTRIDE;
    for (int i = lane; i < h.w * KICP_PSTRIDE; i += 32) dst[i] = src[i];
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

// GetClosestNeighbor for a batch of queries, one thread each, evaluated exactly like the reference:
// shifts in KISS order, per voxel first-minimum of (x - q).norm() under strict <, global strict <.
__global__ void k_nearest(MapView m, const double *__restrict__ q, int64_t n, double *__restrict__ out_pts,
                          double *__restrict__ out_dist) {
    __shared__ MapView s_map[32];
    const MapRegs mr = map_regs(m, s_map);  // per-thread copy of the map view (divergence safety, kicp_device.cuh)
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
    const int vx = voxel_coord(qx, m.voxel_size), vy = voxel_coord(qy, m.voxel_size), vz = voxel_coord(qz, m.voxel_size);
    double bx = 0.0, by = 0.0, bz = 0.0, bd = DBL_MAX;
    for (int k = 0; k < 27; ++k) {
        const uint32_t meta = map_probe(mr, vx + shift_x(k), vy + shift_y(k), vz + shift_z(k));
        if (meta == KICP_SLOT_EMPTY) continue;
        const double *vp = mr.pts + (size_t)(meta >> 8) * mr.cap * KICP_PSTRIDE;
        const int cnt = (int)(meta & 0xFFu);
        for (int j = 0; j < cnt; ++j) {
            const double dx = vp[KICP_PSTRIDE * j] - qx, dy = vp[KICP_PSTRIDE * j + 1] - qy, dz = vp[KICP_PSTRIDE * j + 2] - qz;
            const double d = sqrt(dx * dx + dy * dy + dz * dz);
            if (d < bd) bd = d, bx = vp[KICP_PSTRIDE * j], by = vp[KICP_PSTRIDE * j + 1], bz = vp[KICP_PSTRIDE * j + 2];
        }
    }
    out_pts[3 * i] = bx, out_pts[3 * i + 1] = by, out_pts[3 * i + 2] = bz;
    out_dist[i] = bd;
}
