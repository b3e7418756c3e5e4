// Free-space clearing of the voxel map (kicp_map_clear_free_space and the frame path's option, include/kicp.h).  Included by kicp_map.cu,
// which is compiled with -fmad=false: the ray length, the cut t_end and the traversal's crossing parameters are plain IEEE double
// arithmetic in the order kicp.h states, so the visited voxels do not depend on the build.  A header of its own so that tests/emu can
// compile the kernels for the host against the SIMT emulator.
//
// One uint32 per block (the map's free-space words, zeroed before k_free_rays): bit 31 = hit (a ray ended in the voxel), bits 0..30 =
// misses (rays that passed through it), which stop growing once they reach min_misses.  Each word is read before any atomic, so the
// voxels every ray crosses near the sensor cost one read per ray once they are saturated.  A few racing increments may pass
// min_misses (at most one per resident thread), far below bit 31.  The decision reads only these counts: it does not depend on the
// order of the rays or on the launch shape.
#pragma once
#include "kicp_device.cuh"

using namespace kicp_dev;

constexpr uint32_t kFreeHit = 0x80000000u;
// the statistics words (unsigned long long) in front of the flag words: kicp_free_space_stats in order, padded to 64 bytes
constexpr int kFreeStatWords = 8;

struct FreeRayArgs {
    double sx, sy, sz;  // the sensor origin in the cloud's frame
    double end_margin, max_distance;
    uint32_t min_misses;
};

__device__ __forceinline__ bool free_space_key_ok(int kx, int ky, int kz) { return kx != INT_MIN && ky != INT_MIN && kz != INT_MIN; }

// Rays from o = T s to q_i = T p_i, one lane per ray (rays grid-strided by warp, so every launch shape is correct).  The end voxel of a
// cast ray is hit; every other voxel of the map the ray visits before t_end gets one miss.  `d_n` / `d_res` (the frame path): the ray
// count (n is its upper bound) and the pose come from device memory, and a result block whose status is not KICP_OK casts nothing.
// stats[0] += rays cast, stats[1] += voxels visited (both aggregated per warp).
__global__ void __launch_bounds__(256) k_free_rays(MapView m, const double *__restrict__ xyz, int64_t n, const int *d_n, Pose pose,
                                                   const kicp_reg_result *d_res, FreeRayArgs a, uint32_t *flags,
                                                   unsigned long long *stats) {
    __shared__ MapView s_map[32];
    __shared__ uint32_t *s_flags[32];
    __shared__ uint32_t s_min[32];
    // divergence safety, see kicp_device.cuh: the table view, the flag words and min_misses are read inside the per-lane traversal
    const MapRegs mr = map_regs(m, s_map);
    flags = lane_private(flags, s_flags);
    const uint32_t min_misses = lane_private(a.min_misses, s_min);
    if (d_n) n = min((int64_t)*d_n, n);
    if (d_res) {
        if (d_res->status != KICP_OK) return;
        pose = Pose{d_res->pose[0], d_res->pose[1], d_res->pose[2], d_res->pose[3], d_res->pose[4], d_res->pose[5], d_res->pose[6]};
    }
    const double vs = m.voxel_size;
    double ox, oy, oz;
    pose_apply(pose, a.sx, a.sy, a.sz, ox, oy, oz);
    const int kox = voxel_coord(ox, vs), koy = voxel_coord(oy, vs), koz = voxel_coord(oz, vs);
    const bool origin_ok = free_space_key_ok(kox, koy, koz);
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned long long rays = 0, visits = 0;
    // the loop bound is warp-uniform (the warp's first ray), so every lane reaches the __syncwarp of every round
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
        const int64_t i = base + lane;
        if (i < n && origin_ok) {
            double qx, qy, qz;
            pose_apply(pose, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], qx, qy, qz);
            const int kqx = voxel_coord(qx, vs), kqy = voxel_coord(qy, vs), kqz = voxel_coord(qz, vs);
            if (free_space_key_ok(kqx, kqy, kqz)) {
                ++rays;
                const uint32_t hm = map_probe(mr, kqx, kqy, kqz);
                if (hm != KICP_SLOT_EMPTY) {
                    uint32_t *w = flags + (hm >> 8);
                    if (!(*(volatile uint32_t *)w & kFreeHit)) atomicOr(w, kFreeHit);
                }
                const double dx = qx - ox, dy = qy - oy, dz = qz - oz;
                const double L = sqrt(dx * dx + dy * dy + dz * dz);
                const double cut = L - a.end_margin;
                const double t_end = (cut < a.max_distance ? cut : a.max_distance) / L;
                if (L != 0.0 && t_end > 0.0) {
                    // 3-D DDA from K(o); keys in 64 bits (a key outside the 32-bit range is in no map)
                    long long kx = kox, ky = koy, kz = koz;
                    int sx = 0, sy = 0, sz = 0;
                    double tx = INFINITY, ty = INFINITY, tz = INFINITY, ux = 0.0, uy = 0.0, uz = 0.0;
                    if (dx > 0.0) sx = 1, tx = (((double)kx + 1.0) * vs - ox) / dx, ux = vs / dx;
                    else if (dx < 0.0) sx = -1, tx = ((double)kx * vs - ox) / dx, ux = -vs / dx;
                    if (dy > 0.0) sy = 1, ty = (((double)ky + 1.0) * vs - oy) / dy, uy = vs / dy;
                    else if (dy < 0.0) sy = -1, ty = ((double)ky * vs - oy) / dy, uy = -vs / dy;
                    if (dz > 0.0) sz = 1, tz = (((double)kz + 1.0) * vs - oz) / dz, uz = vs / dz;
                    else if (dz < 0.0) sz = -1, tz = ((double)kz * vs - oz) / dz, uz = -vs / dz;
                    long long steps = llabs((long long)kqx - kx) + llabs((long long)kqy - ky) + llabs((long long)kqz - kz);
                    while (true) {
                        ++visits;  // voxel (kx, ky, kz)
                        if ((kx != kqx || ky != kqy || kz != kqz) && kx >= INT_MIN && kx <= INT_MAX && ky >= INT_MIN && ky <= INT_MAX &&
                            kz >= INT_MIN && kz <= INT_MAX) {
                            const uint32_t meta = map_probe(mr, (int)kx, (int)ky, (int)kz);
                            if (meta != KICP_SLOT_EMPTY) {
                                uint32_t *w = flags + (meta >> 8);
                                const uint32_t v = *(volatile uint32_t *)w;
                                if (!(v & kFreeHit) && v < min_misses) atomicAdd(w, 1u);
                            }
                        }
                        if (steps-- == 0) break;
                        // the axis of the smallest crossing parameter, the lowest index on ties
                        if (tx <= ty && tx <= tz) {
                            if (tx >= t_end) break;
                            kx += sx, tx += ux;
                        } else if (ty <= tz) {
                            if (ty >= t_end) break;
                            ky += sy, ty += uy;
                        } else {
                            if (tz >= t_end) break;
                            kz += sz, tz += uz;
                        }
                    }
                }
            }
        }
        __syncwarp();
    }
    for (int off = 16; off > 0; off >>= 1) {
        rays += __shfl_xor_sync(0xFFFFFFFFu, rays, off);
        visits += __shfl_xor_sync(0xFFFFFFFFu, visits, off);
    }
    if (lane == 0 && rays) {
        atomicAdd(&stats[0], rays);
        atomicAdd(&stats[1], visits);
    }
}

// Occupancy evidence (kicp_map_set_occupancy): the update of a live block's int32 evidence in a clearing call
struct OccupancyArgs {
    int32_t hit_gain, miss_loss, max_evidence;
};

// The decision over blocks [0, num_blocks): a block with at least min_misses misses and no hit is free.  A free prior block
// (b < prior_blocks) is kept and counted in stats[4].  A free live block is cleared: keep[b] = 0, and it is counted in the words that
// kicp_map_finish_update reads (counters[4] blocks, counters[d_res ? 5 : 3] points) and in stats[2] / stats[3].
// Synchronous (`d_res` null): this kernel writes keep[b] for every live block.  Frame path (after k_mark_far): a block k_mark_far
// already evicted stays evicted and is not counted here, and blocks beyond the insert's count (counters[0]) are skipped.
// `evidence` (occupancy on): a live block's evidence gains hit_gain (up to max_evidence) on a hit and loses miss_loss when free; a free
// block is cleared only when its evidence reaches 0 or less.  The prior's evidence is not touched.
__global__ void k_mark_free(const int4 *blk, uint32_t num_blocks, uint32_t prior_blocks, const uint32_t *flags, uint32_t min_misses,
                            uint32_t *keep, uint32_t *counters, unsigned long long *stats, const kicp_reg_result *d_res = nullptr,
                            int32_t *evidence = nullptr, OccupancyArgs occ = OccupancyArgs{0, 0, 0}) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= num_blocks) return;
    if (d_res && b >= counters[0]) return;
    const uint32_t w = flags[b];
    const bool free = !(w & kFreeHit) && w >= min_misses;
    if (b < prior_blocks) {
        if (free) atomicAdd(&stats[4], 1ull);
        return;
    }
    if (d_res && !keep[b]) return;  // evicted by distance
    bool clear = free;
    if (evidence) {
        // |e| <= 2^24 and gain, loss <= 2^24: no overflow
        const int32_t e = evidence[b];
        if (w & kFreeHit) {
            const int32_t g = e + occ.hit_gain;
            evidence[b] = g < occ.max_evidence ? g : occ.max_evidence;
        } else if (free) {
            evidence[b] = e - occ.miss_loss;
            clear = e - occ.miss_loss <= 0;
        }
    }
    if (!d_res) keep[b] = clear ? 0u : 1u;
    else if (!clear) return;
    else keep[b] = 0u;
    if (clear) {
        const uint32_t pts = (uint32_t)blk[b].w;
        atomicAdd(&counters[4], 1u);
        atomicAdd(&counters[d_res ? 5 : 3], pts);
        atomicAdd(&stats[2], 1ull);
        atomicAdd(&stats[3], (unsigned long long)pts);
    }
}
