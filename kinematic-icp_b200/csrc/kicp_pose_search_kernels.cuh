// Kernels of the pose search (kicp_map_pose_search*): k_pose_score counts the inliers and sums d^2 of many hypothesis poses of one
// cloud against the map, k_pose_select keeps the best `keep` of them by the ranking key.  Included by kicp_map.cu, which is compiled
// with -fmad=false: a hypothesis's query points are pose_apply's and its distances are GetClosestNeighbor's, bit for bit.  A header of
// its own so that tests/emu can compile the kernels for the host against the SIMT emulator.
#pragma once
#include "kicp_map_kernels.cuh"
#include "kicp_pose_search.h"

constexpr int kPsThreads = 256;     // k_pose_score / k_pose_select CTA; k_pose_score's reduction order depends on it
constexpr int kPsSelectItems = 8;   // entries per thread of k_pose_select: a CTA selects from up to 2048
static_assert(kPsTile == kPsThreads / 32, "k_pose_score reduces one hypothesis of its tile per warp");

// GetClosestNeighbor(q)'s distance when it is below tau, evaluated by ONE lane: returns true and d for an inlier, false otherwise.
// Only the shifts whose voxel can hold a point with d < tau are probed, in KISS order, with warp_closest_neighbor's rules (a voxel
// whose first point is at a NaN distance drops out; the strict first minimum wins), so the answer is the reference's whenever its
// distance is below tau.  Exactness of the pruning (DESIGN.md §4.2): a map point with a computed d < tau has |p_a - q_a| <
// tau (1 + 2^-51) on each axis; lo / hi below bracket [q_a - that, q_a + that] with room to spare for their own rounding, and
// voxel_coord is monotone wherever it does not saturate, so such a point's key lies in [key(lo), key(hi)].  A bound whose key
// saturates (INT_MIN) falls back to all 27 shifts, as does a gate below 2^-500 (where d^2 could underflow); a non-finite query is
// never an inlier (its distances are NaN or infinite).
__device__ __forceinline__ uint32_t ps_axis_shifts(double q, double tau, double vs, int k, uint32_t m0, uint32_t mp, uint32_t mm) {
    const double s = (fabs(q) + tau) * 0x1p-40;
    const int lo = voxel_coord((q - tau) - s, vs), hi = voxel_coord((q + tau) + s, vs);
    if (lo == INT_MIN || hi == INT_MIN || !(tau >= 0x1p-500)) return m0 | mp | mm;
    uint32_t m = m0;
    if ((int64_t)hi >= (int64_t)k + 1) m |= mp;
    if ((int64_t)lo <= (int64_t)k - 1) m |= mm;
    return m;
}
__device__ __forceinline__ bool lane_gated_neighbor(const MapRegs &mr, double vs, double tau, double qx, double qy, double qz, double &dist) {
    if (!(fabs(qx) <= DBL_MAX && fabs(qy) <= DBL_MAX && fabs(qz) <= DBL_MAX)) return false;
    const int vx = voxel_coord(qx, vs), vy = voxel_coord(qy, vs), vz = voxel_coord(qz, vs);
    uint32_t shifts = ps_axis_shifts(qx, tau, vs, vx, kX0, kXP, kXM) & ps_axis_shifts(qy, tau, vs, vy, kY0, kYP, kYM) &
                      ps_axis_shifts(qz, tau, vs, vz, kZ0, kZP, kZM);
    double bd = tau;  // only a distance below the gate can matter
    while (shifts) {
        const int k = __ffs(shifts) - 1;
        shifts &= shifts - 1u;
        const uint32_t meta = map_probe(mr, vx + shift_x(k), vy + shift_y(k), vz + shift_z(k));
        if (meta == KICP_SLOT_EMPTY) continue;
        const double *vp = mr.pts + (size_t)(meta >> 8) * mr.cap * KICP_PSTRIDE;
        const int cnt = (int)(meta & 0xFFu);
        for (int j = 0; j < cnt; ++j) {
            const double dx = vp[KICP_PSTRIDE * j] - qx, dy = vp[KICP_PSTRIDE * j + 1] - qy, dz = vp[KICP_PSTRIDE * j + 2] - qz;
            const double s2 = dx * dx + dy * dy + dz * dz;
            if (j == 0 && s2 != s2) break;  // the voxel's first point is at a NaN distance: the whole voxel drops out
            const double d = sqrt(s2);
            if (d < bd) bd = d;
        }
    }
    dist = bd;
    return bd < tau;
}

// Scores of hypotheses given as (rotation, translation) pairs: rot[4r..4r+3] a unit quaternion (x, y, z, w), trans[3t..3t+2].
// Hypothesis h's score is out_cnt[h] = #{i : d_i < tau}, out_sum[h] = sum of d_i^2 over those i, with q_i = R_r p_i + t_t (pose_apply).
// Level 0 (pair_t null): the product of nr rotations and nt translations, h = r * nt + t, tiled as ceil(nt / kPsTile) tiles per
// rotation.  Otherwise pair_t[h] is h's translation and tiles[3b..3b+2] = (first hypothesis, count <= kPsTile, rotation) of tile b.
// A CTA owns a tile at a time (tiles grid-strided, so every grid is correct): thread j of the CTA rotates points j, j + 256, ... once
// and evaluates every hypothesis of the tile on them, lane per query (lane_gated_neighbor), keeping its own count and sum per
// hypothesis in shared memory; warp w then adds hypothesis w's 256 columns in a fixed order.  Every hypothesis's bits therefore
// depend on its pose, the points, tau and the map only: not on its tile, its slot, the level or the grid.
__global__ void __launch_bounds__(kPsThreads) k_pose_score(MapView m, const double *__restrict__ src, int64_t n, const double *__restrict__ rot,
                                                           const double *__restrict__ trans, int32_t nt, const int32_t *__restrict__ pair_t,
                                                           const int32_t *__restrict__ tiles, int64_t n_tiles, double tau,
                                                           int64_t *__restrict__ out_cnt, double *__restrict__ out_sum) {
    __shared__ MapView s_map[32];
    __shared__ double s_rot[4], s_tr[kPsTile][3];
    __shared__ double s_sum[kPsTile][kPsThreads];
    __shared__ uint32_t s_cnt[kPsTile][kPsThreads];
    const MapRegs mr = map_regs(m, s_map);  // per-thread copy of the map view (divergence safety, kicp_device.cuh)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tiles_per_rot = ((int64_t)nt + kPsTile - 1) / kPsTile;
    for (int64_t b = blockIdx.x; b < n_tiles; b += gridDim.x) {
        int64_t h0;
        int cnt, r;
        if (!pair_t) {
            r = (int)(b / tiles_per_rot);
            const int64_t first = (b % tiles_per_rot) * kPsTile;
            cnt = (int)min((int64_t)kPsTile, (int64_t)nt - first);
            h0 = (int64_t)r * nt + first;
        } else {
            h0 = tiles[3 * b], cnt = tiles[3 * b + 1], r = tiles[3 * b + 2];
        }
        if (tid < 4) s_rot[tid] = rot[4 * (int64_t)r + tid];
        if (tid < 3 * cnt) {
            const int j = tid / 3, a = tid % 3;
            const int64_t t = pair_t ? (int64_t)pair_t[h0 + j] : (h0 + j) % nt;
            s_tr[j][a] = trans[3 * t + a];
        }
#pragma unroll
        for (int j = 0; j < kPsTile; ++j) s_sum[j][tid] = 0.0, s_cnt[j][tid] = 0u;
        __syncthreads();
        const double qx = s_rot[0], qy = s_rot[1], qz = s_rot[2], qw = s_rot[3];
        for (int64_t c = 0; c < n; c += kPsThreads) {
            const int64_t i = c + tid;
            if (i < n) {
                double rx, ry, rz;
                quat_rotate(qx, qy, qz, qw, src[3 * i], src[3 * i + 1], src[3 * i + 2], rx, ry, rz);
                for (int j = 0; j < cnt; ++j) {
                    double d;
                    if (lane_gated_neighbor(mr, m.voxel_size, tau, rx + s_tr[j][0], ry + s_tr[j][1], rz + s_tr[j][2], d)) {
                        s_cnt[j][tid] += 1u;
                        s_sum[j][tid] += d * d;
                    }
                }
            }
            __syncwarp();
        }
        __syncthreads();
        if (warp < cnt) {
            double s = 0.0;
            unsigned long long c = 0ull;  // a thread's count fits 32 bits (n < 2^40, kPsMaxPoints); the CTA's total may not
#pragma unroll
            for (int k = 0; k < kPsThreads / 32; ++k) s += s_sum[warp][lane + 32 * k], c += s_cnt[warp][lane + 32 * k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o), c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
            if (lane == 0) out_cnt[h0 + warp] = (int64_t)c, out_sum[h0 + warp] = s;
        }
        __syncthreads();
    }
}

// The best `keep` entries by ps_key_less of each CTA's `per_cta` consecutive items, into out[blockIdx.x * keep ...] (padded with
// invalid entries).  Items are entries `in` (a previous pass's lists), or hypotheses [0, n) scored by k_pose_score: with their lattice
// points from `lat` (3 per hypothesis) or, for level 0 (lat null), decoded from the grid `g` (PsGrid).  keep rounds of a CTA-wide
// argmin; the key is total, so the result does not depend on the order of the items or on per_cta (<= kPsThreads * kPsSelectItems).
__device__ __forceinline__ void ps_shfl_min(PsEntry &e, int &who, int o) {
    PsEntry f;
    f.L[0] = __shfl_xor_sync(0xFFFFFFFFu, e.L[0], o), f.L[1] = __shfl_xor_sync(0xFFFFFFFFu, e.L[1], o);
    f.L[2] = __shfl_xor_sync(0xFFFFFFFFu, e.L[2], o), f.valid = __shfl_xor_sync(0xFFFFFFFFu, e.valid, o);
    f.n_inl = __shfl_xor_sync(0xFFFFFFFFu, e.n_inl, o), f.sum_sq = __shfl_xor_sync(0xFFFFFFFFu, e.sum_sq, o);
    const int fw = __shfl_xor_sync(0xFFFFFFFFu, who, o);
    if (ps_key_less(f, e) || (!ps_key_less(e, f) && fw < who)) e = f, who = fw;
}
__global__ void __launch_bounds__(kPsThreads) k_pose_select(const int64_t *__restrict__ cnt, const double *__restrict__ sum,
                                                            const int32_t *__restrict__ lat, PsGrid g, const PsEntry *__restrict__ in,
                                                            int64_t n, int per_cta, int keep, PsEntry *__restrict__ out) {
    __shared__ PsEntry s_best[kPsThreads / 32];
    __shared__ int s_who[kPsThreads / 32], s_win;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t base = (int64_t)blockIdx.x * per_cta;
    PsEntry e[kPsSelectItems];
#pragma unroll
    for (int k = 0; k < kPsSelectItems; ++k) {
        const int64_t off = tid + (int64_t)kPsThreads * k, i = base + off;
        e[k].valid = 0, e[k].L[0] = e[k].L[1] = e[k].L[2] = 0, e[k].n_inl = 0, e[k].sum_sq = 0.0;
        if (off < per_cta && i < n) {
            if (in) {
                e[k] = in[i];
            } else {
                if (lat) {
                    e[k].L[0] = lat[3 * i], e[k].L[1] = lat[3 * i + 1], e[k].L[2] = lat[3 * i + 2];
                } else {
                    const int64_t ny = 2 * (int64_t)g.k[1] + 1, nt = (2 * (int64_t)g.k[0] + 1) * ny, r = i / nt, t = i % nt;
                    e[k].L[0] = (int32_t)((t / ny - g.k[0]) * g.scale), e[k].L[1] = (int32_t)((t % ny - g.k[1]) * g.scale);
                    e[k].L[2] = (int32_t)((r - g.k[2]) * g.scale);
                }
                e[k].valid = 1, e[k].n_inl = cnt[i], e[k].sum_sq = sum[i];
            }
        }
    }
    for (int round = 0; round < keep; ++round) {
        int bk = 0;  // this thread's best remaining item
#pragma unroll
        for (int k = 1; k < kPsSelectItems; ++k)
            if (ps_key_less(e[k], e[bk])) bk = k;
        PsEntry w = e[0];
#pragma unroll
        for (int k = 1; k < kPsSelectItems; ++k)
            if (k == bk) w = e[k];
        int who = tid * kPsSelectItems + bk;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ps_shfl_min(w, who, o);
        if (lane == 0) s_best[warp] = w, s_who[warp] = who;
        __syncthreads();
        if (tid == 0) {
            PsEntry b = s_best[0];
            int bw = s_who[0];
#pragma unroll
            for (int v = 1; v < kPsThreads / 32; ++v)  // unrolled: no per-lane loop (divergence safety, kicp_device.cuh)
                if (ps_key_less(s_best[v], b)) b = s_best[v], bw = s_who[v];
            out[(int64_t)blockIdx.x * keep + round] = b;
            s_win = b.valid ? bw : -1;
        }
        __syncthreads();
        const int win = s_win;
        if (win >= 0 && win / kPsSelectItems == tid) {
#pragma unroll
            for (int k = 0; k < kPsSelectItems; ++k)
                if (k == win % kPsSelectItems) e[k].valid = 0;
        }
        __syncthreads();
    }
}
