// GetClosestNeighbor (KISS-ICP v1.2.0 VoxelHashMap.cpp) of one query by one warp, shared by k_nearest and k_corr_eval
// (kicp_map_kernels.cuh, kicp_corr_kernels.cuh, compiled into kicp_map.cu) and k_align_eval (kicp_align_kernels.cuh, compiled into
// kicp_align.cu).  A header of its own so that a translation unit can use the search without compiling the map's kernels again.
#pragma once
#include <cfloat>

#include "kicp_device.cuh"

using namespace kicp_dev;

// GetClosestNeighbor(q) evaluated by one WARP, exactly like the reference: shifts in KISS order, per voxel first-minimum of
// (x - q).norm() under strict <, global strict <.
//   - lane k < 27 probes shift k;
//   - the candidates of the found voxels are numbered t = (shift, slot) in that order and dealt across the lanes in rounds of 32, so
//     that consecutive lanes read consecutive points of one voxel (a lane finds its voxel by a binary search over the lanes' first t);
//   - each lane keeps its first strict minimum of d, then a warp argmin over the key (d, t) picks the reference's candidate: the
//     smallest d, ties to the earliest voxel in shift order, then the earliest slot.  Only d < DBL_MAX wins (an infinite distance
//     leaves (0,0,0), DBL_MAX), and a NaN distance never does.
// The reference takes a voxel's min_element first: a NaN distance of its FIRST point (a non-finite point in the map or the query) is
// never replaced and never wins, so that whole voxel drops out; its sum of squares is NaN exactly when the distance is.
// All 32 lanes call it with the same query; exactly one lane receives the answer: `emit(x, y, z, d)` with the candidate, or
// `emit_empty()` on lane 0 for an empty neighbourhood, whose answer is (0,0,0), DBL_MAX.  The warp has reconverged when it returns.
template <class Emit, class EmitEmpty>
__device__ __forceinline__ void warp_closest_neighbor(const MapRegs &mr, double voxel_size, int lane, double qx, double qy, double qz,
                                                      Emit emit, EmitEmpty emit_empty) {
    const int vx = voxel_coord(qx, voxel_size), vy = voxel_coord(qy, voxel_size), vz = voxel_coord(qz, voxel_size);
    uint32_t meta = KICP_SLOT_EMPTY;
    if (lane < 27) meta = map_probe(mr, vx + shift_x(lane), vy + shift_y(lane), vz + shift_z(lane));
    __syncwarp();
    int cnt = 0;
    if (meta != KICP_SLOT_EMPTY) {
        const double *vp = mr.pts + (size_t)(meta >> 8) * mr.cap * KICP_PSTRIDE;
        const double dx = vp[0] - qx, dy = vp[1] - qy, dz = vp[2] - qz;
        const double s0 = dx * dx + dy * dy + dz * dz;
        cnt = s0 != s0 ? 0 : (int)(meta & 0xFFu);
    }
    __syncwarp();
    int first = cnt;  // inclusive scan of the counts, then the lane's first candidate number
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, first, o);
        if (lane >= o) first += v;
    }
    const int total = __shfl_sync(0xFFFFFFFFu, first, 31);
    if (total == 0) {  // an empty neighbourhood (warp-uniform): nothing to search or reduce
        if (lane == 0) emit_empty();
        __syncwarp();
        return;
    }
    first -= cnt;
    double bd = DBL_MAX, bx = 0.0, by = 0.0, bz = 0.0;
    int bt = INT_MAX;
    for (int r = 0; r < total; r += 32) {
        const int t = r + lane;
        int f = 0;  // the last lane whose first candidate is <= t: it holds t (lanes without candidates share the next one's first)
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
            if (__shfl_sync(0xFFFFFFFFu, first, f + step) <= t) f += step;
        const int j = t - __shfl_sync(0xFFFFFFFFu, first, f);
        const uint32_t b = __shfl_sync(0xFFFFFFFFu, meta, f) >> 8;
        if (t < total) {
            const double *p = mr.pts + ((size_t)b * mr.cap + j) * KICP_PSTRIDE;
            const double px = p[0], py = p[1], pz = p[2];
            const double dx = px - qx, dy = py - qy, dz = pz - qz;
            const double d = sqrt(dx * dx + dy * dy + dz * dz);
            if (d < bd) bd = d, bx = px, by = py, bz = pz, bt = t;
        }
    }
    __syncwarp();
    double wd = bd;  // the warp's minimum of (d, t); t is unique, so one lane holds it
    int wt = bt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xFFFFFFFFu, wd, o);
        const int ot = __shfl_xor_sync(0xFFFFFFFFu, wt, o);
        if (od < wd || (od == wd && ot < wt)) wd = od, wt = ot;
    }
    if (wt == INT_MAX ? lane == 0 : bt == wt) emit(bx, by, bz, bd);
    __syncwarp();
}
