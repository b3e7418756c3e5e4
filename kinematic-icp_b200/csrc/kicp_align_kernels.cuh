// Kernels of the planar alignment (kicp_map_align_planar*, kicp_align.cu): k_align_eval sums the inliers' normal equations of every
// running alignment at its current pose, k_align_step adds them up and moves the pose (kicp_align.h), k_align_finish writes the
// caller's records.  Compiled with -fmad=false: the query points are pose_apply's and the neighbours and distances GetClosestNeighbor's
// (warp_closest_neighbor), bit for bit.  A header of its own so that tests/emu can compile the kernels for the host against the SIMT
// emulator.
#pragma once
#include "kicp_align.h"
#include "kicp_nearest.cuh"

// Block b of the 1-D grid (grid-strided) covers alignment a = b / C and slot c = b % C (C = align_slots(n)); a block whose alignment
// has stopped skips it, unless `report` is set (the final pass at the returned poses, every alignment).  Slot c owns the 256-point
// chunks c, c + C, ...; in a chunk warp w owns points 32w .. 32w + 31 and runs warp_closest_neighbor for each of them in turn, the
// answering lane writing (nb, d) into the warp's shared slot j; after __syncwarp lane j forms point 32w + j's residual and Jacobian and
// adds the inlier's 1, |r|^2, J^T J and J^T r to its own sums.  A lane adds its chunks in order, the warp reduces its lanes with the
// xor tree (o = 16 .. 1), the CTA adds its warps in index order into partials[(a * C + c) * kAlignStride + k].  The order depends on
// n only: not on the grid, the other alignments or the device.
__global__ void __launch_bounds__(kAlignThreads) k_align_eval(MapView m, const double *__restrict__ src, int64_t n, double tau,
                                                              const AlignState *__restrict__ state, int32_t n_align, int32_t report,
                                                              double *__restrict__ partials) {
    __shared__ MapView s_map[32];
    __shared__ double s_nb[kAlignThreads / 32][32][4];
    __shared__ double s_part[kAlignThreads / 32][kAlignSums];
    const MapRegs mr = map_regs(m, s_map);  // per-thread copy of the map view (divergence safety, kicp_device.cuh)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int C = align_slots(n);
    const int64_t chunks = (n + kAlignThreads - 1) / kAlignThreads;
    for (int64_t b = blockIdx.x; b < (int64_t)n_align * C; b += gridDim.x) {
        const int a = (int)(b / C), c = (int)(b % C);
        if (!report && state[a].done) continue;  // block-uniform
        const double *P = state[a].pose;
        const Pose T{P[0], P[1], P[2], P[3], P[4], P[5], P[6]};
        double acc[kAlignSums];
#pragma unroll
        for (int k = 0; k < kAlignSums; ++k) acc[k] = 0.0;
        for (int64_t ch = c; ch < chunks; ch += C) {
            const int64_t base = ch * kAlignThreads + 32 * warp, i = base + lane;
            const int cnt = (int)min((int64_t)32, n - base);  // warp-uniform; <= 0 for a warp past the end
            double px = 0.0, py = 0.0, pz = 0.0, qx = 0.0, qy = 0.0, qz = 0.0;
            if (i < n) {
                px = src[3 * i], py = src[3 * i + 1], pz = src[3 * i + 2];
                pose_apply(T, px, py, pz, qx, qy, qz);
            }
            for (int j = 0; j < cnt; ++j) {
                const double x = __shfl_sync(0xFFFFFFFFu, qx, j), y = __shfl_sync(0xFFFFFFFFu, qy, j), z = __shfl_sync(0xFFFFFFFFu, qz, j);
                warp_closest_neighbor(mr, m.voxel_size, lane, x, y, z, [&](double nx, double ny, double nz, double d) {
                    s_nb[warp][j][0] = nx, s_nb[warp][j][1] = ny, s_nb[warp][j][2] = nz, s_nb[warp][j][3] = d;
                }, [&]() { s_nb[warp][j][0] = s_nb[warp][j][1] = s_nb[warp][j][2] = 0.0, s_nb[warp][j][3] = DBL_MAX; });
            }
            __syncwarp();
            if (lane < cnt && s_nb[warp][lane][3] < tau) {  // Registration.cpp:75; false for a NaN distance
                const double rx = qx - s_nb[warp][lane][0], ry = qy - s_nb[warp][lane][1], rz = qz - s_nb[warp][lane][2];
                double ax, ay, az, bx, by, bz, cx, cy, cz;  // the three columns of J
                quat_rotate(T.qx, T.qy, T.qz, T.qw, 1.0, 0.0, 0.0, ax, ay, az);
                quat_rotate(T.qx, T.qy, T.qz, T.qw, 0.0, 1.0, 0.0, bx, by, bz);
                quat_rotate(T.qx, T.qy, T.qz, T.qw, -py, px, 0.0, cx, cy, cz);
                acc[0] += 1.0;
                acc[1] += rx * rx + ry * ry + rz * rz;
                acc[2] += ax * ax + ay * ay + az * az;
                acc[3] += ax * bx + ay * by + az * bz;
                acc[4] += ax * cx + ay * cy + az * cz;
                acc[5] += bx * bx + by * by + bz * bz;
                acc[6] += bx * cx + by * cy + bz * cz;
                acc[7] += cx * cx + cy * cy + cz * cz;
                acc[8] += ax * rx + ay * ry + az * rz;
                acc[9] += bx * rx + by * ry + bz * rz;
                acc[10] += cx * rx + cy * ry + cz * rz;
            }
            __syncwarp();
        }
#pragma unroll
        for (int k = 0; k < kAlignSums; ++k) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xFFFFFFFFu, acc[k], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < kAlignSums; ++k) s_part[warp][k] = acc[k];
        }
        __syncthreads();
        if (threadIdx.x < kAlignSums) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < kAlignThreads / 32; ++w) s += s_part[w][threadIdx.x];  // unrolled (divergence safety, kicp_device.cuh)
            partials[((int64_t)a * C + c) * kAlignStride + threadIdx.x] = s;
        }
        __syncthreads();
    }
}

// Lane k < kAlignSums: component k of alignment a's C partials added in slot order; the 11 sums end up in v on every lane.
// `partials` is the kernel's lane_private copy (divergence safety, kicp_device.cuh: the loop runs on 11 lanes)
__device__ __forceinline__ void align_sum_slots(const double *partials, int a, int C, int lane, double v[kAlignSums]) {
    double s = 0.0;
    if (lane < kAlignSums)
        for (int c = 0; c < C; ++c) s += partials[((int64_t)a * C + c) * kAlignStride + lane];
#pragma unroll
    for (int k = 0; k < kAlignSums; ++k) v[k] = __shfl_sync(0xFFFFFFFFu, s, k);
}

// One warp per alignment (warps grid-strided): the sums of the last k_align_eval, then align_advance on lane 0
__global__ void k_align_step(const double *__restrict__ partials, int64_t n, int32_t n_align, double convergence, AlignState *state) {
    __shared__ const double *s_words[32];
    const double *part = lane_private(partials, s_words);
    const int lane = threadIdx.x & 31;
    const int C = align_slots(n);
    const int warps = (int)((gridDim.x * blockDim.x) >> 5);
    for (int a = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); a < n_align; a += warps) {
        if (state[a].done) continue;  // warp-uniform
        double v[kAlignSums];
        align_sum_slots(part, a, C, lane, v);
        if (lane == 0) align_advance(state[a], v, convergence);
        __syncwarp();
    }
}

// One warp per alignment: the record of its state and the sums of the final (report) k_align_eval
__global__ void k_align_finish(const double *__restrict__ partials, int64_t n, int32_t n_align, const AlignState *__restrict__ state,
                               kicp_planar_alignment *__restrict__ out) {
    __shared__ const double *s_words[32];
    const double *part = lane_private(partials, s_words);
    const int lane = threadIdx.x & 31;
    const int C = align_slots(n);
    const int warps = (int)((gridDim.x * blockDim.x) >> 5);
    for (int a = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); a < n_align; a += warps) {
        double v[kAlignSums];
        align_sum_slots(part, a, C, lane, v);
        if (lane == 0) align_record(state[a], v, n, &out[a]);
        __syncwarp();
    }
}
