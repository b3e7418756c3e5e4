// Kernels of the correspondence report (kicp_map_correspondences*, option "correspondences" of the frame calls): the reference's
// DataAssociation (Registration.cpp:62-81) and the sums of ComputePerturbation (Registration.cpp:86-118) evaluated once at a given
// pose.  Included by kicp_map.cu, which is compiled with -fmad=false: the transform is the one k_add_find_or_create applies, and the
// neighbour search is k_nearest's (warp_closest_neighbor), so points, distances and the gate are the oracle's bit for bit.  A header of
// its own so that tests/emu can compile the kernels for the host against the SIMT emulator.
#pragma once
#include "kicp_map_kernels.cuh"

constexpr int kCorrThreads = 256;  // k_corr_eval's CTA: eight warps, one query each at a time
constexpr int kCorrSums = 7;       // per-CTA partial: {inliers, sum |r|^2, JTJ00, JTJ01, JTJ11, JTr0, JTr1}
constexpr int kCorrStride = 8;     // doubles per partial (one spare)

// For source point i < n (n = min(*d_n, n) when d_n is given): q = T * p_i, (n_i, d_i) = GetClosestNeighbor(q), inlier = d_i < tau.
// The pose is `pose`, or the result block of the registration that precedes this launch on the stream when d_res is given.
// Per-point outputs (each may be null): out_pts[3i..3i+2] = n_i, out_dist[i] = d_i, out_inl[i] = inlier.  Per inlier, with
// J = [R e_x | R (-p_y, p_x, 0)] and r = q - n_i (Registration.cpp:89-95), the lane that holds the answer adds 1, |r|^2, J^T J and
// J^T r to its own sums; the CTA reduces its lanes in a fixed order (xor tree per warp, then the warps in index order) into
// partials[blockIdx.x * kCorrStride + k].  One warp per point, points grid-strided by warp: every launch shape is correct, and one
// launch shape gives the same bits every time.
__global__ void __launch_bounds__(kCorrThreads) k_corr_eval(MapView m, const double *__restrict__ src, int64_t n, const int *d_n, Pose pose,
                                                            const kicp_reg_result *d_res, double tau, double *__restrict__ out_pts,
                                                            double *__restrict__ out_dist, uint8_t *__restrict__ out_inl,
                                                            double *__restrict__ partials) {
    __shared__ MapView s_map[32];
    __shared__ double s_part[kCorrThreads / 32][kCorrSums];
    const MapRegs mr = map_regs(m, s_map);  // per-thread copy of the map view (divergence safety, kicp_device.cuh)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (d_n) n = min((int64_t)*d_n, n);
    if (d_res) pose = Pose{d_res->pose[0], d_res->pose[1], d_res->pose[2], d_res->pose[3], d_res->pose[4], d_res->pose[5], d_res->pose[6]};
    double acc[kCorrSums];
#pragma unroll
    for (int k = 0; k < kCorrSums; ++k) acc[k] = 0.0;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double px = src[3 * i], py = src[3 * i + 1], pz = src[3 * i + 2];
        double qx, qy, qz;
        pose_apply(pose, px, py, pz, qx, qy, qz);
        auto emit = [&](double nx, double ny, double nz, double d) {
            const bool inlier = d < tau;  // Registration.cpp:75; false for a NaN distance
            if (out_pts) out_pts[3 * i] = nx, out_pts[3 * i + 1] = ny, out_pts[3 * i + 2] = nz;
            if (out_dist) out_dist[i] = d;
            if (out_inl) out_inl[i] = inlier ? 1 : 0;
            if (!inlier) return;
            const double rx = qx - nx, ry = qy - ny, rz = qz - nz;
            double ax, ay, az, bx, by, bz;  // the two columns of J
            quat_rotate(pose.qx, pose.qy, pose.qz, pose.qw, 1.0, 0.0, 0.0, ax, ay, az);
            quat_rotate(pose.qx, pose.qy, pose.qz, pose.qw, -py, px, 0.0, bx, by, bz);
            acc[0] += 1.0;
            acc[1] += rx * rx + ry * ry + rz * rz;
            acc[2] += ax * ax + ay * ay + az * az;
            acc[3] += ax * bx + ay * by + az * bz;
            acc[4] += bx * bx + by * by + bz * bz;
            acc[5] += ax * rx + ay * ry + az * rz;
            acc[6] += bx * rx + by * ry + bz * rz;
        };
        warp_closest_neighbor(mr, m.voxel_size, lane, qx, qy, qz, emit, [&]() { emit(0.0, 0.0, 0.0, DBL_MAX); });
    }
#pragma unroll
    for (int k = 0; k < kCorrSums; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xFFFFFFFFu, acc[k], o);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < kCorrSums; ++k) s_part[warp][k] = acc[k];
    }
    __syncthreads();
    if (threadIdx.x < kCorrSums) {
        const int nw = (int)(blockDim.x >> 5);
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kCorrThreads / 32; ++w)  // unrolled: no per-lane loop (divergence safety, kicp_device.cuh)
            if (w < nw) s += s_part[w][threadIdx.x];
        partials[(size_t)blockIdx.x * kCorrStride + threadIdx.x] = s;
    }
}

// One warp: lane k < kCorrSums adds component k of the `parts` partials in index order, then lane 0 writes the statistics
// (n_points = min(*d_n, n) when d_n is given).  No atomics anywhere, so equal inputs and launch shapes give equal bits.
__global__ void k_corr_finish(const double *__restrict__ partials, int parts, int64_t n, const int *d_n, kicp_corr_stats *out) {
    const int lane = threadIdx.x & 31;
    if (d_n) n = min((int64_t)*d_n, n);
    double s = 0.0;
    if (lane < kCorrSums)
        for (int b = 0; b < parts; ++b) s += partials[(size_t)b * kCorrStride + lane];
    double v[kCorrSums];
#pragma unroll
    for (int k = 0; k < kCorrSums; ++k) v[k] = __shfl_sync(0xFFFFFFFFu, s, k);
    if (threadIdx.x != 0) return;
    kicp_corr_stats st;
    st.n_points = n;
    st.n_inliers = (int64_t)v[0];
    st.fitness = n > 0 ? v[0] / (double)n : 0.0;
    st.inlier_rmse = v[0] > 0.0 ? sqrt(v[1] / v[0]) : 0.0;
    st.sum_sq = v[1];
    st.jtj[0] = v[2], st.jtj[1] = v[3], st.jtj[2] = v[4];
    st.jtr[0] = v[5], st.jtr[1] = v[6];
    *out = st;
}
