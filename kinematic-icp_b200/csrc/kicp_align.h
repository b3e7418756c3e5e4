// The arithmetic of the planar alignment (kicp_map_align_planar*, kicp_align.cu) that is not a neighbour search: the update
// T [+] dx, the fixed LDL^T solve of the 3x3 normal equations and the step norm.  __host__ __device__, so that the kernels of
// kicp_align_kernels.cuh, the SIMT emulator of tests/emu and the CPU tests run this one copy.  Every operation is +, -, *, / or sqrt,
// written out in the order the tests restate (tests/align_planar_oracle.py): compiled without FMA contraction (the library with
// -fmad=false, the emulator with -ffp-contract=off) the device, the emulator and numpy give the same bits.
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "kicp.h"

#if defined(__CUDACC__)
#define KICP_AL_HD __host__ __device__
#else
#define KICP_AL_HD
#endif

constexpr int kAlignThreads = 256;  // k_align_eval's CTA: 8 warps, one 256-point chunk at a time
constexpr int kAlignCtas = 512;     // CTA slots of one alignment at most: 262 144 points (1 024 chunks) fill an H100 with one start
constexpr int kAlignSums = 11;      // per-slot partial: {inliers, sum |r|^2, JTJ00, 01, 02, 11, 12, 22, JTr0, 1, 2}
constexpr int kAlignStride = 12;    // doubles per partial (one spare)
constexpr int kAlignMaxInitial = 64;  // starting poses of one call (the pose search's `keep` bound)
constexpr int64_t kAlignMaxPoints = (int64_t)1 << 40;  // host points of one call

// The state of one alignment on the device, advanced by k_align_step: the current pose (x, y, z, w, tx, ty, tz), the status
// (KICP_ALIGN_*; MAX_ITERATIONS while it runs), the iterations taken, the norm of the last step and done = 1 once it stopped
struct AlignState {
    double pose[7];
    int32_t status;
    int32_t iterations;
    double last_step;
    int32_t done;
    int32_t pad;
};

// CTA slots per alignment: C = min(kAlignCtas, ceil(n / 256)), at least 1.  Slot c owns the chunks c, c + C, c + 2C, ...
KICP_AL_HD inline int align_slots(int64_t n) {
    const int64_t chunks = (n + kAlignThreads - 1) / kAlignThreads;
    return chunks < 1 ? 1 : chunks > kAlignCtas ? kAlignCtas : (int)chunks;
}

// T [+] dx: T * Delta, Delta = (R_q, (dx0, dx1, 0)), q = (0, 0, dx2 / 2, 1).  The rotation is normalize(q_T * q) in the operation order
// of ps_rotation (kicp_pose_search.h) with (sin, cos) replaced by (dx2 / 2, 1): a turn by 2 atan(dx2 / 2), dx2 to third order, and no
// trigonometry.  The translation is t_T + R_T (dx0, dx1, 0) in ps_translation's (quat_rotate's) order.  pose = (x, y, z, w, t).
KICP_AL_HD inline void align_update(const double T[7], const double dx[3], double out[7]) {
    const double ax = T[0], ay = T[1], az = T[2], aw = T[3];
    const double bx = 0.0, by = 0.0, bz = dx[2] / 2.0, bw = 1.0;
    const double w = aw * bw - ax * bx - ay * by - az * bz;
    const double x = aw * bx + ax * bw + ay * bz - az * by;
    const double y = aw * by + ay * bw + az * bx - ax * bz;
    const double z = aw * bz + az * bw + ax * by - ay * bx;
    double n2 = x * x;
    n2 += y * y;
    n2 += z * z;
    n2 += w * w;
    const double len = sqrt(n2);
    const double px = dx[0], py = dx[1], pz = 0.0;
    double ux = ay * pz - az * py, uy = az * px - ax * pz, uz = ax * py - ay * px;
    ux = ux + ux, uy = uy + uy, uz = uz + uz;
    const double ox = px + aw * ux + (ay * uz - az * uy);
    const double oy = py + aw * uy + (az * ux - ax * uz);
    const double oz = pz + aw * uz + (ax * uy - ay * ux);
    out[0] = x / len, out[1] = y / len, out[2] = z / len, out[3] = w / len;
    out[4] = T[4] + ox, out[5] = T[5] + oy, out[6] = T[6] + oz;
}

// a pivot of the LDL^T factorisation is usable when it is positive and finite (false for NaN)
KICP_AL_HD inline bool align_pivot_ok(double d) { return d > 0.0 && d <= DBL_MAX; }

// dx = -A^-1 b for the symmetric A = {a00, a01, a02, a11, a12, a22} by a fixed LDL^T (no pivoting):
//   d0 = a00, l10 = a01 / d0, l20 = a02 / d0, d1 = a11 - l10 a01, e = a12 - l20 a01, l21 = e / d1, d2 = (a22 - l20 a02) - l21 e;
//   y = L^-1 (-b), z = D^-1 y, dx = L^-T z.
// Returns false (dx unspecified) when a pivot is not positive and finite or a component of dx is not finite.
KICP_AL_HD inline bool align_solve(const double A[6], const double b[3], double dx[3]) {
    const double d0 = A[0];
    if (!align_pivot_ok(d0)) return false;
    const double l10 = A[1] / d0, l20 = A[2] / d0;
    const double d1 = A[3] - l10 * A[1];
    if (!align_pivot_ok(d1)) return false;
    const double e = A[4] - l20 * A[1];
    const double l21 = e / d1;
    const double d2 = (A[5] - l20 * A[2]) - l21 * e;
    if (!align_pivot_ok(d2)) return false;
    const double y0 = -b[0];
    const double y1 = -b[1] - l10 * y0;
    const double y2 = (-b[2] - l20 * y0) - l21 * y1;
    const double z0 = y0 / d0, z1 = y1 / d1, z2 = y2 / d2;
    dx[2] = z2;
    dx[1] = z1 - l21 * dx[2];
    dx[0] = (z0 - l10 * dx[1]) - l20 * dx[2];
    for (int k = 0; k < 3; ++k)
        if (!(fabs(dx[k]) <= DBL_MAX)) return false;
    return true;
}

// |dx| = sqrt((dx0 dx0 + dx1 dx1) + dx2 dx2): the reference's dx.norm() < convergence_criterion test (Registration.cpp:184)
KICP_AL_HD inline double align_step_norm(const double dx[3]) { return sqrt((dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2]); }

// One Gauss-Newton step of an alignment from its summed partials v[kAlignSums] (the layout of a slot's partial): stops it with
// NO_CORRESPONDENCES (no inlier) or SINGULAR (align_solve failed), both with the pose unchanged, or moves the pose and stops it with
// CONVERGED when the step is shorter than `convergence`.
KICP_AL_HD inline void align_advance(AlignState &s, const double v[kAlignSums], double convergence) {
    if (s.done) return;
    const double N = v[0];
    if (!(N > 0.0)) {
        s.status = KICP_ALIGN_NO_CORRESPONDENCES, s.done = 1;
        return;
    }
    const double A[6] = {v[2] / N, v[3] / N, v[4] / N, v[5] / N, v[6] / N, v[7] / N};
    const double b[3] = {v[8] / N, v[9] / N, v[10] / N};
    double dx[3];
    if (!align_solve(A, b, dx)) {
        s.status = KICP_ALIGN_SINGULAR, s.done = 1;
        return;
    }
    double T[7];
    for (int k = 0; k < 7; ++k) T[k] = s.pose[k];
    align_update(T, dx, s.pose);
    s.iterations += 1;
    s.last_step = align_step_norm(dx);
    if (s.last_step < convergence) s.status = KICP_ALIGN_CONVERGED, s.done = 1;
}

// The caller's record of an alignment from its state and the sums at its returned pose; n = the points aligned
KICP_AL_HD inline void align_record(const AlignState &s, const double v[kAlignSums], int64_t n, kicp_planar_alignment *o) {
    for (int k = 0; k < 7; ++k) o->pose[k] = s.pose[k];
    o->status = s.status;
    o->iterations = s.iterations;
    o->last_step = s.last_step;
    o->n_inliers = (int64_t)v[0];
    o->fitness = n > 0 ? v[0] / (double)n : 0.0;
    o->inlier_rmse = v[0] > 0.0 ? sqrt(v[1] / v[0]) : 0.0;
    o->sum_sq = v[1];
    for (int k = 0; k < 6; ++k) o->jtj[k] = v[2 + k];
    for (int k = 0; k < 3; ++k) o->jtr[k] = v[8 + k];
}
