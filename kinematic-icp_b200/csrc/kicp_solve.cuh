// Pose state and the scalar tail of one IRLS iteration (device code shared by the kernels of kicp_register.cu):
// Sophus-compatible SE(3) helpers, the initial estimate (Registration.cpp:156) and ComputePerturbation's solve + motion model + pose
// update + convergence test (Registration.cpp:119-125, 159-167, 181-184).  One thread executes these.
#pragma once
#include <cfloat>
#include <cmath>

#include "kicp_register.cuh"

using namespace kicp_dev;

// Pose + solver state of one registration.  The persistent kernel keeps one replica per CTA in shared memory; the
// multi-launch (NCCL) path keeps it in RegState.
struct PoseState {
    double q[4];  // current estimate: unit quaternion (x, y, z, w) ...
    double t[3];  // ... translation ...
    double R[9];  // ... and the rotation matrix of q, row-major
    double qp[4], tp[3];  // q, t of the previous pass (the nearest-neighbour certificates compare the two)
    double tau, conv, fixed_reg, beta;
    int adaptive, max_iter;
    int iter, done, status;
};


// ------------------------------------------------------------------------------------------ SE3 helpers (Sophus)
__device__ void quat_to_matrix(const double q[4], double R[9]) {  // Eigen::Quaternion::toRotationMatrix
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
    R[3] = txy + twz, R[4] = 1 - (txx + tzz), R[5] = tyz - twx;
    R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1 - (txx + tyy);
}

// Sophus SE3 product: q = normalize(a.q * b.q) (the SO3(quaternion) ctor normalises), t = a.t + a.q * b.t
__device__ void se3_compose(const double aq[4], const double at[3], const double bq[4], const double bt[3], double oq[4],
                            double ot[3]) {
    const double ax = aq[0], ay = aq[1], az = aq[2], aw = aq[3];
    const double bx = bq[0], by = bq[1], bz = bq[2], bw = bq[3];
    double w = aw * bw - ax * bx - ay * by - az * bz;
    double x = aw * bx + ax * bw + ay * bz - az * by;
    double y = aw * by + ay * bw + az * bx - ax * bz;
    double z = aw * bz + az * bw + ax * by - ay * bx;
    const double len = sqrt(x * x + y * y + z * z + w * w);
    x /= len, y /= len, z /= len, w /= len;
    double rx, ry, rz;
    quat_rotate(ax, ay, az, aw, bt[0], bt[1], bt[2], rx, ry, rz);
    oq[0] = x, oq[1] = y, oq[2] = z, oq[3] = w;
    ot[0] = at[0] + rx, ot[1] = at[1] + ry, ot[2] = at[2] + rz;
}

// Sophus SE3::exp for the tangent the motion model produces: (ux, uy, 0, 0, 0, theta)
__device__ void se3_exp_planar(double ux, double uy, double theta_in, double oq[4], double ot[3]) {
    const double eps = 1e-10;  // Sophus::Constants<double>::epsilon()
    const double wx = 0.0, wy = 0.0, wz = theta_in;
    const double theta_sq = wx * wx + wy * wy + wz * wz;
    double theta, imag, real;
    if (theta_sq < eps * eps) {
        theta = 0.0;
        const double theta_po4 = theta_sq * theta_sq;
        imag = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * theta_po4;
        real = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * theta_po4;
    } else {
        theta = sqrt(theta_sq);
        const double half_theta = 0.5 * theta;
        double sh, ch;
        sincos(half_theta, &sh, &ch);
        imag = sh / theta;
        real = ch;
    }
    oq[0] = imag * wx, oq[1] = imag * wy, oq[2] = imag * wz, oq[3] = real;
    // V = I + (1-cos)/th^2 W + (th - sin)/th^3 W^2, or V = R when theta < eps;  W = hat(0, 0, wz)
    double V[9];
    if (theta < eps) {
        quat_to_matrix(oq, V);
    } else {
        double st_, ct_;
        sincos(theta, &st_, &ct_);
        const double c1 = (1.0 - ct_) / (theta * theta);
        const double c2 = (theta - st_) / (theta * theta * theta);
        const double w2 = wz * wz;
        V[0] = 1.0 + c2 * (-w2), V[1] = c1 * (-wz), V[2] = 0.0;
        V[3] = c1 * wz, V[4] = 1.0 + c2 * (-w2), V[5] = 0.0;
        V[6] = 0.0, V[7] = 0.0, V[8] = 1.0;
    }
    ot[0] = V[0] * ux + V[1] * uy;
    ot[1] = V[3] * ux + V[4] * uy;
    ot[2] = V[6] * ux + V[7] * uy;
}

// current_estimate = last_robot_pose * relative_wheel_odometry   (Registration.cpp:156)
__device__ void pose_init(PoseState *ps, const RegArgs &a) {
    const double lq[4] = {a.last.qx, a.last.qy, a.last.qz, a.last.qw}, lt[3] = {a.last.tx, a.last.ty, a.last.tz};
    const double oq[4] = {a.odom.qx, a.odom.qy, a.odom.qz, a.odom.qw}, ot[3] = {a.odom.tx, a.odom.ty, a.odom.tz};
    double q[4], t[3], R[9];
    se3_compose(lq, lt, oq, ot, q, t);
    quat_to_matrix(q, R);
    for (int k = 0; k < 4; ++k) ps->q[k] = q[k], ps->qp[k] = q[k];
    for (int k = 0; k < 3; ++k) ps->t[k] = t[k];
    for (int k = 0; k < 9; ++k) ps->R[k] = R[k];
    for (int k = 0; k < 3; ++k) ps->tp[k] = t[k];
    ps->tau = a.tau, ps->conv = a.conv, ps->fixed_reg = a.fixed_reg, ps->beta = 0.0;
    ps->adaptive = a.adaptive, ps->max_iter = a.max_iter;
    ps->iter = 0, ps->done = a.max_iter <= 0 ? 1 : 0, ps->status = KICP_OK;
}
__device__ void result_init(kicp_reg_result *r, const PoseState *ps) {
    for (int k = 0; k < 4; ++k) r->pose[k] = ps->q[k];
    for (int k = 0; k < 3; ++k) r->pose[4 + k] = ps->t[k];
    r->beta = 0.0, r->last_dx_norm = 0.0, r->iterations = 0, r->status = ps->status;
}

// ComputePerturbation's tail + motion model + pose update + convergence test (one thread).  `s` holds the (all-reduced)
// sums of this iteration; `res` (optional) receives the public result fields.
__device__ void solve_and_update(PoseState *ps, const double *s, kicp_reg_result *res, int *iters_out) {
    const int j = ps->iter;
    if (res && j < KICP_MAX_ITERATIONS)
        for (int k = 0; k < 8; ++k) res->sums[j][k] = k < 7 ? s[k] : 0.0;
    const double N = s[5];
    if (j == 0) {
        // ComputeOdometryRegularization (Registration.cpp:48-60): beta = 1 / (mean |T0 p - n|^2 + DBL_MIN), computed
        // once from the first association; the fixed value otherwise (:171-177)
        ps->beta = ps->adaptive ? 1.0 / (s[6] / N + DBL_MIN) : ps->fixed_reg;
        if (res) res->beta = ps->beta;
    }
    // JTJ /= N; JTr /= N; JTJ += diag(beta, 0); dx = -(JTJ^-1 JTr)     (Registration.cpp:119-125)
    const double a = s[0] / N + ps->beta, b = s[1] / N, d = s[2] / N + 0.0;
    const double r0 = s[3] / N, r1 = s[4] / N;
    const double invdet = 1.0 / (a * d - b * b);
    const double i00 = d * invdet, i01 = -b * invdet, i10 = -b * invdet, i11 = a * invdet;
    const double dx0 = -(i00 * r0 + i01 * r1), dx1 = -(i10 * r0 + i11 * r1);
    // motion_model (Registration.cpp:159-167), epsilon = DBL_MIN
    double sn, cs;
    sincos(dx1, &sn, &cs);
    const double ux = dx0 * sn / (dx1 + DBL_MIN);
    const double uy = dx0 * (1.0 - cs) / (dx1 + DBL_MIN);
    double dq[4], dt[3], nq[4], nt[3], cq[4], ct[3], nR[9];
    for (int k = 0; k < 4; ++k) cq[k] = ps->q[k];
    for (int k = 0; k < 3; ++k) ct[k] = ps->t[k];
    se3_exp_planar(ux, uy, dx1, dq, dt);
    se3_compose(cq, ct, dq, dt, nq, nt);  // current_estimate = current_estimate * delta_motion  (:182)
    quat_to_matrix(nq, nR);
    for (int k = 0; k < 4; ++k) ps->qp[k] = ps->q[k];
    for (int k = 0; k < 3; ++k) ps->tp[k] = ps->t[k];
    for (int k = 0; k < 4; ++k) ps->q[k] = nq[k];
    for (int k = 0; k < 3; ++k) ps->t[k] = nt[k];
    for (int k = 0; k < 9; ++k) ps->R[k] = nR[k];
    const double dxn = sqrt(dx0 * dx0 + dx1 * dx1);
    ps->iter = j + 1;
    int done = (dxn < ps->conv) || (j + 1 >= ps->max_iter);  // break BEFORE re-association (:184)
    if (!(N > 0.0)) {  // the reference has no guard: the pose is NaN from here on; stop early and say so
        ps->status = KICP_WARN_NO_CORRESPONDENCES;
        done = 1;
    }
    ps->done = done;
    if (res) {
        if (j < KICP_MAX_ITERATIONS) res->dx[j][0] = dx0, res->dx[j][1] = dx1;
        res->last_dx_norm = dxn;
        res->iterations = j + 1;
        for (int k = 0; k < 4; ++k) res->pose[k] = nq[k];
        for (int k = 0; k < 3; ++k) res->pose[4 + k] = nt[k];
        res->status = ps->status;
    }
    if (iters_out) *iters_out = j + 1;
}
