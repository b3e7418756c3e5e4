// TEST INFRASTRUCTURE — NOT PRODUCT CODE.  See kicp_oracle.hpp for the scope statement.
// Compiled with -ffp-contract=off: every expression is evaluated left-to-right in plain IEEE
// double arithmetic, so that decision points (floor, <, argmin) are reproducible.
#include "kicp_oracle.hpp"

#include <algorithm>
#include <cmath>
#include <limits>
#include <thread>

namespace kicp_oracle {

double norm(const Vec3 &a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }
static inline double squaredNorm(const Vec3 &a) { return a.x * a.x + a.y * a.y + a.z * a.z; }

// ------------------------------------------------------------------ Sophus-style SE3 math
SE3 SE3::from_pose7(const double *p) {
    SE3 T;
    T.q = {p[0], p[1], p[2], p[3]};
    T.t = {p[4], p[5], p[6]};
    return T;
}
void SE3::to_pose7(double *p) const {
    p[0] = q.x, p[1] = q.y, p[2] = q.z, p[3] = q.w;
    p[4] = t.x, p[5] = t.y, p[6] = t.z;
}

// Sophus SO3Base::operator*(Point): uv = 2 (q.vec x p); p + w uv + q.vec x uv
Vec3 rotate(const Quat &q, const Vec3 &p) {
    const Vec3 qv{q.x, q.y, q.z};
    Vec3 uv = cross(qv, p);
    uv = uv + uv;
    return p + q.w * uv + cross(qv, uv);
}
Vec3 transform(const SE3 &T, const Vec3 &p) { return rotate(T.q, p) + T.t; }

// Sophus SO3Base::operator*(SO3): Hamilton product, then the SO3(quaternion) ctor normalises.
static Quat quat_mul_normalized(const Quat &a, const Quat &b) {
    Quat r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    const double len = std::sqrt(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
    r.x /= len, r.y /= len, r.z /= len, r.w /= len;
    return r;
}
SE3 compose(const SE3 &a, const SE3 &b) {
    SE3 r;
    r.q = quat_mul_normalized(a.q, b.q);
    r.t = a.t + rotate(a.q, b.t);
    return r;
}
SE3 inverse(const SE3 &a) {
    SE3 r;
    r.q = {-a.q.x, -a.q.y, -a.q.z, a.q.w};
    const Vec3 rt = rotate(r.q, a.t);
    r.t = {-rt.x, -rt.y, -rt.z};
    return r;
}

struct Mat3 {
    double m[3][3];
};
static Mat3 hat(const Vec3 &w) { return {{{0, -w.z, w.y}, {w.z, 0, -w.x}, {-w.y, w.x, 0}}}; }
static Mat3 matmul(const Mat3 &a, const Mat3 &b) {
    Mat3 r{};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}
static Vec3 matvec(const Mat3 &a, const Vec3 &v) {
    return {a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z, a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
            a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z};
}
static Mat3 quat_matrix(const Quat &q) {  // Eigen::Quaternion::toRotationMatrix
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    return {{{1 - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1 - (txx + tzz), tyz - twx}, {txz - twy, tyz + twx, 1 - (txx + tyy)}}};
}

static constexpr double kSophusEps = 1e-10;  // Sophus::Constants<double>::epsilon()

// Sophus SO3::expAndTheta
static Quat so3_exp_and_theta(const Vec3 &omega, double *theta) {
    const double theta_sq = squaredNorm(omega);
    double imag_factor, real_factor;
    if (theta_sq < kSophusEps * kSophusEps) {
        *theta = 0.0;
        const double theta_po4 = theta_sq * theta_sq;
        imag_factor = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * theta_po4;
        real_factor = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * theta_po4;
    } else {
        *theta = std::sqrt(theta_sq);
        const double half_theta = 0.5 * (*theta);
        imag_factor = std::sin(half_theta) / (*theta);
        real_factor = std::cos(half_theta);
    }
    return {imag_factor * omega.x, imag_factor * omega.y, imag_factor * omega.z, real_factor};
}

// Sophus SE3::exp: t = V * upsilon, V = I + (1-cos)/th^2 W + (th-sin)/th^3 W^2, V = R when th < eps
SE3 se3_exp(const double a[6]) {
    const Vec3 upsilon{a[0], a[1], a[2]}, omega{a[3], a[4], a[5]};
    double theta;
    SE3 r;
    r.q = so3_exp_and_theta(omega, &theta);
    const Mat3 Omega = hat(omega);
    const Mat3 Omega_sq = matmul(Omega, Omega);
    Mat3 V;
    if (theta < kSophusEps) {
        V = quat_matrix(r.q);
    } else {
        const double theta_sq = theta * theta;
        const double c1 = (1.0 - std::cos(theta)) / theta_sq;
        const double c2 = (theta - std::sin(theta)) / (theta_sq * theta);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) V.m[i][j] = (i == j ? 1.0 : 0.0) + c1 * Omega.m[i][j] + c2 * Omega_sq.m[i][j];
    }
    r.t = matvec(V, upsilon);
    return r;
}

// Sophus SO3::logAndTheta
static Vec3 so3_log_and_theta(const Quat &q, double *theta_out) {
    const double squared_n = q.x * q.x + q.y * q.y + q.z * q.z;
    const double w = q.w;
    double two_atan_nbyw_by_n, theta;
    if (squared_n < kSophusEps * kSophusEps) {
        const double squared_w = w * w;
        two_atan_nbyw_by_n = 2.0 / w - (2.0 / 3.0) * squared_n / (w * squared_w);
        theta = 2.0 * squared_n / w;
    } else {
        const double n = std::sqrt(squared_n);
        const double atan_nbyw = (w < 0.0) ? std::atan2(-n, -w) : std::atan2(n, w);
        two_atan_nbyw_by_n = 2.0 * atan_nbyw / n;
        theta = two_atan_nbyw_by_n * n;
    }
    *theta_out = theta;
    return {two_atan_nbyw_by_n * q.x, two_atan_nbyw_by_n * q.y, two_atan_nbyw_by_n * q.z};
}
double so3_log_theta(const Quat &q) {
    double th;
    so3_log_and_theta(q, &th);
    return th;
}

// Sophus SE3::log
void se3_log(const SE3 &T, double out[6]) {
    double theta;
    const Vec3 omega = so3_log_and_theta(T.q, &theta);
    const Mat3 Omega = hat(omega);
    const Mat3 Omega_sq = matmul(Omega, Omega);
    Mat3 V_inv;
    double c;
    if (std::abs(theta) < kSophusEps) {
        c = 1.0 / 12.0;
    } else {
        const double half_theta = 0.5 * theta;
        c = (1.0 - theta * std::cos(half_theta) / (2.0 * std::sin(half_theta))) / (theta * theta);
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) V_inv.m[i][j] = (i == j ? 1.0 : 0.0) - 0.5 * Omega.m[i][j] + c * Omega_sq.m[i][j];
    const Vec3 u = matvec(V_inv, T.t);
    out[0] = u.x, out[1] = u.y, out[2] = u.z, out[3] = omega.x, out[4] = omega.y, out[5] = omega.z;
}

// ------------------------------------------------------------------ KISS-ICP v1.2.0 map
// VoxelUtils.hpp PointToVoxel: floor, not truncation.  static_cast<int> of a NaN, an infinity or a value outside the int range is
// undefined behaviour in C++; the reference's x86-64 build (cvttsd2si) gives INT_MIN for all of them, spelled out here.
static int32_t floor_to_voxel(double q) {
    const double f = std::floor(q);
    return f >= -2147483648.0 && f < 2147483648.0 ? static_cast<int32_t>(f) : INT32_MIN;
}
Voxel PointToVoxel(const Vec3 &p, double vs) { return {floor_to_voxel(p.x / vs), floor_to_voxel(p.y / vs), floor_to_voxel(p.z / vs)}; }

// VoxelHashMap.cpp voxel_shifts: centre, 6 faces, 12 edges, 8 corners
const Voxel kVoxelShifts[27] = {
    {0, 0, 0},   {1, 0, 0},   {-1, 0, 0},  {0, 1, 0},   {0, -1, 0},  {0, 0, 1},   {0, 0, -1},  {1, 1, 0},   {1, -1, 0},
    {-1, 1, 0},  {-1, -1, 0}, {1, 0, 1},   {1, 0, -1},  {-1, 0, 1},  {-1, 0, -1}, {0, 1, 1},   {0, 1, -1},  {0, -1, 1},
    {0, -1, -1}, {1, 1, 1},   {1, 1, -1},  {1, -1, 1},  {1, -1, -1}, {-1, 1, 1},  {-1, 1, -1}, {-1, -1, 1}, {-1, -1, -1}};

// VoxelHashMap::GetClosestNeighbor: per found voxel min_element by (x-q).norm() (strict <, first
// minimum wins), global minimum by strict < in shift order; init (0,0,0), DBL_MAX.
std::pair<Vec3, double> VoxelHashMap::GetClosestNeighbor(const Vec3 &query) const {
    const Voxel voxel = PointToVoxel(query, voxel_size_);
    Vec3 closest_neighbor{0, 0, 0};
    double closest_distance = std::numeric_limits<double>::max();
    for (const Voxel &s : kVoxelShifts) {
        const Voxel qv{voxel.x + s.x, voxel.y + s.y, voxel.z + s.z};
        auto search = map_.find(qv);
        if (search == map_.end()) continue;
        const std::vector<Vec3> &points = search->second;
        const Vec3 *best = &points.front();
        double best_d = norm(*best - query);
        for (size_t i = 1; i < points.size(); ++i) {
            const double d = norm(points[i] - query);
            if (d < best_d) {
                best_d = d;
                best = &points[i];
            }
        }
        if (best_d < closest_distance) {
            closest_neighbor = *best;
            closest_distance = best_d;
        }
    }
    return {closest_neighbor, closest_distance};
}

// VoxelHashMap::AddPoints: greedy, input-order dependent; min spacing checked in the point's
// own voxel only; voxel capacity max_points_per_voxel_.
void VoxelHashMap::AddPoints(const std::vector<Vec3> &points) {
    const double map_resolution = std::sqrt(voxel_size_ * voxel_size_ / max_points_per_voxel_);
    for (const Vec3 &point : points) {
        const Voxel voxel = PointToVoxel(point, voxel_size_);
        auto search = map_.find(voxel);
        if (search != map_.end()) {
            std::vector<Vec3> &voxel_points = search->second;
            if (voxel_points.size() == max_points_per_voxel_) continue;
            bool too_close = false;
            for (const Vec3 &vp : voxel_points) {
                if (norm(vp - point) < map_resolution) {
                    too_close = true;
                    break;
                }
            }
            if (too_close) continue;
            voxel_points.emplace_back(point);
        } else {
            std::vector<Vec3> voxel_points;
            voxel_points.reserve(max_points_per_voxel_);
            voxel_points.emplace_back(point);
            map_.insert({voxel, std::move(voxel_points)});
        }
    }
}

// VoxelHashMap::RemovePointsFarFromLocation: a voxel is erased when its FIRST point is >= max_distance away.
void VoxelHashMap::RemovePointsFarFromLocation(const Vec3 &origin) {
    const double max_distance2 = max_distance_ * max_distance_;
    for (auto it = map_.begin(); it != map_.end();) {
        const Vec3 &pt = it->second.front();
        if (squaredNorm(pt - origin) >= max_distance2) {
            it = map_.erase(it);
        } else {
            ++it;
        }
    }
}
void VoxelHashMap::Update(const std::vector<Vec3> &points, const Vec3 &origin) {
    AddPoints(points);
    RemovePointsFarFromLocation(origin);
}
void VoxelHashMap::Update(const std::vector<Vec3> &points, const SE3 &pose) {
    std::vector<Vec3> points_transformed(points.size());
    for (size_t i = 0; i < points.size(); ++i) points_transformed[i] = transform(pose, points[i]);
    Update(points_transformed, pose.t);
}
std::vector<Vec3> VoxelHashMap::Pointcloud() const {
    std::vector<Vec3> points;
    points.reserve(map_.size() * static_cast<size_t>(max_points_per_voxel_));
    for (const auto &kv : map_) points.insert(points.end(), kv.second.begin(), kv.second.end());
    points.shrink_to_fit();
    return points;
}
size_t VoxelHashMap::NumPoints() const {
    size_t n = 0;
    for (const auto &kv : map_) n += kv.second.size();
    return n;
}

// tsl::robin_map<Voxel, T> as VoxelDownsample uses it, restated from memory (tsl/robin_hash.h; UNPINNED, see the header):
// reserve(n) -> rehash(ceil(float(n) / 0.5f)) -> bucket count = next power of two; insert: start at hash & mask, walk while the
// walker's distance from its ideal bucket is <= the resident's; place in an empty bucket, else swap with the poorer resident and carry
// it on (richer stays on equal distance); iteration visits the buckets in index order.  With at most n distinct keys the load never
// reaches 0.5, so the table does not grow; the probe-length limits of the library (rehash after 4096 / 128 probes) are far away.
std::vector<size_t> RobinMapIterationOrder(const std::vector<Voxel> &keys, size_t reserve_count, bool mask20) {
    size_t want = static_cast<size_t>(std::ceil(static_cast<float>(reserve_count) / 0.5f));
    want = std::max(want, static_cast<size_t>(std::ceil(static_cast<float>(keys.size()) / 0.5f)));
    size_t nb = 1;
    while (nb < want) nb <<= 1;
    const size_t mask = nb - 1;
    struct Bucket {
        long dist = -1;  // distance from the ideal bucket, -1 = empty
        size_t idx = 0;
    };
    std::vector<Bucket> b(nb);
    for (size_t i = 0; i < keys.size(); ++i) {
        size_t h = VoxelHash()(keys[i]);
        if (mask20) h &= (static_cast<size_t>(1) << 20) - 1;
        size_t ib = h & mask;
        long dist = 0;
        while (dist <= b[ib].dist) ib = (ib + 1) & mask, ++dist;  // (keys are distinct: no equality test needed)
        Bucket carry{dist, i};
        while (b[ib].dist >= 0) {  // robin hood: the walker takes the bucket of a resident that is closer to home, the resident walks on
            if (carry.dist > b[ib].dist) std::swap(carry, b[ib]);
            ib = (ib + 1) & mask, ++carry.dist;
        }
        b[ib] = carry;
    }
    std::vector<size_t> order;
    order.reserve(keys.size());
    for (const Bucket &k : b)
        if (k.dist >= 0) order.push_back(k.idx);
    return order;
}

static int g_downsample_order = 0;
void SetDownsampleOrder(int mode) { g_downsample_order = mode; }
int GetDownsampleOrder() { return g_downsample_order; }

// VoxelUtils.cpp VoxelDownsample: first point (input order) per voxel.  Output order: the order of first occurrence by default
// (the reference's is robin_map iteration order — a permutation of it; SetDownsampleOrder(1 | 2) emits that order as recalled).
std::vector<Vec3> VoxelDownsample(const std::vector<Vec3> &frame, double voxel_size) {
    std::unordered_map<Voxel, size_t, VoxelHash> grid;
    grid.reserve(frame.size());
    std::vector<Vec3> out;
    std::vector<Voxel> keys;
    for (const Vec3 &p : frame) {
        const Voxel v = PointToVoxel(p, voxel_size);
        if (grid.find(v) == grid.end()) {
            grid.insert({v, out.size()});
            out.push_back(p);
            keys.push_back(v);
        }
    }
    if (g_downsample_order == 1 || g_downsample_order == 2) {
        const std::vector<size_t> order = RobinMapIterationOrder(keys, frame.size(), g_downsample_order == 2);
        std::vector<Vec3> permuted(out.size());
        for (size_t k = 0; k < order.size(); ++k) permuted[k] = out[order[k]];
        return permuted;
    }
    return out;
}

// Preprocessing.cpp Preprocessor::Preprocess: deskew p <- exp((s-1) log(relative_motion)) p with
// stamps normalised to [0,1]; then keep min_range < |p| < max_range.
std::vector<Vec3> Preprocess(const std::vector<Vec3> &frame, const std::vector<double> &timestamps,
                             const SE3 &relative_motion, double max_range, double min_range, bool deskew) {
    std::vector<Vec3> deskewed;
    const std::vector<Vec3> *src = &frame;
    if (deskew && !timestamps.empty()) {
        const auto mm = std::minmax_element(timestamps.begin(), timestamps.end());
        const double min_time = *mm.first, max_time = *mm.second;
        double omega[6];
        se3_log(relative_motion, omega);
        deskewed.resize(frame.size());
        for (size_t i = 0; i < frame.size(); ++i) {
            const double stamp = (timestamps[i] - min_time) / (max_time - min_time);
            double a[6];
            for (int k = 0; k < 6; ++k) a[k] = (stamp - 1.0) * omega[k];
            deskewed[i] = transform(se3_exp(a), frame[i]);
        }
        src = &deskewed;
    }
    std::vector<Vec3> out;
    out.reserve(src->size());
    for (const Vec3 &p : *src) {
        const double r = norm(p);
        if (r < max_range && r > min_range) out.push_back(p);
    }
    return out;
}

// ------------------------------------------------------------------ Registration.cpp
namespace {
constexpr double epsilon = std::numeric_limits<double>::min();  // Registration.cpp:46 (DBL_MIN, not epsilon())

using Correspondences = std::vector<std::pair<Vec3, Vec3>>;

// Registration.cpp:62-81.  Index-ordered (the reference's concurrent_vector order is nondeterministic).
Correspondences DataAssociation(const std::vector<Vec3> &points, const VoxelHashMap &voxel_map, const SE3 &T,
                                double max_correspondance_distance, int num_threads) {
    Correspondences correspondences;
    correspondences.reserve(points.size());
    if (num_threads <= 1) {
        for (const Vec3 &point : points) {
            const auto [closest_neighbor, distance] = voxel_map.GetClosestNeighbor(transform(T, point));
            if (distance < max_correspondance_distance) correspondences.emplace_back(point, closest_neighbor);
        }
        return correspondences;
    }
    // static contiguous ranges, concatenated in thread order => same order as the sequential pass
    std::vector<Correspondences> parts(num_threads);
    std::vector<std::thread> workers;
    const size_t n = points.size();
    for (int t = 0; t < num_threads; ++t) {
        workers.emplace_back([&, t]() {
            const size_t lo = n * t / num_threads, hi = n * (t + 1) / num_threads;
            parts[t].reserve(hi - lo);
            for (size_t i = lo; i < hi; ++i) {
                const auto [closest_neighbor, distance] = voxel_map.GetClosestNeighbor(transform(T, points[i]));
                if (distance < max_correspondance_distance) parts[t].emplace_back(points[i], closest_neighbor);
            }
        });
    }
    for (auto &w : workers) w.join();
    for (auto &p : parts) correspondences.insert(correspondences.end(), p.begin(), p.end());
    return correspondences;
}

// std::transform_reduce as libstdc++ (GCC 13) evaluates it for random-access iterators — the reference calls it at
// Registration.cpp:50-55 and :104-113.  It is NOT a left fold: elements are combined in groups of four,
// init = op(init, op(op(f(x0), f(x1)), op(f(x2), f(x3)))), then the remainder one by one.  Mirrored here so that the
// single-threaded reference and the oracle agree bit for bit.
template <typename T, typename It, typename BinaryOp, typename UnaryOp>
T transform_reduce_like_libstdcxx(It first, It last, T init, BinaryOp binary_op, UnaryOp unary_op) {
    while ((last - first) >= 4) {
        T v1 = binary_op(unary_op(first[0]), unary_op(first[1]));
        T v2 = binary_op(unary_op(first[2]), unary_op(first[3]));
        T v3 = binary_op(v1, v2);
        init = binary_op(init, v3);
        first += 4;
    }
    for (; first != last; ++first) init = binary_op(init, unary_op(*first));
    return init;
}

// Registration.cpp:48-60
double ComputeOdometryRegularization(const Correspondences &associations, const SE3 &odometry_initial_guess,
                                     double *sumsq_out) {
    const double sum_of_squared_residuals = transform_reduce_like_libstdcxx(
        associations.cbegin(), associations.cend(), 0.0, [](double a, double b) { return a + b; },
        [&](const std::pair<Vec3, Vec3> &association) {
            return squaredNorm(transform(odometry_initial_guess, association.first) - association.second);
        });
    const double N = static_cast<double>(associations.size());
    const double mean_squared_residual = sum_of_squared_residuals / N;
    if (sumsq_out) *sumsq_out = sum_of_squared_residuals;
    return 1.0 / (mean_squared_residual + epsilon);
}

// Registration.cpp:83-126.  J = [R e_x | R (-p_y, p_x, 0)], r = T p - n, w == 1.
void ComputePerturbation(const Correspondences &correspondences, const SE3 &current_estimate, double beta, double dx[2],
                         IterSums *sums_out) {
    struct LS {
        double JTJ00, JTJ01, JTJ11, JTr0, JTr1;
    };
    const Vec3 c0 = rotate(current_estimate.q, Vec3{1.0, 0.0, 0.0});
    const LS total = transform_reduce_like_libstdcxx(
        correspondences.cbegin(), correspondences.cend(), LS{0, 0, 0, 0, 0},
        [](LS a, const LS &b) {
            return LS{a.JTJ00 + b.JTJ00, a.JTJ01 + b.JTJ01, a.JTJ11 + b.JTJ11, a.JTr0 + b.JTr0, a.JTr1 + b.JTr1};
        },
        [&](const std::pair<Vec3, Vec3> &c) {
            const Vec3 &source = c.first, &target = c.second;
            const Vec3 residual = transform(current_estimate, source) - target;
            const Vec3 c1 = rotate(current_estimate.q, Vec3{-source.y, source.x, 0.0});
            return LS{dot(c0, c0), dot(c0, c1), dot(c1, c1), dot(c0, residual), dot(c1, residual)};
        });
    const double JTJ00 = total.JTJ00, JTJ01 = total.JTJ01, JTJ11 = total.JTJ11, JTr0 = total.JTr0, JTr1 = total.JTr1;
    const double num_correspondences = static_cast<double>(correspondences.size());
    if (sums_out) *sums_out = {JTJ00, JTJ01, JTJ11, JTr0, JTr1, num_correspondences, 0.0};
    // JTJ /= N; JTr /= N; JTJ += diag(beta, 0); dx = -(JTJ^-1 JTr)      (:119-125)
    const double a = JTJ00 / num_correspondences + beta;
    const double b = JTJ01 / num_correspondences;
    const double d = JTJ11 / num_correspondences + 0.0;
    const double r0 = JTr0 / num_correspondences, r1 = JTr1 / num_correspondences;
    // Eigen fixed-size 2x2 inverse: adjugate scaled by 1/det
    const double invdet = 1.0 / (a * d - b * b);
    const double i00 = d * invdet, i01 = -b * invdet, i10 = -b * invdet, i11 = a * invdet;
    dx[0] = -(i00 * r0 + i01 * r1);
    dx[1] = -(i10 * r0 + i11 * r1);
}
}  // namespace

// Registration.cpp:151-190
SE3 ComputeRobotMotion(const std::vector<Vec3> &frame, const VoxelHashMap &voxel_map, const SE3 &last_robot_pose,
                       const SE3 &relative_wheel_odometry, double max_correspondence_distance, const RegParams &params,
                       RegStats *stats, int num_threads) {
    SE3 current_estimate = compose(last_robot_pose, relative_wheel_odometry);
    if (stats) *stats = RegStats{};
    if (voxel_map.Empty()) return current_estimate;

    // motion_model (:159-167): unicycle arc, eps = DBL_MIN so theta == 0 exactly gives dx(0) = dx(1) = 0
    auto motion_model = [](const double c[2]) {
        double dx[6] = {0, 0, 0, 0, 0, 0};
        const double displacement = c[0], theta = c[1];
        dx[0] = displacement * std::sin(theta) / (theta + epsilon);
        dx[1] = displacement * (1.0 - std::cos(theta)) / (theta + epsilon);
        dx[5] = theta;
        return se3_exp(dx);
    };
    Correspondences correspondences =
        DataAssociation(frame, voxel_map, current_estimate, max_correspondence_distance, num_threads);
    if (stats) stats->associations = 1;

    double sumsq0 = 0.0;
    const double regularization_term =
        params.use_adaptive_odometry_regularization
            ? ComputeOdometryRegularization(correspondences, current_estimate, &sumsq0)
            : params.fixed_regularization;
    if (stats) stats->beta = regularization_term;

    for (int j = 0; j < params.max_num_iterations; ++j) {
        double dx[2];
        IterSums sums;
        ComputePerturbation(correspondences, current_estimate, regularization_term, dx, &sums);
        if (j == 0) sums.sumsq = sumsq0;
        current_estimate = compose(current_estimate, motion_model(dx));
        const double dxn = std::sqrt(dx[0] * dx[0] + dx[1] * dx[1]);
        if (stats) {
            stats->iterations = j + 1;
            stats->sums.push_back(sums);
            stats->dx.push_back(dx[0]);
            stats->dx.push_back(dx[1]);
            stats->last_dx_norm = dxn;
        }
        if (dxn < params.convergence_criterion) break;
        correspondences = DataAssociation(frame, voxel_map, current_estimate, max_correspondence_distance, num_threads);
        if (stats) stats->associations += 1;
    }
    return current_estimate;
}

// ------------------------------------------------------------------ CorrespondenceThreshold.cpp
// :29-34
static double OdometryErrorInPointSpace(const SE3 &pose, double max_range) {
    const double theta = so3_log_theta(pose.q);
    const double delta_rot = 2.0 * max_range * std::sin(theta / 2.0);
    const double delta_trans = norm(pose.t);
    return delta_trans + delta_rot;
}
// :49-56
double CorrespondenceThreshold::ComputeThreshold() const {
    if (!use_adaptive_threshold_) return fixed_threshold_;
    const double sigma_odom = std::sqrt(odom_sse_ / num_samples_);
    const double sigma_map = map_discretization_error_;
    return 3.0 * (sigma_map + sigma_odom);
}
// :58-64
void CorrespondenceThreshold::UpdateOdometryError(const SE3 &odometry_error) {
    if (!use_adaptive_threshold_) return;
    const double e = OdometryErrorInPointSpace(odometry_error, max_range_);
    odom_sse_ += e * e;
    num_samples_ += 1.0;
}

}  // namespace kicp_oracle
