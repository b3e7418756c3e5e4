// Implementation of the C++ facade over the C ABI (libkicp_b200.so).  Builds libkinematic_icp_b200.so, the library a
// ROS 2 workspace links instead of kinematic_icp_registration / _threshold / _pipeline (INTEGRATION.md).
#include <array>
#include <cstdlib>
#include <mutex>
#include <string>
#include <utility>

#include "kicp/facade_core.hpp"
#include "kicp/runtime.hpp"
#ifndef KICP_FACADE_NO_PIPELINE
#include "kicp/facade_pipeline.hpp"
#endif

namespace kicp {
kicp_ctx *default_context() {
    static kicp_ctx *ctx = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *dev = std::getenv("KICP_DEVICE");
        check(kicp_ctx_create(dev ? std::atoi(dev) : 0, &ctx), "kicp_ctx_create");
        // KICP_DOWNSAMPLE_ORDER=0|1: context option "downsample_order" (kicp.h), for programs that cannot set it themselves; any other
        // value throws
        if (const char *order = std::getenv("KICP_DOWNSAMPLE_ORDER")) {
            const std::string v = order;
            check(kicp_ctx_set_option(ctx, "downsample_order", v == "0" ? 0 : v == "1" ? 1 : -1), "KICP_DOWNSAMPLE_ORDER");
        }
        // KICP_CORRESPONDENCES=0|1: context option "correspondences" (every frame reports its correspondences at the returned pose,
        // KinematicICP::LastCorrespondenceStats); any other value throws
        if (const char *corr = std::getenv("KICP_CORRESPONDENCES")) {
            const std::string v = corr;
            check(kicp_ctx_set_option(ctx, "correspondences", v == "0" ? 0 : v == "1" ? 1 : -1), "KICP_CORRESPONDENCES");
        }
    });
    return ctx;
}
}  // namespace kicp

namespace kinematic_icp {

// registration/Registration.cpp:132-149 (the TBB thread cap has no GPU meaning)
KinematicRegistration::KinematicRegistration(const int max_num_iteration, const double convergence_criterion, const int max_num_threads,
                                             const bool use_adaptive_odometry_regularization, const double fixed_regularization)
    : max_num_iterations_(max_num_iteration),
      convergence_criterion_(convergence_criterion),
      max_num_threads_(max_num_threads),
      use_adaptive_odometry_regularization_(use_adaptive_odometry_regularization),
      fixed_regularization_(fixed_regularization) {}

// registration/Registration.cpp:151-190, on the device
Sophus::SE3d KinematicRegistration::ComputeRobotMotion(const std::vector<Eigen::Vector3d> &frame, const kiss_icp::VoxelHashMap &voxel_map,
                                                       const Sophus::SE3d &last_robot_pose, const Sophus::SE3d &relative_wheel_odometry,
                                                       const double max_correspondence_distance) {
    double last[7], odom[7], out[7];
    kicp::to_pose7(last_robot_pose, last);
    kicp::to_pose7(relative_wheel_odometry, odom);
    kicp_reg_params p;
    p.max_num_iterations = max_num_iterations_;
    p.use_adaptive_odometry_regularization = use_adaptive_odometry_regularization_ ? 1 : 0;
    p.convergence_criterion = convergence_criterion_;
    p.fixed_regularization = fixed_regularization_;
    kicp::check(kicp_register(voxel_map.handle_, kicp::xyz(frame), (int64_t)frame.size(), last, odom, max_correspondence_distance, &p, out,
                              nullptr),
                "kicp_register");
    return kicp::from_pose7(out);
}

// correspondence_threshold/CorrespondenceThreshold.cpp:36-64
CorrespondenceThreshold::CorrespondenceThreshold(const double map_discretization_error, const double max_range,
                                                 const bool use_adaptive_threshold, const double fixed_threshold)
    : map_discretization_error_(map_discretization_error),
      max_range_(max_range),
      use_adaptive_threshold_(use_adaptive_threshold),
      fixed_threshold_(fixed_threshold),
      odom_sse_(0.0),
      num_samples_(1e-8) {}

double CorrespondenceThreshold::ComputeThreshold() const {
    if (!use_adaptive_threshold_) return fixed_threshold_;
    const double sigma_odom = std::sqrt(odom_sse_ / num_samples_);
    return 3.0 * (map_discretization_error_ + sigma_odom);
}

void CorrespondenceThreshold::Reset() {
    odom_sse_ = 0.0;
    num_samples_ = 1e-8;
}

void CorrespondenceThreshold::UpdateOdometryError(const Sophus::SE3d &odometry_error) {
    if (!use_adaptive_threshold_) return;
    // odometry error expressed in point space (:29-34): translation plus the chord a max_range lever arm sweeps
    const double theta = odometry_error.so3().logAndTheta().theta;
    const double e = odometry_error.translation().norm() + 2.0 * max_range_ * std::sin(theta / 2.0);
    odom_sse_ += e * e;
    num_samples_ += 1.0;
}

#ifndef KICP_FACADE_NO_PIPELINE  // the reference's own pipeline/KinematicICP.cpp can be compiled in its place
namespace pipeline {
// pipeline/KinematicICP.hpp:73-79
KinematicICP::KinematicICP(const Config &config)
    : registration_(config.max_num_iterations, config.convergence_criterion, config.max_num_threads,
                    config.use_adaptive_odometry_regularization, config.fixed_regularization),
      correspondence_threshold_(config.map_resolution(), config.max_range, config.use_adaptive_threshold, config.fixed_threshold),
      config_(config),
      preprocessor_(config.max_range, config.min_range, config.deskew, config.max_num_threads),
      local_map_(config.voxel_size, config.max_range, config.max_points_per_voxel) {}

// pipeline/KinematicICP.hpp:85-89
void KinematicICP::SetPose(const Sophus::SE3d &pose) {
    last_pose_ = pose;
    local_map_.Clear();
    correspondence_threshold_.Reset();
}

// pipeline/KinematicICP.cpp:48-85: one kicp_register_frame call does the per-point work (ingest, de-skew, range filter,
// base transform, both voxel down-samples, registration, map update) with the frame resident in HBM throughout; the
// scalar threshold model and the pose bookkeeping stay here.
KinematicICP::Vector3dVectorTuple KinematicICP::RegisterFrame(const kicp_frame_input &input, const Sophus::SE3d &lidar_to_base,
                                                              const Sophus::SE3d &relative_odometry) {
    RegisterOnDevice(&input, &lidar_to_base, 1, false, relative_odometry, KICP_STAGE_F64);
    return StagedClouds();
}

namespace {
// TimeStampHandler::ProcessTimestamps (utils/TimeStampHandler.cpp:108-139) with the stamps decoded and reduced on the device, by
// kicp_frame_stage (host records) or kicp_frame_stage_device
kicp::SweepTiming stage_frame(decltype(&kicp_frame_stage) stage, const char *where, const kicp::PointCloud2View &msg, double header_stamp,
                              double &last_processed_stamp, double range[2]) {
    const kicp_frame_input input = kicp::make_frame_input(msg);
    const kicp::StampField field = kicp::stamp_field(msg);
    int64_t n_stamps = 0;
    kicp::check(stage(kicp::default_context(), &input, field.datatype, static_cast<int32_t>(field.offset), range, &n_stamps), where);
    return kicp::sweep_timing(n_stamps > 0, range[0], range[1], header_stamp, last_processed_stamp);
}

// laser_geometry::LaserProjection::projectLaser + ProcessTimestamps on the device (the reference's use_2d_lidar path), by
// kicp_frame_stage_laser_scan (host ranges) or kicp_frame_stage_laser_scan_device
kicp::SweepTiming stage_laser_scan(decltype(&kicp_frame_stage_laser_scan) stage, const char *where, const kicp::LaserScanView &scan,
                                   double header_stamp, double &last_processed_stamp, double range[2]) {
    const kicp_laser_scan s = kicp::make_laser_scan(scan);
    int64_t n_points = 0;
    kicp::check(stage(kicp::default_context(), &s, range, &n_points), where);
    return kicp::sweep_timing(n_points > 0, range[0], range[1], header_stamp, last_processed_stamp);
}
}  // namespace

kicp::SweepTiming KinematicICP::StageFrame(const kicp::PointCloud2View &msg, double header_stamp, double &last_processed_stamp) {
    staged_sweep_ = stage_frame(kicp_frame_stage, "kicp_frame_stage", msg, header_stamp, last_processed_stamp, staged_window_);
    return staged_sweep_;
}
kicp::SweepTiming KinematicICP::StageDeviceFrame(const kicp::PointCloud2View &msg, double header_stamp, double &last_processed_stamp) {
    staged_sweep_ = stage_frame(kicp_frame_stage_device, "kicp_frame_stage_device", msg, header_stamp, last_processed_stamp, staged_window_);
    return staged_sweep_;
}
kicp::SweepTiming KinematicICP::StageLaserScan(const kicp::LaserScanView &scan, double header_stamp, double &last_processed_stamp) {
    staged_sweep_ = stage_laser_scan(kicp_frame_stage_laser_scan, "kicp_frame_stage_laser_scan", scan, header_stamp, last_processed_stamp,
                                     staged_window_);
    return staged_sweep_;
}
kicp::SweepTiming KinematicICP::StageDeviceLaserScan(const kicp::LaserScanView &scan, double header_stamp, double &last_processed_stamp) {
    staged_sweep_ = stage_laser_scan(kicp_frame_stage_laser_scan_device, "kicp_frame_stage_laser_scan_device", scan, header_stamp,
                                     last_processed_stamp, staged_window_);
    return staged_sweep_;
}

KinematicICP::Vector3dVectorTuple KinematicICP::RegisterStagedFrame(const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry) {
    RegisterOnDevice(nullptr, &lidar_to_base, 1, false, relative_odometry, KICP_STAGE_F64);
    return StagedClouds();
}

// the frame of several LiDARs, staged with one kicp_frame_stage_sensors call; the interval by sweep_timing's rule per sensor, on the
// sensor's own clock (its stamps' range on the common clock minus its offset), the latest end winning
kicp::SweepTiming KinematicICP::StageSensors(const std::vector<kicp::SensorFrame> &sensors, double &last_processed_stamp) {
    std::vector<kicp_sensor_input> in(sensors.size());
    for (size_t i = 0; i < sensors.size(); ++i) {
        const kicp::SensorFrame &s = sensors[i];
        kicp_sensor_input &d = in[i];
        d = kicp_sensor_input{};
        d.device = s.device ? 1 : 0, d.time_offset = s.offset();
        if (s.kind == kicp::SensorFrame::Kind::LaserScan) {
            d.kind = KICP_SENSOR_LASER_SCAN, d.scan = kicp::make_laser_scan(s.scan);
        } else {
            const kicp::StampField field = kicp::stamp_field(s.cloud);
            d.kind = KICP_SENSOR_POINTS, d.points = kicp::make_frame_input(s.cloud);
            d.stamp_datatype = field.datatype, d.stamp_offset = static_cast<int32_t>(field.offset);
        }
    }
    std::vector<kicp_sensor_stats> stats(sensors.size());
    double range[2];
    kicp::check(kicp_frame_stage_sensors(kicp::default_context(), in.data(), static_cast<int32_t>(in.size()), range, stats.data()),
                "kicp_frame_stage_sensors");
    kicp::SweepTiming t;
    t.begin = last_processed_stamp;
    for (size_t i = 0; i < sensors.size(); ++i) {
        double last = last_processed_stamp;
        const double off = in[i].time_offset;
        const kicp::SweepTiming ti = kicp::sweep_timing(stats[i].n_stamps > 0, stats[i].stamp_range[0] - off, stats[i].stamp_range[1] - off,
                                                        sensors[i].header_stamp, last);
        t.end = i == 0 || ti.end > t.end ? ti.end : t.end;
    }
    last_processed_stamp = t.end;
    staged_sweep_ = t, staged_window_[0] = range[0], staged_window_[1] = range[1];
    return t;
}

KinematicICP::Vector3dVectorTuple KinematicICP::RegisterStagedSensors(const std::vector<Sophus::SE3d> &lidar_to_base,
                                                                      const Sophus::SE3d &relative_odometry) {
    RegisterOnDevice(nullptr, lidar_to_base.data(), lidar_to_base.size(), true, relative_odometry, KICP_STAGE_F64);
    return StagedClouds();
}

std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> KinematicICP::RegisterStagedSensorsPointCloud2(
    const std::vector<Sophus::SE3d> &lidar_to_base, const Sophus::SE3d &relative_odometry) {
    RegisterOnDevice(nullptr, lidar_to_base.data(), lidar_to_base.size(), true, relative_odometry, KICP_STAGE_F32);
    return StagedCloudsPointCloud2();
}

KinematicICP::Vector3dVectorTuple KinematicICP::RegisterStagedFrame(const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry,
                                                                    const std::vector<kicp::OdometrySample> &samples) {
    RegisterOnDevice(nullptr, &lidar_to_base, 1, false, relative_odometry, KICP_STAGE_F64, &samples);
    return StagedClouds();
}
std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> KinematicICP::RegisterStagedFramePointCloud2(
    const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry, const std::vector<kicp::OdometrySample> &samples) {
    RegisterOnDevice(nullptr, &lidar_to_base, 1, false, relative_odometry, KICP_STAGE_F32, &samples);
    return StagedCloudsPointCloud2();
}
KinematicICP::Vector3dVectorTuple KinematicICP::RegisterStagedSensors(const std::vector<Sophus::SE3d> &lidar_to_base,
                                                                      const Sophus::SE3d &relative_odometry,
                                                                      const std::vector<kicp::OdometrySample> &samples) {
    RegisterOnDevice(nullptr, lidar_to_base.data(), lidar_to_base.size(), true, relative_odometry, KICP_STAGE_F64, &samples);
    return StagedClouds();
}
std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> KinematicICP::RegisterStagedSensorsPointCloud2(
    const std::vector<Sophus::SE3d> &lidar_to_base, const Sophus::SE3d &relative_odometry, const std::vector<kicp::OdometrySample> &samples) {
    RegisterOnDevice(nullptr, lidar_to_base.data(), lidar_to_base.size(), true, relative_odometry, KICP_STAGE_F32, &samples);
    return StagedCloudsPointCloud2();
}

// the correspondence report of the last frame on the process-wide context (zero without option "correspondences")
kicp_corr_stats KinematicICP::LastCorrespondenceStats() const {
    kicp_corr_stats st{};
    kicp::check(kicp_frame_correspondences(kicp::default_context(), &st), "kicp_frame_correspondences");
    return st;
}
void KinematicICP::SetCorrespondences(bool on) {
    kicp::check(kicp_ctx_set_option(kicp::default_context(), "correspondences", on ? 1 : 0), "kicp_ctx_set_option");
}
void KinematicICP::SetMapUpdate(const kicp_map_update_policy &policy) {
    kicp::check(kicp_ctx_set_map_update(kicp::default_context(), &policy), "kicp_ctx_set_map_update");
}
int32_t KinematicICP::LastMapUpdate() const {
    int32_t outcome = KICP_FRAME_UPDATE_NONE;
    kicp::check(kicp_frame_map_update(kicp::default_context(), &outcome), "kicp_frame_map_update");
    return outcome;
}
void KinematicICP::SetFreeSpace(int32_t min_misses, double end_margin) {
    const kicp_free_space_params params{end_margin, min_misses};
    kicp::check(kicp_ctx_set_free_space(kicp::default_context(), &params), "kicp_ctx_set_free_space");
}
kicp_free_space_stats KinematicICP::LastFreeSpace() const {
    kicp_free_space_stats st{};
    kicp::check(kicp_frame_free_space(kicp::default_context(), &st), "kicp_frame_free_space");
    return st;
}

// the two clouds of the last frame, built in one pass each from the library's pinned staging
KinematicICP::Vector3dVectorTuple KinematicICP::StagedClouds() {
    const double *frame_xyz = nullptr, *source_xyz = nullptr;
    int64_t n_frame = 0, n_source = 0;
    kicp::check(kicp_frame_clouds(kicp::default_context(), &frame_xyz, &n_frame, &source_xyz, &n_source), "kicp_frame_clouds");
    const auto *fb = reinterpret_cast<const Eigen::Vector3d *>(frame_xyz);
    const auto *sb = reinterpret_cast<const Eigen::Vector3d *>(source_xyz);
    return {Vector3dVector(fb, fb + n_frame), Vector3dVector(sb, sb + n_source)};
}

// RegisterStagedFrame + EigenToPointCloud2 of both clouds: the records are encoded on the device inside the frame and copied once
std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> KinematicICP::RegisterStagedFramePointCloud2(const Sophus::SE3d &lidar_to_base,
                                                                                                     const Sophus::SE3d &relative_odometry) {
    RegisterOnDevice(nullptr, &lidar_to_base, 1, false, relative_odometry, KICP_STAGE_F32);
    return StagedCloudsPointCloud2();
}

// the two clouds of the last frame as the float32 records the device encoded
std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> KinematicICP::StagedCloudsPointCloud2() {
    const float *frame_xyz = nullptr, *source_xyz = nullptr;
    int64_t n_frame = 0, n_source = 0;
    kicp::check(kicp_frame_clouds_f32(kicp::default_context(), &frame_xyz, &n_frame, &source_xyz, &n_source), "kicp_frame_clouds_f32");
    return {kicp::PointCloud2Data::from_xyz(frame_xyz, (size_t)n_frame), kicp::PointCloud2Data::from_xyz(source_xyz, (size_t)n_source)};
}

// EigenToPointCloud2(LocalMap()): one device-to-host copy straight into the message's data
kicp::PointCloud2Data KinematicICP::LocalMapPointCloud2() const {
    int64_t n = 0;
    kicp::check(kicp_map_num_points(local_map_.handle_, &n), "kicp_map_num_points");
    kicp::PointCloud2Data m;
    m.resize((size_t)n);
    if (n > 0)
        kicp::check(kicp_map_pointcloud_f32(local_map_.handle_, reinterpret_cast<float *>(m.data.data()), n, &n), "kicp_map_pointcloud_f32");
    return m;
}

// EigenToPointCloud2(LocalMap()) kept up to date in the map's page-locked buffer: only the changed records cross PCIe
std::tuple<kicp::PointCloud2View, kicp_map_live_stats> KinematicICP::LocalMapPointCloud2Live() {
    const float *records = nullptr;
    int64_t n = 0;
    kicp_map_live_stats stats{};
    kicp::check(kicp_map_pointcloud_f32_live(local_map_.handle_, &records, &n, &stats), "kicp_map_pointcloud_f32_live");
    kicp::PointCloud2View v;
    v.data = reinterpret_cast<const uint8_t *>(records);
    v.width = static_cast<uint32_t>(n), v.height = 1, v.point_step = 12;
    v.fields = {{"x", 0, kicp::PF_FLOAT32, 1}, {"y", 4, kicp::PF_FLOAT32, 1}, {"z", 8, kicp::PF_FLOAT32, 1}};
    return {v, stats};
}

void KinematicICP::RegisterOnDevice(const kicp_frame_input *input, const Sophus::SE3d *lidar_to_base, size_t k, bool sensors,
                                    const Sophus::SE3d &relative_odometry, int32_t stage_clouds,
                                    const std::vector<kicp::OdometrySample> *samples) {
    // deskew in the lidar frame (of every sensor)
    std::vector<std::array<double, 7>> motions(k), l2bs(k);
    for (size_t i = 0; i < k; ++i) {
        const Sophus::SE3d relative_odometry_in_lidar = lidar_to_base[i].inverse() * relative_odometry * lidar_to_base[i];
        kicp::to_pose7(relative_odometry_in_lidar, motions[i].data());
        kicp::to_pose7(lidar_to_base[i], l2bs[i].data());
    }
    const double(*motion7)[7] = reinterpret_cast<const double(*)[7]>(motions.data());
    const double(*l2b7)[7] = reinterpret_cast<const double(*)[7]>(l2bs.data());
    const double *motion = k ? motion7[0] : nullptr, *l2b = k ? l2b7[0] : nullptr;
    double last[7], odom[7], out[7];
    kicp::to_pose7(last_pose_, last);
    kicp::to_pose7(relative_odometry, odom);
    kicp_frame_params fp;
    fp.max_range = preprocessor_.max_range_, fp.min_range = preprocessor_.min_range_, fp.deskew = preprocessor_.deskew_ ? 1 : 0;
    fp.voxel_size = config_.voxel_size;
    fp.reg.max_num_iterations = registration_.max_num_iterations_;
    fp.reg.use_adaptive_odometry_regularization = registration_.use_adaptive_odometry_regularization_ ? 1 : 0;
    fp.reg.convergence_criterion = registration_.convergence_criterion_;
    fp.reg.fixed_regularization = registration_.fixed_regularization_;
    const double tau = correspondence_threshold_.ComputeThreshold();
    fp.stage_clouds = stage_clouds;
    // the segments of every sensor (built before anything is registered: a throw leaves the staged frame staged)
    std::vector<std::vector<kicp_deskew_segment>> segments(samples ? k : 0);
    std::vector<const kicp_deskew_segment *> seg_ptr(segments.size());
    std::vector<int32_t> seg_n(segments.size());
    for (size_t i = 0; i < segments.size(); ++i) {
        segments[i] = kicp::deskew_segments(*samples, lidar_to_base[i], staged_sweep_, staged_window_);
        seg_ptr[i] = segments[i].data(), seg_n[i] = static_cast<int32_t>(segments[i].size());
    }
    if (samples && sensors)
        kicp::check(kicp_register_staged_sensors_segments(local_map_.handle_, static_cast<int32_t>(k), seg_n.data(), seg_ptr.data(), l2b7, last,
                                                          odom, tau, &fp, out, nullptr, 0, nullptr, nullptr, 0, nullptr, nullptr),
                    "kicp_register_staged_sensors_segments");
    else if (samples)
        kicp::check(kicp_register_staged_frame_segments(local_map_.handle_, seg_n[0], seg_ptr[0], l2b, last, odom, tau, &fp, out, nullptr, 0,
                                                        nullptr, nullptr, 0, nullptr, nullptr),
                    "kicp_register_staged_frame_segments");
    else if (input)
        kicp::check(kicp_register_frame(local_map_.handle_, input, motion, l2b, last, odom, tau, &fp, out, nullptr, 0, nullptr, nullptr, 0,
                                        nullptr, nullptr),
                    "kicp_register_frame");
    else if (sensors)
        kicp::check(kicp_register_staged_sensors(local_map_.handle_, static_cast<int32_t>(k), motion7, l2b7, last, odom, tau, &fp, out, nullptr,
                                                 0, nullptr, nullptr, 0, nullptr, nullptr),
                    "kicp_register_staged_sensors");
    else
        kicp::check(kicp_register_staged_frame(local_map_.handle_, motion, l2b, last, odom, tau, &fp, out, nullptr, 0, nullptr, nullptr, 0,
                                               nullptr, nullptr),
                    "kicp_register_staged_frame");
    const Sophus::SE3d new_pose = kicp::from_pose7(out);
    const Sophus::SE3d odometry_error = (last_pose_ * relative_odometry).inverse() * new_pose;
    correspondence_threshold_.UpdateOdometryError(odometry_error);
    last_pose_ = new_pose;
}

KinematicICP::Vector3dVectorTuple KinematicICP::RegisterFrame(const std::vector<Eigen::Vector3d> &frame, const std::vector<double> &timestamps,
                                                              const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry) {
    kicp_frame_input input{};
    input.data = kicp::xyz(frame), input.n = (int64_t)frame.size(), input.dtype = KICP_DTYPE_F64, input.point_step = 0;
    input.stamps = timestamps.empty() ? nullptr : timestamps.data(), input.n_stamps = (int64_t)timestamps.size();
    return RegisterFrame(input, lidar_to_base, relative_odometry);
}
}  // namespace pipeline
#endif
}  // namespace kinematic_icp
