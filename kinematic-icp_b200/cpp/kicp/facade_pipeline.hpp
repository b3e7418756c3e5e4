// kinematic_icp::pipeline::{Config, KinematicICP} of this repo, reached through a forwarding header at the reference's
// include path kinematic_icp/pipeline/KinematicICP.hpp.  The public surface (field names and defaults of Config, the
// constructor, RegisterFrame, SetPose, LocalMap, VoxelMap, pose) is the one ros/src/kinematic_icp_ros/server/
// LidarOdometryServer.cpp:72-105,205-206 uses (reference: pipeline/KinematicICP.hpp:38-111); RegisterFrame itself is one
// device-resident call, kicp_register_frame (include/kicp.h).  Definitions: facade.cpp.
// Both down-samples of RegisterFrame emit the order of first occurrence.  With KICP_DOWNSAMPLE_ORDER=1 in the environment when the
// process-wide default context is created (kicp/runtime.hpp), they emit the iteration order of KISS-ICP v1.2.0's robin_map instead
// (context option "downsample_order", include/kicp.h; unpinned like the test oracle's mode 1); a value other than 0 or 1 throws.
// With KICP_CORRESPONDENCES=1 in the environment at that moment (or after KinematicICP::SetCorrespondences(true)), every frame also
// reports its correspondences at the returned pose (context option "correspondences"), read with LastCorrespondenceStats; 0 leaves the
// option off, any other value throws.
#pragma once
#include <Eigen/Core>
#include <cmath>
#include <sophus/se3.hpp>
#include <tuple>
#include <vector>

#include "kicp/deskew_segments.hpp"
#include "kicp/facade_core.hpp"
#include "kicp/laser_scan.hpp"
#include "kicp/pointcloud2.hpp"
#include "kicp/sensor_frame.hpp"
#include "kiss_icp/core/Preprocessing.hpp"
#include "kiss_icp/core/VoxelHashMap.hpp"

namespace kinematic_icp::pipeline {

// Field order, names and defaults exactly as pipeline/KinematicICP.hpp:38-60 — callers aggregate-initialise this struct
// and assign its fields by name (ros/src/kinematic_icp_ros/server/LidarOdometryServer.cpp:72-97); the layout is part of
// the interface (tests/test_facade_layout_cpu.py compiles one TU against both headers).
struct Config {
    // Preprocessing
    double max_range = 100.0;
    double min_range = 0.0;
    // Mapping parameters
    double voxel_size = 1.0;
    unsigned int max_points_per_voxel = 20;
    // Derived parameter, will be computed from other parts of the configuration
    constexpr double map_resolution() const { return voxel_size / std::sqrt(max_points_per_voxel); }
    // Correspondence threshold parameters
    bool use_adaptive_threshold = true;
    double fixed_threshold = 1.0;  // <-- Ignored if use_adaptive_threshold = true

    // Registration Parameters
    int max_num_iterations = 10;
    double convergence_criterion = 0.001;
    int max_num_threads = 1;  // TBB width in the reference; accepted and ignored on the device
    bool use_adaptive_odometry_regularization = true;
    double fixed_regularization = 0.0;  // <-- Ignored if use_adaptive_odometry_regularization = true

    // Motion compensation
    bool deskew = false;
};

class KinematicICP {
public:
    using Vector3dVector = std::vector<Eigen::Vector3d>;
    using Vector3dVectorTuple = std::tuple<Vector3dVector, Vector3dVector>;

    explicit KinematicICP(const Config &config);

    // {preprocessed frame in the base frame, registration source}; advances pose() and the local map
    Vector3dVectorTuple RegisterFrame(const std::vector<Eigen::Vector3d> &frame,
                                      const std::vector<double> &timestamps,
                                      const Sophus::SE3d &lidar_to_base,
                                      const Sophus::SE3d &relative_odometry);
    // Extension (not in the reference): the same frame straight from a PointCloud2-shaped buffer (float32 or float64 fields
    // at a byte stride, include/kicp.h kicp_frame_input), skipping the host-side widening of RosUtils.cpp:30-39.
    Vector3dVectorTuple RegisterFrame(const kicp_frame_input &input, const Sophus::SE3d &lidar_to_base,
                                      const Sophus::SE3d &relative_odometry);
    // Extension (not in the reference): RegisterFrame in two steps for an online node, which needs the sweep's interval before
    // it can look up the wheel odometry (LidarOdometryServer.cpp:186-210).  StageFrame uploads the message's records once,
    // decodes x/y/z and the time field (kicp::stamp_field) on the device and returns the interval process_timestamps would
    // return for the same message (kicp_frame_stage, include/kicp.h).  RegisterStagedFrame then registers that frame with the
    // odometry of the interval: same results as RegisterFrame(make_frame_input(msg) + extract_timestamps(msg), ...).  A staged
    // frame is consumed by one RegisterStagedFrame and discarded by any other frame call on the process-wide context.
    kicp::SweepTiming StageFrame(const kicp::PointCloud2View &msg, double header_stamp, double &last_processed_stamp);
    // Extension (not in the reference): StageFrame for a 2D LiDAR (the reference's use_2d_lidar).  The scan is staged as the frame
    // laser_geometry's projectLaser(scan, cloud, -1.0, channel_option::Timestamp) makes of it, with its per-beam stamps, and the
    // ranges cross PCIe once (kicp_frame_stage_laser_scan, include/kicp.h).  The interval is process_timestamps' for that cloud;
    // RegisterStagedFrame / RegisterStagedFramePointCloud2 then register it unchanged.
    kicp::SweepTiming StageLaserScan(const kicp::LaserScanView &scan, double header_stamp, double &last_processed_stamp);
    // Extension (not in the reference): StageFrame / StageLaserScan for a message whose msg.data / scan.ranges point into device
    // memory of the process-wide context's device (a GPU producer: a ray-caster, a device-side decoder or transport).  The records
    // are read in place (kicp_frame_stage_device / kicp_frame_stage_laser_scan_device, include/kicp.h); field lookup, interval and
    // staging rules are StageFrame's / StageLaserScan's, and RegisterStagedFrame* register the frame unchanged.  A producer on its
    // own stream orders itself first with kicp_ctx_wait_stream(kicp::default_context(), stream).
    kicp::SweepTiming StageDeviceFrame(const kicp::PointCloud2View &msg, double header_stamp, double &last_processed_stamp);
    kicp::SweepTiming StageDeviceLaserScan(const kicp::LaserScanView &scan, double header_stamp, double &last_processed_stamp);
    Vector3dVectorTuple RegisterStagedFrame(const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry);
    // Extension (not in the reference): a frame of several LiDARs (kicp_frame_stage_sensors / kicp_register_staged_sensors,
    // include/kicp.h).  StageSensors stages all of them with one host synchronisation and returns the frame's interval: it begins at
    // last_processed_stamp and ends at the latest of the sensors' ends, each by StageFrame's rule applied to that sensor's header and
    // stamps (on its own clock); last_processed_stamp becomes that end.  RegisterStagedSensors registers the frame with one extrinsic
    // per staged sensor: sensor k is de-skewed in its own frame with lidar_to_base[k]^-1 * relative_odometry * lidar_to_base[k]
    // (RegisterFrame's expression) over the common window and moved to base by lidar_to_base[k]; the rest is RegisterStagedFrame's.
    // One sensor with offset 0 gives what StageFrame / StageLaserScan + RegisterStagedFrame give.  A frame staged by StageFrame or
    // StageLaserScan is one sensor to RegisterStagedSensors; RegisterStagedFrame refuses a frame of several sensors.
    kicp::SweepTiming StageSensors(const std::vector<kicp::SensorFrame> &sensors, double &last_processed_stamp);
    Vector3dVectorTuple RegisterStagedSensors(const std::vector<Sophus::SE3d> &lidar_to_base, const Sophus::SE3d &relative_odometry);
    std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> RegisterStagedSensorsPointCloud2(const std::vector<Sophus::SE3d> &lidar_to_base,
                                                                                             const Sophus::SE3d &relative_odometry);
    // Extension (not in the reference): the staged frame de-skewed along the wheel odometry sampled during the sweep instead of one
    // motion (kicp_register_staged_frame_segments / kicp_register_staged_sensors_segments, include/kicp.h).  `samples` are base poses in
    // the odometry frame on the odometry clock, covering the SweepTiming the last Stage* call returned (a node looks them up in tf
    // between begin and end); each sensor's segments are kicp::deskew_segments(samples, lidar_to_base[k], sweep, window) with that
    // call's sweep and staged window (kicp/deskew_segments.hpp).  relative_odometry keeps its role in the motion model and the
    // threshold.  Samples {(begin, identity), (end, relative_odometry)} give bit for bit what the overloads without samples give.
    // Throws std::invalid_argument (and leaves the staged frame staged) when the samples do not cover the sweep.
    Vector3dVectorTuple RegisterStagedFrame(const Sophus::SE3d &lidar_to_base, const Sophus::SE3d &relative_odometry,
                                            const std::vector<kicp::OdometrySample> &samples);
    std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> RegisterStagedFramePointCloud2(const Sophus::SE3d &lidar_to_base,
                                                                                           const Sophus::SE3d &relative_odometry,
                                                                                           const std::vector<kicp::OdometrySample> &samples);
    Vector3dVectorTuple RegisterStagedSensors(const std::vector<Sophus::SE3d> &lidar_to_base, const Sophus::SE3d &relative_odometry,
                                              const std::vector<kicp::OdometrySample> &samples);
    std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> RegisterStagedSensorsPointCloud2(const std::vector<Sophus::SE3d> &lidar_to_base,
                                                                                             const Sophus::SE3d &relative_odometry,
                                                                                             const std::vector<kicp::OdometrySample> &samples);

    // Extension (not in the reference): the publish step of an online node (LidarOdometryServer::PublishClouds,
    // LidarOdometryServer.cpp:240-263) without its host loops.  RegisterStagedFramePointCloud2 has exactly RegisterStagedFrame's
    // effects on the pose, the threshold model and the map, and returns {frame, keypoints} as the records EigenToPointCloud2 builds
    // from RegisterStagedFrame's two clouds; LocalMapPointCloud2 is EigenToPointCloud2(LocalMap()).  Both narrow on the device
    // (static_cast<float> as on x86-64, NaN bits included) and move 12 bytes per point over PCIe (kicp_frame_clouds_f32,
    // kicp_map_pointcloud_f32).
    std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> RegisterStagedFramePointCloud2(const Sophus::SE3d &lidar_to_base,
                                                                                           const Sophus::SE3d &relative_odometry);
    kicp::PointCloud2Data LocalMapPointCloud2() const;
    // Extension (not in the reference): LocalMapPointCloud2 for a node that publishes the local map every frame.  The map keeps the
    // records in a page-locked buffer of its own and each call writes into it only the records that changed since the previous call
    // (kicp_map_pointcloud_f32_live): a few percent of the map per frame instead of all of it.  Returns a view over that buffer
    // (width n, x/y/z FLOAT32 at 0/4/8, point_step 12, the records in an unspecified order) and what the call wrote.  The view is valid
    // until the next call or the map's destruction.  A node keeps one PointCloud2 message and refills its data from the view before
    // each publication, or, with a zero-copy publisher, publishes the view's bytes directly.
    std::tuple<kicp::PointCloud2View, kicp_map_live_stats> LocalMapPointCloud2Live();

    // Extension (not in the reference): how well the last frame registered.  With the report switched on, every RegisterFrame /
    // RegisterStaged* call also evaluates its registration source at the returned pose against the local map as it was before the
    // frame's update (context option "correspondences", include/kicp.h: two more kernel launches, no more host synchronisations).
    // LastCorrespondenceStats returns kicp_frame_correspondences of the process-wide context: the last frame registered on it by any
    // KinematicICP, all zero when the report was off or that frame failed.  Fitness, inlier RMSE, and J^T J / J^T r of
    // ComputePerturbation at the returned pose, from which a node may build a covariance (INTEGRATION.md §10; the facade imposes
    // none).  SetCorrespondences switches the report for the process-wide context, as KICP_CORRESPONDENCES does at its creation.
    kicp_corr_stats LastCorrespondenceStats() const;
    static void SetCorrespondences(bool on);
    // Extension: the map-update policy of the process-wide context (kicp_ctx_set_map_update): ALWAYS (the reference's Update after every
    // frame), NEVER (register against the local map as it is, e.g. one restored with VoxelMap().load_voxels) or GATED (update only
    // when the frame's correspondence report passes the thresholds).  LastMapUpdate returns kicp_frame_map_update of that context: the
    // KICP_FRAME_UPDATE_* outcome of the last frame registered on it by any KinematicICP.  Both throw on an error the C call returns.
    static void SetMapUpdate(const kicp_map_update_policy &policy);
    int32_t LastMapUpdate() const;
    // Extension: free-space clearing in the frame path of the process-wide context (kicp_ctx_set_free_space; min_misses 0 turns it
    // off): after every applied Update the frame's down-sampled points clear the live voxels their rays pass through.  LastFreeSpace
    // returns kicp_frame_free_space of that context.  Both throw on an error the C call returns.
    static void SetFreeSpace(int32_t min_misses = 2, double end_margin = 0.5);
    kicp_free_space_stats LastFreeSpace() const;

    void SetPose(const Sophus::SE3d &pose);  // also clears the map and the threshold statistics (KinematicICP.hpp:85-89)

    std::vector<Eigen::Vector3d> LocalMap() const { return local_map_.Pointcloud(); };

    const kiss_icp::VoxelHashMap &VoxelMap() const { return local_map_; };
    kiss_icp::VoxelHashMap &VoxelMap() { return local_map_; };

    const Sophus::SE3d &pose() const { return last_pose_; }
    Sophus::SE3d &pose() { return last_pose_; }

protected:  // same members, names and order as pipeline/KinematicICP.hpp:101-108 (subclasses reach them by name)
    Sophus::SE3d last_pose_;
    // Kinematic module
    KinematicRegistration registration_;
    CorrespondenceThreshold correspondence_threshold_;
    Config config_;
    // KISS-ICP pipeline modules
    kiss_icp::Preprocessor preprocessor_;
    kiss_icp::VoxelHashMap local_map_;  // HBM-resident

private:
    // every RegisterFrame extension: `input` null = the staged frame, registered per sensor (`sensors`, k extrinsics) or as one frame
    // (lidar_to_base[0]); `stage_clouds` = kicp_frame_params.stage_clouds (the caller reads the clouds it asked for with
    // kicp_frame_clouds / kicp_frame_clouds_f32); `samples` (optional): the staged frame de-skewed by the segments built from them
    void RegisterOnDevice(const kicp_frame_input *input, const Sophus::SE3d *lidar_to_base, size_t k, bool sensors,
                          const Sophus::SE3d &relative_odometry, int32_t stage_clouds,
                          const std::vector<kicp::OdometrySample> *samples = nullptr);
    static std::tuple<kicp::PointCloud2Data, kicp::PointCloud2Data> StagedCloudsPointCloud2();
    static Vector3dVectorTuple StagedClouds();
    // the SweepTiming and the staged window {T0, T1} of the last Stage* call (the segments' clock correspondence)
    kicp::SweepTiming staged_sweep_;
    double staged_window_[2] = {0.0, 0.0};
};

}  // namespace kinematic_icp::pipeline
