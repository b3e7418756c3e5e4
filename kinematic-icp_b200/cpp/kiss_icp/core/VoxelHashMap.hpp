// kiss_icp::VoxelHashMap — same name, namespace, constructor and methods as KISS-ICP v1.2.0's
// cpp/kiss_icp/core/VoxelHashMap.hpp (the header the reference includes at registration/Registration.hpp:26 and
// pipeline/KinematicICP.hpp:29), with the storage and every operation in HBM behind include/kicp.h.
// The robin_map member `map_` of the original has no counterpart (no code of the reference reads it).
#pragma once
#include <Eigen/Core>
#include <sophus/se3.hpp>
#include <algorithm>
#include <array>
#include <tuple>
#include <vector>

#include "kicp/runtime.hpp"
#include "kiss_icp/core/VoxelUtils.hpp"

namespace kicp {
// kicp_map_pose_search's parameters (x, y, yaw half extents and steps of level 0, the gate, levels, keep) and one returned hypothesis
using PoseSearchParams = kicp_pose_search_params;
struct PoseHypothesis {
    Sophus::SE3d pose;                // prior * Delta
    Eigen::Vector3d offset;           // x, y, yaw of Delta
    std::array<int32_t, 3> lattice;   // ix, iy, ipsi in units of step / 2^(levels-1)
    int level;
    int64_t n_inliers;
    double fitness, inlier_rmse, sum_sq;
};
// kicp_map_align_planar's parameters (gate, convergence, max_iterations) and one start's result
using PlanarAlignParams = kicp_planar_align_params;
struct PlanarAlignment {
    Sophus::SE3d pose;  // the returned pose
    int status;         // KICP_ALIGN_*
    int iterations;
    double last_step;
    int64_t n_inliers;  // the correspondence report at `pose`
    double fitness, inlier_rmse, sum_sq;
    std::array<double, 6> jtj;  // J^T J over (x, y, yaw): 00, 01, 02, 11, 12, 22
    std::array<double, 3> jtr;
};
}  // namespace kicp

namespace kiss_icp {
struct VoxelHashMap {
    explicit VoxelHashMap(double voxel_size, double max_distance, unsigned int max_points_per_voxel)
        : voxel_size_(voxel_size), max_distance_(max_distance), max_points_per_voxel_(max_points_per_voxel) {
        kicp::check(kicp_map_create(kicp::default_context(), voxel_size, max_distance, max_points_per_voxel, &handle_),
                    "kicp_map_create");
    }
    ~VoxelHashMap() { kicp_map_destroy(handle_); }
    VoxelHashMap(const VoxelHashMap &) = delete;
    VoxelHashMap &operator=(const VoxelHashMap &) = delete;
    VoxelHashMap(VoxelHashMap &&o) noexcept
        : voxel_size_(o.voxel_size_), max_distance_(o.max_distance_), max_points_per_voxel_(o.max_points_per_voxel_), handle_(o.handle_) {
        o.handle_ = nullptr;
    }

    inline void Clear() { kicp::check(kicp_map_clear(handle_), "kicp_map_clear"); }
    inline bool Empty() const {
        int32_t e = 1;
        kicp::check(kicp_map_empty(handle_, &e), "kicp_map_empty");
        return e != 0;
    }
    void Update(const std::vector<Eigen::Vector3d> &points, const Eigen::Vector3d &origin) {
        kicp::check(kicp_map_update(handle_, kicp::xyz(points), (int64_t)points.size(), origin.data()), "kicp_map_update");
    }
    void Update(const std::vector<Eigen::Vector3d> &points, const Sophus::SE3d &pose) {
        double p[7];
        kicp::to_pose7(pose, p);
        kicp::check(kicp_map_update_pose(handle_, kicp::xyz(points), (int64_t)points.size(), p), "kicp_map_update_pose");
    }
    // Free-space clearing (kicp_map_clear_free_space): every point of `points` (frame F) is a ray from pose * sensor_origin to
    // pose * p; live voxels that at least min_misses rays pass through and in which no ray ends leave the map.  Throws on an error.
    kicp_free_space_stats ClearFreeSpace(const std::vector<Eigen::Vector3d> &points, const Sophus::SE3d &pose,
                                         const Eigen::Vector3d &sensor_origin, int32_t min_misses = 2, double end_margin = 0.5) {
        double p[7];
        kicp::to_pose7(pose, p);
        const kicp_free_space_params params{end_margin, min_misses};
        kicp_free_space_stats st{};
        kicp::check(kicp_map_clear_free_space(handle_, kicp::xyz(points), (int64_t)points.size(), p, sensor_origin.data(), &params, &st),
                    "kicp_map_clear_free_space");
        return st;
    }
    // the defaults of occupancy evidence (README, "Clearing free space"; the Python OCCUPANCY_* constants)
    static constexpr kicp_occupancy_params kDefaultOccupancy{3, 1, 1, 3};
    // Occupancy evidence of the clearing calls (kicp_map_set_occupancy): a live voxel keeps an integer evidence across calls and is
    // cleared when it reaches 0; nullptr turns it off.  A setting of the map: Clear() (and so KinematicICP::SetPose) keeps it.  The
    // pipeline reaches it through KinematicICP::VoxelMap().  Throws on an error (a field out of range is named).
    void SetOccupancy(const kicp_occupancy_params *params) {
        kicp::check(kicp_map_set_occupancy(handle_, params), "kicp_map_set_occupancy");
    }
    // the evidence of every voxel in the block order of kicp_map_export_voxels (prior first); throws when occupancy is off
    std::vector<int32_t> Occupancy() const {
        int64_t n = 0;
        kicp::check(kicp_map_num_voxels(handle_, &n), "kicp_map_num_voxels");
        std::vector<int32_t> out(static_cast<size_t>(n));
        kicp::check(kicp_map_export_occupancy(handle_, out.data(), n, &n), "kicp_map_export_occupancy");
        out.resize(static_cast<size_t>(n));
        return out;
    }
    void AddPoints(const std::vector<Eigen::Vector3d> &points) {
        kicp::check(kicp_map_add_points(handle_, kicp::xyz(points), (int64_t)points.size()), "kicp_map_add_points");
    }
    void RemovePointsFarFromLocation(const Eigen::Vector3d &origin) {
        kicp::check(kicp_map_remove_far(handle_, origin.data()), "kicp_map_remove_far");
    }
    std::vector<Eigen::Vector3d> Pointcloud() const {
        int64_t n = 0;
        kicp::check(kicp_map_num_points(handle_, &n), "kicp_map_num_points");
        std::vector<Eigen::Vector3d> out(static_cast<size_t>(n));
        if (n > 0) kicp::check(kicp_map_pointcloud(handle_, out.front().data(), n, &n), "kicp_map_pointcloud");
        return out;
    }
    // A frozen prior inside the map (kicp_map_freeze): every voxel now in the map becomes read-only and is never evicted; later
    // Updates build the live layer beside it.  Clear() (and so KinematicICP::SetPose) and load_voxels remove the prior too.
    void Freeze() { kicp::check(kicp_map_freeze(handle_), "kicp_map_freeze"); }
    void Thaw() { kicp::check(kicp_map_thaw(handle_), "kicp_map_thaw"); }
    int64_t PriorVoxels() const {
        int64_t v = 0, n = 0;
        kicp::check(kicp_map_prior_size(handle_, &v, &n), "kicp_map_prior_size");
        return v;
    }
    int64_t PriorPoints() const {
        int64_t v = 0, n = 0;
        kicp::check(kicp_map_prior_size(handle_, &v, &n), "kicp_map_prior_size");
        return n;
    }
    // Pointcloud() of one layer (KICP_MAP_LAYER_ALL, _PRIOR or _LIVE): ALL is PRIOR followed by LIVE
    std::vector<Eigen::Vector3d> Pointcloud(int32_t layer) const {
        int64_t n = 0, total = 0;
        kicp::check(kicp_map_num_points(handle_, &total), "kicp_map_num_points");
        const int64_t prior = PriorPoints();
        n = layer == KICP_MAP_LAYER_PRIOR ? prior : layer == KICP_MAP_LAYER_LIVE ? total - prior : total;
        std::vector<Eigen::Vector3d> out(static_cast<size_t>(n));
        if (n == 0) kicp::check(kicp_map_pointcloud_layer(handle_, layer, KICP_DTYPE_F64, nullptr, 0, &n), "kicp_map_pointcloud_layer");
        if (n > 0) kicp::check(kicp_map_pointcloud_layer(handle_, layer, KICP_DTYPE_F64, out.front().data(), n, &n), "kicp_map_pointcloud_layer");
        return out;
    }
    std::tuple<Eigen::Vector3d, double> GetClosestNeighbor(const Eigen::Vector3d &query) const {
        Eigen::Vector3d p;
        double d = 0.0;
        kicp::check(kicp_map_nearest(handle_, query.data(), 1, p.data(), &d), "kicp_map_nearest");
        return std::make_tuple(p, d);
    }

    // Where `points` (robot base frame) fit the map around `prior`: the best hypotheses of kicp_map_pose_search, best first.  A node
    // relocalises with `kicp.pose() = hyps[0].pose`, which keeps the map (SetPose clears it).
    std::vector<kicp::PoseHypothesis> SearchPose(const std::vector<Eigen::Vector3d> &points, const Sophus::SE3d &prior,
                                                 const kicp::PoseSearchParams &params) const {
        double p[7];
        kicp::to_pose7(prior, p);
        std::vector<kicp_pose_hypothesis> h(params.keep > 0 ? (size_t)params.keep : 1);
        int32_t n_out = 0;
        int64_t n_scored = 0;
        kicp::check(kicp_map_pose_search(handle_, kicp::xyz(points), (int64_t)points.size(), p, &params, h.data(), (int32_t)h.size(),
                                         &n_out, &n_scored),
                    "kicp_map_pose_search");
        std::vector<kicp::PoseHypothesis> out;
        for (int32_t i = 0; i < n_out; ++i) {
            const kicp_pose_hypothesis &c = h[i];
            out.push_back(kicp::PoseHypothesis{kicp::from_pose7(c.pose), Eigen::Vector3d(c.offset[0], c.offset[1], c.offset[2]),
                                               {c.lattice[0], c.lattice[1], c.lattice[2]}, c.level, c.n_inliers, c.fitness,
                                               c.inlier_rmse, c.sum_sq});
        }
        return out;
    }

    // Gauss-Newton in (x, y, yaw) of `points` (robot base frame) against the map from each of `initial` (1 to 64 starts, each aligned
    // on its own; kicp_map_align_planar), one result per start in input order.  After SearchPose: align its hypotheses' poses and
    // pick the best result by the caller's rule.
    std::vector<kicp::PlanarAlignment> AlignPlanar(const std::vector<Eigen::Vector3d> &points, const std::vector<Sophus::SE3d> &initial,
                                                   const kicp::PlanarAlignParams &params) const {
        std::vector<double> starts(7 * initial.size());
        for (size_t k = 0; k < initial.size(); ++k) kicp::to_pose7(initial[k], &starts[7 * k]);
        std::vector<kicp_planar_alignment> r(std::max<size_t>(initial.size(), 1));
        kicp::check(kicp_map_align_planar(handle_, kicp::xyz(points), (int64_t)points.size(), starts.data(), (int32_t)initial.size(),
                                          &params, r.data()),
                    "kicp_map_align_planar");
        std::vector<kicp::PlanarAlignment> out;
        for (size_t k = 0; k < initial.size(); ++k) {
            const kicp_planar_alignment &c = r[k];
            kicp::PlanarAlignment a{kicp::from_pose7(c.pose), c.status, c.iterations, c.last_step, c.n_inliers, c.fitness,
                                    c.inlier_rmse, c.sum_sq, {}, {}};
            for (int j = 0; j < 6; ++j) a.jtj[j] = c.jtj[j];
            for (int j = 0; j < 3; ++j) a.jtr[j] = c.jtr[j];
            out.push_back(a);
        }
        return out;
    }

    double voxel_size_;
    double max_distance_;
    unsigned int max_points_per_voxel_;
    kicp_map *handle_ = nullptr;  // the HBM-resident map (replaces tsl::robin_map<Voxel, std::vector<Eigen::Vector3d>> map_)
};
}  // namespace kiss_icp
