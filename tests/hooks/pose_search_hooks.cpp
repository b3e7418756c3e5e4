// extern "C" test hooks over the pose search of the C++ facade: kiss_icp::VoxelHashMap::SearchPose on a map of the process-wide
// context, its handle for the C call on the same map, and relocalising a pipeline made by kfac_pipeline_create (facade_hooks.cpp)
// through its mutable pose().  Test infrastructure: built as tests/hooks/_build/libkicp_pose_search_hooks.so by
// kinematic-icp_b200/cpp/Makefile, linked AGAINST the product libraries, never into them.
#include <cstdint>
#include <vector>

#include "kinematic_icp/pipeline/KinematicICP.hpp"
#include "kiss_icp/core/VoxelHashMap.hpp"

namespace {
std::vector<Eigen::Vector3d> to_eigen(const double *xyz, int64_t n) {
    std::vector<Eigen::Vector3d> v((size_t)n);
    for (int64_t i = 0; i < n; ++i) v[i] = Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    return v;
}
// SearchPose's hypotheses written back as the C records (pose through to_pose7); their number, or -1 when it throws
int32_t search(const kiss_icp::VoxelHashMap &m, const double *xyz, int64_t n, const double *prior7, const kicp_pose_search_params *p,
               kicp_pose_hypothesis *out) {
    try {
        const auto hyps = m.SearchPose(to_eigen(xyz, n), kicp::from_pose7(prior7), *p);
        for (size_t i = 0; i < hyps.size(); ++i) {
            const kicp::PoseHypothesis &h = hyps[i];
            kicp_pose_hypothesis &o = out[i];
            kicp::to_pose7(h.pose, o.pose);
            for (int a = 0; a < 3; ++a) o.offset[a] = h.offset[a], o.lattice[a] = h.lattice[a];
            o.level = h.level, o.n_inliers = h.n_inliers, o.fitness = h.fitness, o.inlier_rmse = h.inlier_rmse, o.sum_sq = h.sum_sq;
        }
        return (int32_t)hyps.size();
    } catch (const std::exception &) {
        return -1;
    }
}
}  // namespace

extern "C" {
void *kfps_map_create(double voxel_size, double max_distance, unsigned max_points_per_voxel) {
    return new kiss_icp::VoxelHashMap(voxel_size, max_distance, max_points_per_voxel);
}
void kfps_map_destroy(void *h) { delete static_cast<kiss_icp::VoxelHashMap *>(h); }
void kfps_map_add_points(void *h, const double *xyz, int64_t n) { static_cast<kiss_icp::VoxelHashMap *>(h)->AddPoints(to_eigen(xyz, n)); }
// the C handle behind the facade map (for kicp_map_pose_search on the same map)
void *kfps_map_handle(void *h) { return static_cast<kiss_icp::VoxelHashMap *>(h)->handle_; }
int32_t kfps_map_search_pose(void *h, const double *xyz, int64_t n, const double *prior7, const kicp_pose_search_params *p,
                             kicp_pose_hypothesis *out) {
    return search(*static_cast<kiss_icp::VoxelHashMap *>(h), xyz, n, prior7, p, out);
}
// SearchPose on a pipeline's local map (KinematicICP::VoxelMap())
int32_t kfps_pipeline_search_pose(void *h, const double *xyz, int64_t n, const double *prior7, const kicp_pose_search_params *p,
                                  kicp_pose_hypothesis *out) {
    return search(static_cast<kinematic_icp::pipeline::KinematicICP *>(h)->VoxelMap(), xyz, n, prior7, p, out);
}
// relocalise: kicp.pose() = pose (the map stays, unlike SetPose)
void kfps_pipeline_assign_pose(void *h, const double *pose7) {
    static_cast<kinematic_icp::pipeline::KinematicICP *>(h)->pose() = kicp::from_pose7(pose7);
}
void kfps_pipeline_pose(void *h, double *pose7) { kicp::to_pose7(static_cast<kinematic_icp::pipeline::KinematicICP *>(h)->pose(), pose7); }
}
