// extern "C" test hooks over the planar alignment of the C++ facade: kiss_icp::VoxelHashMap::AlignPlanar on a map of the
// process-wide context, and its handle for the C call on the same map.  Test infrastructure: built as
// tests/hooks/_build/libkicp_align_planar_hooks.so by kinematic-icp_b200/cpp/Makefile, linked AGAINST the product libraries, never
// into them.
#include <cstdint>
#include <vector>

#include "kiss_icp/core/VoxelHashMap.hpp"

extern "C" {
void *kfal_map_create(double voxel_size, double max_distance, unsigned max_points_per_voxel) {
    return new kiss_icp::VoxelHashMap(voxel_size, max_distance, max_points_per_voxel);
}
void kfal_map_destroy(void *h) { delete static_cast<kiss_icp::VoxelHashMap *>(h); }
void kfal_map_add_points(void *h, const double *xyz, int64_t n) {
    std::vector<Eigen::Vector3d> v((size_t)n);
    for (int64_t i = 0; i < n; ++i) v[i] = Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    static_cast<kiss_icp::VoxelHashMap *>(h)->AddPoints(v);
}
// the C handle behind the facade map (for kicp_map_align_planar on the same map)
void *kfal_map_handle(void *h) { return static_cast<kiss_icp::VoxelHashMap *>(h)->handle_; }
// AlignPlanar's results written back as the C records (pose through to_pose7); their number, or -1 when it throws
int32_t kfal_map_align_planar(void *h, const double *xyz, int64_t n, const double *initial, int32_t n_initial,
                              const kicp_planar_align_params *p, kicp_planar_alignment *out) {
    try {
        std::vector<Eigen::Vector3d> pts((size_t)n);
        for (int64_t i = 0; i < n; ++i) pts[i] = Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        std::vector<Sophus::SE3d> starts;
        for (int32_t k = 0; k < n_initial; ++k) starts.push_back(kicp::from_pose7(initial + 7 * k));
        const auto r = static_cast<kiss_icp::VoxelHashMap *>(h)->AlignPlanar(pts, starts, *p);
        for (size_t k = 0; k < r.size(); ++k) {
            const kicp::PlanarAlignment &a = r[k];
            kicp_planar_alignment &o = out[k];
            kicp::to_pose7(a.pose, o.pose);
            o.status = a.status, o.iterations = a.iterations, o.last_step = a.last_step, o.n_inliers = a.n_inliers;
            o.fitness = a.fitness, o.inlier_rmse = a.inlier_rmse, o.sum_sq = a.sum_sq;
            for (int j = 0; j < 6; ++j) o.jtj[j] = a.jtj[j];
            for (int j = 0; j < 3; ++j) o.jtr[j] = a.jtr[j];
        }
        return (int32_t)r.size();
    } catch (const std::exception &) {
        return -1;
    }
}
}
