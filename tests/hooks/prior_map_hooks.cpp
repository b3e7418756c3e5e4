// extern "C" test hooks over the frozen prior of the C++ facade (kiss_icp::VoxelHashMap::Freeze / Thaw / PriorVoxels / PriorPoints /
// Pointcloud(layer)), on maps of the process-wide context.  Test infrastructure: built as tests/hooks/_build/libkicp_prior_map_hooks.so
// by kinematic-icp_b200/cpp/Makefile, linked AGAINST the product libraries, never into them.
#include <cstdint>
#include <cstring>
#include <exception>
#include <vector>

#include "kicp/runtime.hpp"
#include "kiss_icp/core/VoxelHashMap.hpp"

namespace {
std::vector<Eigen::Vector3d> to_vec(const double *xyz, int64_t n) {
    std::vector<Eigen::Vector3d> v((size_t)n);
    for (int64_t i = 0; i < n; ++i) v[(size_t)i] = Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    return v;
}
}  // namespace

extern "C" {
void *kpm_create(double voxel_size, double max_distance, uint32_t cap) { return new kiss_icp::VoxelHashMap(voxel_size, max_distance, cap); }
void kpm_destroy(void *m) { delete static_cast<kiss_icp::VoxelHashMap *>(m); }
kicp_map *kpm_handle(void *m) { return static_cast<kiss_icp::VoxelHashMap *>(m)->handle_; }
kicp_ctx *kpm_default_context() { return kicp::default_context(); }
void kpm_freeze(void *m) { static_cast<kiss_icp::VoxelHashMap *>(m)->Freeze(); }
void kpm_thaw(void *m) { static_cast<kiss_icp::VoxelHashMap *>(m)->Thaw(); }
void kpm_clear(void *m) { static_cast<kiss_icp::VoxelHashMap *>(m)->Clear(); }
int64_t kpm_prior_voxels(void *m) { return static_cast<kiss_icp::VoxelHashMap *>(m)->PriorVoxels(); }
int64_t kpm_prior_points(void *m) { return static_cast<kiss_icp::VoxelHashMap *>(m)->PriorPoints(); }
void kpm_update_pose(void *m, const double *xyz, int64_t n, const double pose7[7]) {
    static_cast<kiss_icp::VoxelHashMap *>(m)->Update(to_vec(xyz, n), kicp::from_pose7(pose7));
}
// Pointcloud(layer) into out (cap points); returns the point count, or -1 when the call throws (its message in err)
int64_t kpm_pointcloud(void *m, int32_t layer, double *out, int64_t cap, char *err, int64_t n_err) {
    try {
        const std::vector<Eigen::Vector3d> p = static_cast<kiss_icp::VoxelHashMap *>(m)->Pointcloud(layer);
        for (size_t i = 0; i < p.size() && (int64_t)i < cap; ++i) std::memcpy(out + 3 * i, p[i].data(), 3 * sizeof(double));
        return (int64_t)p.size();
    } catch (const std::exception &e) {
        if (err && n_err > 0) {
            std::strncpy(err, e.what(), (size_t)n_err - 1);
            err[n_err - 1] = '\0';
        }
        return -1;
    }
}
}
