// extern "C" test hooks over the map-update policy of the C++ facade (KinematicICP::SetMapUpdate / LastMapUpdate on the process-wide
// context, and that context for the C calls) and over the map file of kicp_replay (kicp/map_file.hpp).  Test infrastructure: built as
// tests/hooks/_build/libkicp_map_update_hooks.so by kinematic-icp_b200/cpp/Makefile, linked AGAINST the product libraries, never into
// them.
#include <cstdint>
#include <cstring>
#include <exception>

#include "kicp/map_file.hpp"
#include "kicp/runtime.hpp"
#include "kinematic_icp/pipeline/KinematicICP.hpp"

namespace {
void set_error(const std::exception &e, char *err, int64_t n_err) {
    if (err && n_err > 0) {
        std::strncpy(err, e.what(), (size_t)n_err - 1);
        err[n_err - 1] = '\0';
    }
}
}  // namespace

extern "C" {
// 0, or -1 when SetMapUpdate throws (its message in err)
int32_t kmu_set_map_update(const kicp_map_update_policy *p, char *err, int64_t n_err) {
    try {
        kinematic_icp::pipeline::KinematicICP::SetMapUpdate(*p);
        return 0;
    } catch (const std::exception &e) {
        set_error(e, err, n_err);
        return -1;
    }
}
// LastMapUpdate of a pipeline of kfac_pipeline_create (libkicp_facade_hooks.so)
int32_t kmu_last_map_update(void *pipeline) { return static_cast<kinematic_icp::pipeline::KinematicICP *>(pipeline)->LastMapUpdate(); }
kicp_ctx *kmu_default_context() { return kicp::default_context(); }

// map files: write (0, or -1 with the message), read (a handle, or null with the message), then its header and arrays
int32_t kmu_map_write(const char *path, double voxel_size, uint32_t cap, const int32_t *keys, const int32_t *counts, const double *points,
                      int64_t nv, int64_t np, char *err, int64_t n_err) {
    try {
        kicp::MapFile m;
        m.voxel_size = voxel_size, m.max_points_per_voxel = cap;
        m.keys.assign(keys, keys + 3 * nv), m.counts.assign(counts, counts + nv), m.points.assign(points, points + 3 * np);
        kicp::write_map_file(path, m);
        return 0;
    } catch (const std::exception &e) {
        set_error(e, err, n_err);
        return -1;
    }
}
void *kmu_map_read(const char *path, char *err, int64_t n_err) {
    try {
        return new kicp::MapFile(kicp::read_map_file(path));
    } catch (const std::exception &e) {
        set_error(e, err, n_err);
        return nullptr;
    }
}
void kmu_map_info(void *h, double *voxel_size, uint32_t *cap, int64_t *nv, int64_t *np) {
    const kicp::MapFile &m = *static_cast<kicp::MapFile *>(h);
    *voxel_size = m.voxel_size, *cap = m.max_points_per_voxel, *nv = m.num_voxels(), *np = m.num_points();
}
void kmu_map_copy(void *h, int32_t *keys, int32_t *counts, double *points) {
    const kicp::MapFile &m = *static_cast<kicp::MapFile *>(h);
    std::memcpy(keys, m.keys.data(), m.keys.size() * 4), std::memcpy(counts, m.counts.data(), m.counts.size() * 4);
    std::memcpy(points, m.points.data(), m.points.size() * 8);
}
void kmu_map_free(void *h) { delete static_cast<kicp::MapFile *>(h); }
}
