// Host-side emulation of the correspondence report (kinematic-icp_b200/csrc/kicp_corr_kernels.cuh): k_corr_eval at any launch shape,
// then k_corr_finish, on a map built by the launch sequences of tests/emu/km_emu.cpp (k_load_voxels, AddPoints).  The source count
// may come from a device word and the pose from a registration result block, as in the frame path.  Test infrastructure
// (tests/test_correspondences_emu_cpu.py); never part of the product library.
#include "km_emu.cpp"

#include "../../kinematic-icp_b200/csrc/kicp_corr_kernels.cuh"

extern "C" int kc_emu_correspondences(void *h, const double *src, int64_t n, int32_t n_dev, const double *pose7, int32_t from_result,
                                      int32_t status, double tau, int32_t grid, int32_t threads, double *out_pts, double *out_dist,
                                      uint8_t *out_inl, double *partials, kicp_corr_stats *stats) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    if (threads % 32 || threads <= 0 || threads > kCorrThreads || grid <= 0) return -1;
    const MapView v = m.view();
    static int count;
    count = n_dev;
    const int *d_n = n_dev >= 0 ? &count : nullptr;
    static kicp_reg_result res;
    res = kicp_reg_result{};
    Pose pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const kicp_reg_result *d_res = nullptr;
    if (from_result) {
        for (int k = 0; k < 7; ++k) res.pose[k] = pose7[k];
        res.status = status;
        d_res = &res;
        pose = Pose{0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0};  // must not be used
    }
    emu::launch_waves(grid, threads, [=]() { k_corr_eval(v, src, n, d_n, pose, d_res, tau, out_pts, out_dist, out_inl, partials); });
    emu::launch_waves(1, 32, [=]() { k_corr_finish(partials, grid, n, d_n, stats); });
    return 0;
}
