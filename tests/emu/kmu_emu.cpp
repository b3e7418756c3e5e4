// Host-side emulation of the frame path's map-update gate (kinematic-icp_b200/csrc/kicp_map_update_kernels.cuh): k_map_update_gate at
// any launch shape, and the rule of kicp_map_update.h on the host, on top of the map's launch sequences of tests/emu/km_emu.cpp (whose
// km_emu_update_pose_async then runs the frame's Update with the gate's shadow block).  Test infrastructure
// (tests/test_map_update_cpu.py, tests/test_map_update_emu_cpu.py); never part of the product library.
#include "km_emu.cpp"

#include "../../kinematic-icp_b200/csrc/kicp_map_update_kernels.cuh"

extern "C" {
// the rule as the host applies it in the read-back order
int32_t kmu_rule(const kicp_map_update_policy *p, int32_t reg_status, int32_t map_was_empty, const kicp_corr_stats *st) {
    return map_update_outcome(*p, reg_status, map_was_empty != 0, *st);
}
// the gate kernel on the emulated device: `res` and `st` as the registration and the report left them, `shadow` and `outcome` written
int32_t kmu_emu_gate(const kicp_reg_result *res, const kicp_corr_stats *st, const kicp_map_update_policy *p, int32_t map_was_empty,
                     int32_t grid, int32_t threads, kicp_reg_result *shadow, int32_t *outcome) {
    if (grid <= 0 || threads <= 0) return -1;
    const kicp_map_update_policy policy = *p;
    emu::launch_waves(grid, threads, [=]() { k_map_update_gate(res, st, policy, map_was_empty, shadow, outcome); });
    return 0;
}
}
