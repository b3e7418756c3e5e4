// The gate of the frame path's map-update policy (KICP_MAP_UPDATE_GATED, single-synchronisation order): one thread decides, on the
// device, whether the frame's Update is applied, and hands the map's update launches a result block that says so.  Included by
// kicp_frontend.cu; a header of its own so that tests/emu can compile the kernel for the host against the SIMT emulator.
#pragma once
#include "kicp_map_update.h"

// From the registration's result block `d_res` and the report `d_stats` of the frame (k_corr_finish's output, the bytes the report
// returns): `shadow` gets the registration's pose and status KICP_OK when the update is applied, KICP_WARN_NO_CORRESPONDENCES otherwise,
// and `outcome` the KICP_FRAME_UPDATE_* word.  The map's kernels (k_add_find_or_create, k_mark_far) read `shadow` in place of `d_res`
// and leave the map untouched for a status other than KICP_OK, as they do for a NaN pose.  Launch with one thread.
__global__ void k_map_update_gate(const kicp_reg_result *__restrict__ d_res, const kicp_corr_stats *__restrict__ d_stats,
                                  kicp_map_update_policy policy, int map_was_empty, kicp_reg_result *__restrict__ shadow,
                                  int32_t *__restrict__ outcome) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int32_t o = map_update_outcome(policy, d_res->status, map_was_empty != 0, *d_stats);
    for (int k = 0; k < 7; ++k) shadow->pose[k] = d_res->pose[k];
    shadow->status = o == KICP_FRAME_UPDATE_APPLIED ? KICP_OK : KICP_WARN_NO_CORRESPONDENCES;
    *outcome = o;
}
