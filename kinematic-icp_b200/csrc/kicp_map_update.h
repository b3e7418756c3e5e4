// The map-update policy of the frame path (kicp_ctx_set_map_update): the rule that decides whether a frame's Update is applied.
// __host__ __device__, so that the gate kernel (kicp_map_update_kernels.cuh), the read-back order of register_ingested, the SIMT
// emulator of tests/emu and the CPU tests all run this one copy.  It only compares: the outcome is exact for any inputs.
#pragma once
#include <stdint.h>

#include "kicp.h"

#if defined(__CUDACC__)
#define KICP_MU_HD __host__ __device__
#else
#define KICP_MU_HD
#endif

// The outcome (KICP_FRAME_UPDATE_*) of a frame whose registration ended with `reg_status`, under `p`, given the report `st` of its
// source at the returned pose against the map before the frame, and whether that map held no points.  In order: NEVER skips; a status
// other than KICP_OK (a NaN pose) updates nothing; ALWAYS applies; GATED applies on an empty map, else when the report passes all three
// thresholds.  A NaN fitness or RMSE fails its comparison, so it rejects.
KICP_MU_HD inline int32_t map_update_outcome(const kicp_map_update_policy &p, int32_t reg_status, bool map_was_empty,
                                             const kicp_corr_stats &st) {
    if (p.mode == KICP_MAP_UPDATE_NEVER) return KICP_FRAME_UPDATE_SKIPPED;
    if (reg_status != KICP_OK) return KICP_FRAME_UPDATE_NO_CORRESPONDENCES;
    if (p.mode == KICP_MAP_UPDATE_ALWAYS || map_was_empty) return KICP_FRAME_UPDATE_APPLIED;
    const bool pass = st.n_inliers >= p.min_inliers && st.fitness >= p.min_fitness && st.inlier_rmse <= p.max_inlier_rmse;
    return pass ? KICP_FRAME_UPDATE_APPLIED : KICP_FRAME_UPDATE_REJECTED;
}
