// Host-side emulation of free-space clearing (kinematic-icp_b200/csrc/kicp_free_space_kernels.cuh): the kernels compiled unchanged
// against tests/emu/cuda_emu.hpp, and the launch sequences of kicp_map.cu restated on the emulated map of km_emu.cpp / kpm_emu.cpp (a
// frozen prior prefix P >= 0):
//   - kicp_map_clear_free_space_packed: flags cleared, k_free_rays, k_mark_free, and when a voxel was cleared the compaction of [P, nb)
//     and the table restore;
//   - kicp_map_update_pose_async with the option: the insert, flags cleared, k_free_rays (count and pose read from device words),
//     k_mark_far, k_mark_free, the compaction and the table restore.
// Test infrastructure (tests/test_free_space_emu_cpu.py); never part of the product library.
#include "kpm_emu.cpp"

inline unsigned atomicOr(unsigned *p, unsigned v) {
    emu::chaos_point();
    return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST);
}

#include "../../kinematic-icp_b200/csrc/kicp_free_space_kernels.cuh"

namespace {
struct FreeWords {
    std::vector<unsigned long long> stats = std::vector<unsigned long long>(kFreeStatWords, 0ull);
    std::vector<uint32_t> flags;
};

// k_free_rays on `grid` CTAs (0: one lane per ray, as many CTAs as that takes)
void free_rays(EmuMap &m, FreeWords &w, uint32_t nb, const double *xyz, int64_t n, const int *d_n, const double *pose7,
               const kicp_reg_result *d_res, const double origin[3], double end_margin, int32_t min_misses, int grid) {
    w.flags.assign(std::max<uint32_t>(nb, 1), 0u);
    std::fill(w.stats.begin(), w.stats.end(), 0ull);
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const FreeRayArgs a{origin[0], origin[1], origin[2], end_margin, m.max_distance, (uint32_t)min_misses};
    const MapView v = m.view();
    uint32_t *fl = w.flags.data();
    unsigned long long *st = w.stats.data();
    const int g = grid > 0 ? grid : (int)std::max<int64_t>(1, (n + 255) / 256);
    emu::launch_waves(g, 256, [=]() { k_free_rays(v, xyz, n, d_n, pose, d_res, a, fl, st); });
}

void mark_free(EmuMap &m, FreeWords &w, uint32_t nb, uint32_t P, int32_t min_misses, std::vector<uint32_t> &keep, uint32_t *ctr,
               const kicp_reg_result *d_res) {
    const int4 *blk = m.blk.data();
    const uint32_t *fl = w.flags.data();
    uint32_t *kp = keep.data();
    unsigned long long *st = w.stats.data();
    const uint32_t mm = (uint32_t)min_misses;
    emu::launch_waves((int)((nb + 255) / 256), 256, [=]() { k_mark_free(blk, nb, P, fl, mm, kp, ctr, st, d_res); });
}

// map_compact: the survivors of [P, nb) into the spare arrays, the swap
void compact(EmuMap &m, uint32_t P, uint32_t nb, std::vector<uint32_t> &keep, std::vector<uint32_t> &new_id) {
    const uint32_t nl = nb - P;
    exclusive_sum(keep.data() + P, new_id.data() + P, nl);
    const int4 *blk = m.blk.data();
    const double *pts = m.pts.data();
    const uint32_t *kp = keep.data(), *ni = new_id.data();
    int4 *bo = m.blk_spare.data();
    double *po = m.pts_spare.data();
    const int cap = m.cap;
    emu::launch_waves((int)(((uint64_t)nl * 32 + 255) / 256), 256, [=]() { k_compact_blocks(blk, pts, cap, nb, kp, ni, bo, po, P); });
    std::swap(m.blk, m.blk_spare);
    std::swap(m.pts, m.pts_spare);
}

void copy_stats(const FreeWords &w, int64_t *out) {
    for (int k = 0; k < 5; ++k) out[k] = (int64_t)w.stats[k];
}
}  // namespace

extern "C" {
// kicp_map_clear_free_space on the emulated map: returns 0
int kfree_emu_clear(void *h, const double *xyz, int64_t n, const double pose7[7], const double origin[3], double end_margin,
                    int32_t min_misses, int32_t grid, int64_t *stats) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    const Prior pr = g_prior.count(h) ? g_prior[h] : Prior{};
    FreeWords w;
    if (n > 0) {
        const uint32_t nb = m.num_blocks;
        uint32_t counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        free_rays(m, w, nb, xyz, n, nullptr, pose7, nullptr, origin, end_margin, min_misses, grid);
        std::vector<uint32_t> keep(std::max<uint32_t>(nb, 1)), new_id(std::max<uint32_t>(nb, 1));
        if (nb) mark_free(m, w, nb, pr.P, min_misses, keep, counters, nullptr);
        if (counters[4]) {
            compact(m, pr.P, nb, keep, new_id);
            m.num_blocks -= counters[4];
            m.num_points -= counters[3];
            if (pr.P) restore_table(m, pr, m.num_blocks, nullptr);
            else rebuild_table(m);
        }
    }
    copy_stats(w, stats);
    return 0;
}

// kicp_map_update_pose_async with free-space clearing (the frame path's sequence): returns 0, or < 0 on an emulator limit
int kfree_emu_update_pose_async(void *h, const double *xyz, int64_t n_max, int32_t n_actual, const double pose7[7], int32_t status,
                                const double origin[3], double end_margin, int32_t min_misses, int32_t grid, int64_t *stats) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    const Prior pr = g_prior.count(h) ? g_prior[h] : Prior{};
    if (n_max <= 0) return -3;
    if ((uint64_t)m.num_blocks + (uint64_t)n_max > m.blocks_cap) return -1;
    std::vector<double> xyz_t((size_t)n_max * 3);
    std::vector<int32_t> next((size_t)n_max), touched((size_t)n_max);
    uint32_t counters[8] = {m.num_blocks, 0, 0, 0, 0, 0, 0, 0};
    const int d_n_word = n_actual;
    kicp_reg_result res;
    memset(&res, 0, sizeof(res));
    for (int k = 0; k < 7; ++k) res.pose[k] = pose7[k];
    res.status = status;
    MapRW rw = m.rw();
    double *xt = xyz_t.data();
    int32_t *nx = next.data(), *tc = touched.data();
    uint32_t *ctr = counters;
    const int *d_n = &d_n_word;
    const kicp_reg_result *d_res = &res;
    const uint32_t P = pr.P;
    const int pgrid = (int)((n_max + 255) / 256);
    emu::launch_waves(pgrid, 256,
                      [=]() { k_add_find_or_create(rw, xyz, n_max, 1, Pose{0, 0, 0, 1, 0, 0, 0}, xt, nx, ctr, tc, d_n, d_res, P); });
    const double map_resolution = std::sqrt(m.voxel_size * m.voxel_size / (double)m.cap);
    emu::launch_waves(pgrid, 256, [=]() { k_add_commit(rw, xt, nx, ctr, tc, map_resolution); });
    const uint32_t ub = (uint32_t)std::min<uint64_t>((uint64_t)m.num_blocks + (uint64_t)n_max, m.blocks_cap);
    FreeWords w;
    free_rays(m, w, ub, xyz, n_max, d_n, nullptr, d_res, origin, end_margin, min_misses, grid);
    std::vector<uint32_t> keep(ub), new_id(ub);
    {
        const int4 *blk = m.blk.data();
        const double *pts = m.pts.data();
        uint32_t *kp = keep.data();
        const int cap = m.cap;
        const double md2 = m.max_distance * m.max_distance;
        const uint32_t nl = ub - P;
        emu::launch_waves((int)((nl + 255) / 256), 256, [=]() { k_mark_far(blk, pts, cap, ub, 0.0, 0.0, 0.0, md2, kp, ctr, d_res, P); });
    }
    mark_free(m, w, ub, P, min_misses, keep, ctr, d_res);
    compact(m, P, ub, keep, new_id);
    if (P) {
        restore_table(m, pr, ub, ctr);
    } else {
        std::fill(m.slots.begin(), m.slots.end(), make_int4(-1, -1, -1, (int)KICP_SLOT_EMPTY));
        int4 *slots = m.slots.data();
        const int4 *blk = m.blk.data();
        const uint32_t mask = m.nslots - 1;
        emu::launch_waves((int)((ub + 255) / 256), 256, [=]() { k_table_rebuild(slots, mask, blk, ub, ctr); });
    }
    m.num_blocks = counters[0] - counters[4];
    m.num_points += (int64_t)counters[3] - (int64_t)counters[5];
    copy_stats(w, stats);
    return counters[2] ? -2 : 0;
}
}
