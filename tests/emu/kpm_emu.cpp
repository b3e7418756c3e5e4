// Host-side emulation of the voxel map with a frozen prior prefix (kicp_map_freeze): the launch sequences of kicp_map.cu's map_insert
// and map_evict with prior_blocks = P > 0, restated on the emulated map of tests/emu/km_emu.cpp — k_add_find_or_create drops the points
// of prior voxels, k_mark_far / the exclusive sum / k_compact_blocks run over the suffix [P, nb) into spare arrays that hold a copy of
// the prefix, and the table is restored from the prior's snapshot before k_table_rebuild re-inserts the suffix.  Test infrastructure
// (tests/test_prior_map_emu_cpu.py); never part of the product library.
#include <map>

#include "km_emu.cpp"

namespace {
struct Prior {
    uint32_t P = 0;
    std::vector<int4> snapshot;  // the table holding the prior alone
};
std::map<void *, Prior> g_prior;

// map_rebuild_table(..., restore = true): the snapshot in place of the clear, then the suffix (`ctr`: the frame path's counters)
void restore_table(EmuMap &m, const Prior &pr, uint32_t nb, const uint32_t *ctr) {
    m.slots = pr.snapshot;
    if (nb > pr.P) {
        int4 *slots = m.slots.data();
        const int4 *blk = m.blk.data();
        const uint32_t mask = m.nslots - 1, P = pr.P;
        emu::launch_waves((int)((nb - P + 255) / 256), 256, [=]() { k_table_rebuild(slots, mask, blk, nb, ctr, P); });
    }
}

// map_evict's suffix launches: k_mark_far, the exclusive sum and k_compact_blocks over [P, nb), then the swap
void evict_suffix(EmuMap &m, const Prior &pr, uint32_t nb, double ox, double oy, double oz, uint32_t *ctr, const kicp_reg_result *d_res,
                  std::vector<uint32_t> &keep, std::vector<uint32_t> &new_id, bool sync) {
    const uint32_t P = pr.P, nl = nb - P;
    const int4 *blk = m.blk.data();
    const double *pts = m.pts.data();
    uint32_t *kp = keep.data();
    const int cap = m.cap;
    const double md2 = m.max_distance * m.max_distance;
    emu::launch_waves((int)((nl + 255) / 256), 256, [=]() { k_mark_far(blk, pts, cap, nb, ox, oy, oz, md2, kp, ctr, d_res, P); });
    if (sync && ctr[4] == 0) return;
    exclusive_sum(keep.data() + P, new_id.data() + P, nl);
    const uint32_t *ni = new_id.data();
    int4 *bo = m.blk_spare.data();
    double *po = m.pts_spare.data();
    emu::launch_waves((int)(((uint64_t)nl * 32 + 255) / 256), 256, [=]() { k_compact_blocks(blk, pts, cap, nb, kp, ni, bo, po, P); });
    std::swap(m.blk, m.blk_spare);
    std::swap(m.pts, m.pts_spare);
}
}  // namespace

extern "C" {
// kicp_map_freeze: every block becomes prior; the spare arrays get the prefix, the snapshot is the table as it stands
void kpm_emu_freeze(void *h) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    Prior &pr = g_prior[h];
    pr.P = m.num_blocks;
    pr.snapshot = m.slots;
    std::copy(m.blk.begin(), m.blk.begin() + pr.P, m.blk_spare.begin());
    std::copy(m.pts.begin(), m.pts.begin() + (size_t)pr.P * m.cap * KICP_PSTRIDE, m.pts_spare.begin());
}
void kpm_emu_thaw(void *h) { g_prior.erase(h); }
uint32_t kpm_emu_prior_blocks(void *h) { return g_prior.count(h) ? g_prior[h].P : 0; }

// AddPoints / the insert half of Update(points, pose) with the prior's blocks read-only (map_add_points_impl)
int kpm_emu_add_points(void *h, const double *xyz, int64_t n, const double *pose7) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    if (n == 0) return 0;
    if ((uint64_t)m.num_blocks + (uint64_t)n > m.blocks_cap) return -1;
    const uint32_t P = kpm_emu_prior_blocks(h);
    std::vector<double> xyz_t((size_t)n * 3);
    std::vector<int32_t> next((size_t)n), touched((size_t)n);
    uint32_t counters[8] = {m.num_blocks, 0, 0, 0, 0, 0, 0, 0};
    MapRW rw = m.rw();
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    const int has_pose = pose7 ? 1 : 0;
    double *xt = xyz_t.data();
    int32_t *nx = next.data(), *tc = touched.data();
    uint32_t *ctr = counters;
    const int grid = (int)((n + 255) / 256);
    emu::launch_waves(grid, 256, [=]() { k_add_find_or_create(rw, xyz, n, has_pose, pose, xt, nx, ctr, tc, nullptr, nullptr, P); });
    const double map_resolution = std::sqrt(m.voxel_size * m.voxel_size / (double)m.cap);
    emu::launch_waves(grid, 256, [=]() { k_add_commit(rw, xt, nx, ctr, tc, map_resolution); });
    if (counters[2]) return -2;
    m.num_blocks = counters[0];
    m.num_points += counters[3];
    return 0;
}

// RemovePointsFarFromLocation with the prior (kicp_map_remove_far -> map_evict, synchronous)
int kpm_emu_remove_far(void *h, const double origin[3]) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    const Prior pr = g_prior.count(h) ? g_prior[h] : Prior{};
    if (m.num_blocks <= pr.P) return 0;
    std::vector<uint32_t> keep(m.num_blocks), new_id(m.num_blocks);
    uint32_t counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    evict_suffix(m, pr, m.num_blocks, origin[0], origin[1], origin[2], counters, nullptr, keep, new_id, true);
    if (counters[4] == 0) return 0;
    m.num_blocks -= counters[4];
    m.num_points -= counters[3];
    if (pr.P) restore_table(m, pr, m.num_blocks, nullptr);
    else rebuild_table(m);
    return 0;
}

// the frame path's Update (kicp_map_update_pose_async) with the prior: count and pose read from device words, nothing read back
int kpm_emu_update_pose_async(void *h, const double *xyz, int64_t n_max, int32_t n_actual, const double pose7[7], int32_t status) {
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
    std::vector<uint32_t> keep(ub), new_id(ub);
    evict_suffix(m, pr, ub, 0.0, 0.0, 0.0, ctr, d_res, keep, new_id, false);
    restore_table(m, pr, ub, ctr);
    m.num_blocks = counters[0] - counters[4];
    m.num_points += (int64_t)counters[3] - (int64_t)counters[5];
    return counters[2] ? -2 : 0;
}

// 1 when the spare arrays hold the live arrays' prior prefix byte for byte (what the next compaction's swap keeps)
int kpm_emu_spare_mirrors_prior(void *h) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    const uint32_t P = kpm_emu_prior_blocks(h);
    if (memcmp(m.blk.data(), m.blk_spare.data(), (size_t)P * sizeof(int4))) return 0;
    return memcmp(m.pts.data(), m.pts_spare.data(), (size_t)P * m.cap * KICP_PSTRIDE * sizeof(double)) == 0;
}

// the occupied slots of the table (key, meta), and of a table rebuilt from scratch over every block: returns the count of each, or
// -1 when cap is too small
int64_t kpm_emu_table(void *h, int32_t fresh, int32_t *out, int64_t cap) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    std::vector<int4> table = m.slots;
    if (fresh) {
        EmuMap t = m;
        rebuild_table(t);
        table = t.slots;
    }
    int64_t n = 0;
    for (const int4 &s : table) {
        if ((uint32_t)s.w == KICP_SLOT_EMPTY) continue;
        if (n >= cap) return -1;
        out[4 * n] = s.x, out[4 * n + 1] = s.y, out[4 * n + 2] = s.z, out[4 * n + 3] = s.w;
        ++n;
    }
    return n;
}
}
