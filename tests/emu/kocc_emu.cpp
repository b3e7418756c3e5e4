// Host-side emulation of occupancy evidence (kicp_map_set_occupancy): the changed kernels (k_add_find_or_create, k_mark_free and
// k_compact_blocks with their evidence pointers) compiled unchanged against tests/emu/cuda_emu.hpp, and kicp_map.cu's launch sequences
// restated on the emulated map of km_emu.cpp / kpm_emu.cpp (a frozen prior prefix P >= 0) with the evidence array and its spare:
//   - the inserts (map_insert): new blocks start at `initial` inside k_add_find_or_create;
//   - the synchronous eviction (map_evict) and the clearing (kicp_map_clear_free_space_packed): the compaction carries the evidence;
//   - the frame path's Update (kicp_map_update_pose_async), with or without clearing;
//   - freeze (the spare mirrors the prior's prefix) and load (one fill of the loaded blocks).
// Test infrastructure (tests/test_occupancy_emu_cpu.py); never part of the product library.
#include "kfree_emu.cpp"

namespace {
struct Occ {
    std::vector<int32_t> ev, spare;
    int32_t initial = 0;
    OccupancyArgs a{0, 0, 0};
};
std::map<void *, Occ> g_occ;

Occ *occ_of(void *h) {
    auto it = g_occ.find(h);
    return it == g_occ.end() ? nullptr : &it->second;
}
uint32_t prior_of(void *h) { return g_prior.count(h) ? g_prior[h].P : 0; }

// map_insert: k_add_find_or_create (new blocks get `initial` when occupancy is on) and k_add_commit
void insert(EmuMap &m, Occ *o, uint32_t P, const double *xyz, int64_t n, int has_pose, Pose pose, uint32_t *ctr, const int *d_n,
            const kicp_reg_result *d_res) {
    std::vector<double> xyz_t((size_t)n * 3);
    std::vector<int32_t> next((size_t)n), touched((size_t)n);
    MapRW rw = m.rw();
    double *xt = xyz_t.data();
    int32_t *nx = next.data(), *tc = touched.data();
    int32_t *ev = o ? o->ev.data() : nullptr;
    const int32_t init = o ? o->initial : 0;
    const int grid = (int)((n + 255) / 256);
    emu::launch_waves(grid, 256, [=]() { k_add_find_or_create(rw, xyz, n, has_pose, pose, xt, nx, ctr, tc, d_n, d_res, P, ev, init); });
    const double map_resolution = std::sqrt(m.voxel_size * m.voxel_size / (double)m.cap);
    emu::launch_waves(grid, 256, [=]() { k_add_commit(rw, xt, nx, ctr, tc, map_resolution); });
}

// map_compact: the survivors of [P, nb) and their evidence into the spare arrays, the swap
void compact_occ(EmuMap &m, Occ *o, uint32_t P, uint32_t nb, std::vector<uint32_t> &keep, std::vector<uint32_t> &new_id) {
    const uint32_t nl = nb - P;
    exclusive_sum(keep.data() + P, new_id.data() + P, nl);
    const int4 *blk = m.blk.data();
    const double *pts = m.pts.data();
    const uint32_t *kp = keep.data(), *ni = new_id.data();
    int4 *bo = m.blk_spare.data();
    double *po = m.pts_spare.data();
    const int32_t *ev = o ? o->ev.data() : nullptr;
    int32_t *evo = o ? o->spare.data() : nullptr;
    const int cap = m.cap;
    emu::launch_waves((int)(((uint64_t)nl * 32 + 255) / 256), 256,
                      [=]() { k_compact_blocks(blk, pts, cap, nb, kp, ni, bo, po, P, ev, evo); });
    std::swap(m.blk, m.blk_spare);
    std::swap(m.pts, m.pts_spare);
    if (o) std::swap(o->ev, o->spare);
}

void mark_free_occ(EmuMap &m, Occ *o, FreeWords &w, uint32_t nb, uint32_t P, int32_t min_misses, std::vector<uint32_t> &keep, uint32_t *ctr,
                   const kicp_reg_result *d_res) {
    const int4 *blk = m.blk.data();
    const uint32_t *fl = w.flags.data();
    uint32_t *kp = keep.data();
    unsigned long long *st = w.stats.data();
    const uint32_t mm = (uint32_t)min_misses;
    int32_t *ev = o ? o->ev.data() : nullptr;
    const OccupancyArgs a = o ? o->a : OccupancyArgs{0, 0, 0};
    emu::launch_waves((int)((nb + 255) / 256), 256, [=]() { k_mark_free(blk, nb, P, fl, mm, kp, ctr, st, d_res, ev, a); });
}

// the table after a compaction: restored from the prior's snapshot, or rebuilt (`ctr`: the frame path's counters)
void table_after(EmuMap &m, void *h, uint32_t nb, const uint32_t *ctr) {
    const Prior pr = g_prior.count(h) ? g_prior[h] : Prior{};
    if (pr.P) {
        restore_table(m, pr, nb, ctr);
    } else if (!ctr) {
        rebuild_table(m);
    } else {
        std::fill(m.slots.begin(), m.slots.end(), make_int4(-1, -1, -1, (int)KICP_SLOT_EMPTY));
        int4 *slots = m.slots.data();
        const int4 *blk = m.blk.data();
        const uint32_t mask = m.nslots - 1;
        emu::launch_waves((int)((nb + 255) / 256), 256, [=]() { k_table_rebuild(slots, mask, blk, nb, ctr); });
    }
}
}  // namespace

extern "C" {
// kicp_map_set_occupancy: initial 0 turns it off; otherwise both arrays are filled with `initial` over the block capacity
void kocc_emu_set(void *h, int32_t initial, int32_t hit_gain, int32_t miss_loss, int32_t max_evidence) {
    if (!initial) {
        g_occ.erase(h);
        return;
    }
    const EmuMap &m = *static_cast<EmuMap *>(h);
    Occ &o = g_occ[h];
    o.ev.assign(m.blocks_cap, initial), o.spare.assign(m.blocks_cap, initial);
    o.initial = initial, o.a = OccupancyArgs{hit_gain, miss_loss, max_evidence};
}

// kicp_map_export_occupancy: the evidence of blocks [0, num_blocks); returns the count, or -1 when occupancy is off
int64_t kocc_emu_evidence(void *h, int32_t *out) {
    const EmuMap &m = *static_cast<EmuMap *>(h);
    const Occ *o = occ_of(h);
    if (!o) return -1;
    std::copy(o->ev.begin(), o->ev.begin() + m.num_blocks, out);
    return m.num_blocks;
}

// 1 when the spare evidence holds the prior's prefix (what the next compaction's swap keeps)
int kocc_emu_spare_mirrors_prior(void *h) {
    const Occ *o = occ_of(h);
    const uint32_t P = prior_of(h);
    return !o || std::equal(o->ev.begin(), o->ev.begin() + P, o->spare.begin());
}

// kicp_map_freeze: map_mirror_prior copies the evidence prefix too
void kocc_emu_freeze(void *h) {
    kpm_emu_freeze(h);
    if (Occ *o = occ_of(h)) {
        const uint32_t P = prior_of(h);
        std::copy(o->ev.begin(), o->ev.begin() + P, o->spare.begin());
    }
}

// kicp_map_load_voxels: clear (the prior goes), k_load_voxels, the table, and one fill of the loaded blocks' evidence
int kocc_emu_load(void *h, const int32_t *keys, const int32_t *counts, const double *points, int64_t nvox) {
    kpm_emu_thaw(h);
    const int rc = km_emu_load_voxels(h, keys, counts, points, nvox);
    if (rc) return rc;
    if (Occ *o = occ_of(h)) {
        int32_t *ev = o->ev.data();
        const int32_t init = o->initial;
        const uint32_t nv = (uint32_t)nvox;
        if (nv) emu::launch_waves((int)((nv + 255) / 256), 256, [=]() { k_fill_i32(ev, init, nv); });
    }
    return 0;
}

// AddPoints / the insert half of Update(points, pose) (map_add_points_impl): returns 0, or < 0 on an emulator limit
int kocc_emu_add_points(void *h, const double *xyz, int64_t n, const double *pose7) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    if (n == 0) return 0;
    if ((uint64_t)m.num_blocks + (uint64_t)n > m.blocks_cap) return -1;
    uint32_t counters[8] = {m.num_blocks, 0, 0, 0, 0, 0, 0, 0};
    Pose pose{0, 0, 0, 1, 0, 0, 0};
    if (pose7) pose = Pose{pose7[0], pose7[1], pose7[2], pose7[3], pose7[4], pose7[5], pose7[6]};
    insert(m, occ_of(h), prior_of(h), xyz, n, pose7 ? 1 : 0, pose, counters, nullptr, nullptr);
    if (counters[2]) return -2;
    m.num_blocks = counters[0];
    m.num_points += counters[3];
    return 0;
}

// RemovePointsFarFromLocation (map_evict, synchronous): k_mark_far over [P, nb), the compaction only when a block died
int kocc_emu_remove_far(void *h, const double origin[3]) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    const uint32_t P = prior_of(h), nb = m.num_blocks;
    if (nb <= P) return 0;
    std::vector<uint32_t> keep(nb), new_id(nb);
    uint32_t counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    {
        const int4 *blk = m.blk.data();
        const double *pts = m.pts.data();
        uint32_t *kp = keep.data(), *ctr = counters;
        const int cap = m.cap;
        const double ox = origin[0], oy = origin[1], oz = origin[2], md2 = m.max_distance * m.max_distance;
        emu::launch_waves((int)((nb - P + 255) / 256), 256, [=]() { k_mark_far(blk, pts, cap, nb, ox, oy, oz, md2, kp, ctr, nullptr, P); });
    }
    if (counters[4] == 0) return 0;
    compact_occ(m, occ_of(h), P, nb, keep, new_id);
    m.num_blocks -= counters[4];
    m.num_points -= counters[3];
    table_after(m, h, m.num_blocks, nullptr);
    return 0;
}

// kicp_map_clear_free_space_packed: flags, k_free_rays, k_mark_free (with the evidence when on), and when a block was cleared the
// compaction and the table; returns 0
int kocc_emu_clear(void *h, const double *xyz, int64_t n, const double pose7[7], const double origin[3], double end_margin,
                   int32_t min_misses, int32_t grid, int64_t *stats) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    Occ *o = occ_of(h);
    const uint32_t P = prior_of(h);
    FreeWords w;
    if (n > 0) {
        const uint32_t nb = m.num_blocks;
        uint32_t counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        free_rays(m, w, nb, xyz, n, nullptr, pose7, nullptr, origin, end_margin, min_misses, grid);
        std::vector<uint32_t> keep(std::max<uint32_t>(nb, 1)), new_id(std::max<uint32_t>(nb, 1));
        if (nb) mark_free_occ(m, o, w, nb, P, min_misses, keep, counters, nullptr);
        if (counters[4]) {
            compact_occ(m, o, P, nb, keep, new_id);
            m.num_blocks -= counters[4];
            m.num_points -= counters[3];
            table_after(m, h, m.num_blocks, nullptr);
        }
    }
    copy_stats(w, stats);
    return 0;
}

// kicp_map_update_pose_async (the frame path's Update): the insert, with min_misses > 0 the clearing's flags and k_free_rays, then
// k_mark_far, k_mark_free, the compaction and the table; count and pose read from device words.  Returns 0, or < 0 on an emulator limit
int kocc_emu_update_pose_async(void *h, const double *xyz, int64_t n_max, int32_t n_actual, const double pose7[7], int32_t status,
                               const double origin[3], double end_margin, int32_t min_misses, int32_t grid, int64_t *stats) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    Occ *o = occ_of(h);
    const uint32_t P = prior_of(h);
    if (n_max <= 0) return -3;
    if ((uint64_t)m.num_blocks + (uint64_t)n_max > m.blocks_cap) return -1;
    uint32_t counters[8] = {m.num_blocks, 0, 0, 0, 0, 0, 0, 0};
    const int d_n_word = n_actual;
    kicp_reg_result res;
    memset(&res, 0, sizeof(res));
    for (int k = 0; k < 7; ++k) res.pose[k] = pose7[k];
    res.status = status;
    uint32_t *ctr = counters;
    const kicp_reg_result *d_res = &res;
    insert(m, o, P, xyz, n_max, 1, Pose{0, 0, 0, 1, 0, 0, 0}, ctr, &d_n_word, d_res);
    const uint32_t ub = (uint32_t)std::min<uint64_t>((uint64_t)m.num_blocks + (uint64_t)n_max, m.blocks_cap);
    FreeWords w;
    if (min_misses) free_rays(m, w, ub, xyz, n_max, &d_n_word, nullptr, d_res, origin, end_margin, min_misses, grid);
    std::vector<uint32_t> keep(ub), new_id(ub);
    {
        const int4 *blk = m.blk.data();
        const double *pts = m.pts.data();
        uint32_t *kp = keep.data();
        const int cap = m.cap;
        const double md2 = m.max_distance * m.max_distance;
        emu::launch_waves((int)((ub - P + 255) / 256), 256, [=]() { k_mark_far(blk, pts, cap, ub, 0.0, 0.0, 0.0, md2, kp, ctr, d_res, P); });
    }
    if (min_misses) mark_free_occ(m, o, w, ub, P, min_misses, keep, ctr, d_res);
    compact_occ(m, o, P, ub, keep, new_id);
    table_after(m, h, ub, ctr);
    m.num_blocks = counters[0] - counters[4];
    m.num_points += (int64_t)counters[3] - (int64_t)counters[5];
    if (stats) copy_stats(w, stats);
    return counters[2] ? -2 : 0;
}
}
