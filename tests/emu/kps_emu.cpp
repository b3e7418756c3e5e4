// Host-side emulation of the pose search (kinematic-icp_b200/csrc/kicp_pose_search_kernels.cuh): k_pose_score and k_pose_select at any
// grid, driven by a level loop restated here on host memory over the library's own host logic (kicp_pose_search.h), on a map built
// by the launch sequences of tests/emu/km_emu.cpp.  Also exports that host logic alone (validation, poses, key, children) for
// tests/test_pose_search_cpu.py.  Test infrastructure (tests/test_pose_search_emu_cpu.py); never part of the product library.
#include "km_emu.cpp"

#include "../../kinematic-icp_b200/csrc/kicp_pose_search_kernels.cuh"

namespace {
// the best `keep` of n scored hypotheses (or entries), k_pose_select's passes as kicp_map.cu runs them, with `per_cta` items a CTA
std::vector<PsEntry> select_best(const int64_t *cnt, const double *sum, const int32_t *lat, PsGrid g, int64_t n, int per_cta, int keep) {
    int64_t parts = (n + per_cta - 1) / per_cta;
    std::vector<PsEntry> a((size_t)parts * keep), b;
    PsEntry *pa = a.data();
    emu::launch_waves((int)parts, kPsThreads, [=]() { k_pose_select(cnt, sum, lat, g, nullptr, n, per_cta, keep, pa); });
    for (int64_t items = parts * keep; items > keep; items = ((items + per_cta - 1) / per_cta) * keep) {
        const int64_t gr = (items + per_cta - 1) / per_cta;
        b.assign((size_t)gr * keep, PsEntry{});
        const PsEntry *in = a.data();
        PsEntry *o = b.data();
        emu::launch_waves((int)gr, kPsThreads, [=]() { k_pose_select(nullptr, nullptr, nullptr, g, in, items, per_cta, keep, o); });
        a.swap(b);
    }
    a.resize(keep);
    return a;
}
}  // namespace

extern "C" {
// ps_plan: 0 and the level-0 geometry, or -1 and the error text
int kps_plan(const kicp_pose_search_params *p, int32_t cap, int64_t *n0, int32_t *k3, int32_t *scale, char *err, int32_t errlen) {
    PsPlan P;
    const std::string why = ps_plan(p, cap, &P);
    snprintf(err, (size_t)errlen, "%s", why.c_str());
    if (!why.empty()) return -1;
    *n0 = P.n0, *scale = P.g.scale;
    for (int a = 0; a < 3; ++a) k3[a] = P.g.k[a];
    return 0;
}
// ps_pose of lattice point L (valid parameters)
void kps_pose(const kicp_pose_search_params *p, const double *prior, const int32_t *L, double *pose, double *off) {
    PsPlan P;
    ps_plan(p, p->keep, &P);
    ps_pose(P, prior, L, pose, off);
}
int kps_key_less(const PsEntry *a, const PsEntry *b) { return ps_key_less(*a, *b) ? 1 : 0; }
// the children of level `level` of the kept lattice points kept[3 * n_kept], given the points scored before: level 0's box and
// refined[3 * n_refined]; returns their number (written to out, at most cap)
int32_t kps_children(const kicp_pose_search_params *p, int32_t level, const int32_t *kept, int32_t n_kept, const int32_t *refined,
                     int32_t n_refined, int32_t *out, int32_t cap) {
    PsPlan P;
    ps_plan(p, p->keep, &P);
    PsScored s{&P, {}, 0};
    for (int i = 0; i < n_refined; ++i) s.refined.insert({refined[3 * i], refined[3 * i + 1], refined[3 * i + 2]});
    std::vector<PsEntry> k(n_kept);
    for (int i = 0; i < n_kept; ++i) k[i] = PsEntry{{kept[3 * i], kept[3 * i + 1], kept[3 * i + 2]}, 1, 0, 0.0};
    const auto kids = ps_children(P, level, k, s);
    for (size_t i = 0; i < kids.size() && (int)i < cap; ++i)
        for (int a = 0; a < 3; ++a) out[3 * i + a] = kids[i][a];
    return (int32_t)kids.size();
}

// The whole search under the emulator: k_pose_score with `score_grid` CTAs, k_pose_select with `per_cta` items a CTA.  level_kept
// [levels][keep][3] and level_n[levels]: the kept lattice points after each level.  Returns 0, or -1 for invalid parameters.
int kps_emu_search(void *h, const double *src, int64_t n, const double *prior, const kicp_pose_search_params *p, int32_t score_grid,
                   int32_t per_cta, kicp_pose_hypothesis *out, int32_t cap, int32_t *n_out, int64_t *n_scored, int32_t *level_kept,
                   int32_t *level_n) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    PsPlan P;
    if (!ps_plan(p, cap, &P).empty() || score_grid <= 0 || per_cta <= 0 || per_cta > kPsThreads * kPsSelectItems) return -1;
    const MapView v = m.view();
    PsTables T;
    std::vector<int64_t> cnt;
    std::vector<double> sum;
    std::vector<PsKept> kept;
    PsScored scored{&P, {}, P.n0};
    for (int level = 0; level < P.levels; ++level) {
        int64_t n_hyp, n_tiles;
        if (level == 0) {
            ps_tables0(P, prior, T);
            n_hyp = P.n0, n_tiles = P.nr0 * ((P.nt0 + kPsTile - 1) / kPsTile);
        } else {
            std::vector<PsEntry> parents;
            for (const PsKept &k : kept) parents.push_back(k.e);
            const auto kids = ps_children(P, level, parents, scored);
            n_hyp = (int64_t)kids.size();
            if (n_hyp) ps_tables(P, prior, kids, T);
            n_tiles = (int64_t)T.tiles.size() / 3;
        }
        if (n_hyp) {
            cnt.assign(n_hyp, -1), sum.assign(n_hyp, NAN);
            const double *rot = T.rot.data(), *tr = T.trans.data();
            const int32_t *pt = level ? T.pair_t.data() : nullptr, *tl = level ? T.tiles.data() : nullptr;
            const int32_t nt = level ? 0 : (int32_t)P.nt0;
            int64_t *c = cnt.data();
            double *s = sum.data();
            const double tau = P.tau;
            const int grid = (int)std::min<int64_t>(score_grid, n_tiles);
            emu::launch_waves(grid, kPsThreads, [=]() { k_pose_score(v, src, n, rot, tr, nt, pt, tl, n_tiles, tau, c, s); });
            const auto best = select_best(cnt.data(), sum.data(), level ? T.lat.data() : nullptr, P.g, n_hyp, per_cta, P.keep);
            ps_merge(kept, best, level, P.keep);
        }
        level_n[level] = (int32_t)kept.size();
        for (size_t i = 0; i < kept.size(); ++i)
            for (int a = 0; a < 3; ++a) level_kept[((size_t)level * P.keep + i) * 3 + a] = kept[i].e.L[a];
    }
    for (size_t i = 0; i < kept.size(); ++i) ps_output(P, prior, kept[i], n, &out[i]);
    *n_out = (int32_t)kept.size();
    *n_scored = scored.count;
    return 0;
}
}
