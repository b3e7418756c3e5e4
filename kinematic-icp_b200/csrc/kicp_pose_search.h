// Host side of the pose search (kicp_map_pose_search, kicp_map.cu): validation, the lattice of each level, the children of a level,
// the set of lattice points already scored, the composition of a hypothesis's pose, the ranking key and the merge of the kept
// hypotheses.  Host-only (the key alone is also compiled for the device, for k_pose_select), so that the SIMT emulator harness of
// tests/emu runs its level loop on the same code as the library.
#pragma once
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <array>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "kicp.h"

#if defined(__CUDACC__)
#define KICP_PS_HD __host__ __device__
#else
#define KICP_PS_HD
#endif

constexpr int kPsTile = 8;                     // hypotheses of one rotation per tile of k_pose_score
constexpr int64_t kPsMaxLevel0 = 4194304;      // level-0 hypotheses of one call
constexpr int kPsMaxKeep = 64, kPsMaxLevels = 8;
// points of one call: k_pose_score counts a thread's inliers per hypothesis in 32 bits, and a thread sees n / 256 points at most
constexpr int64_t kPsMaxPoints = (int64_t)1 << 40;

// One scored hypothesis as k_pose_select reads and writes it: lattice point (ix, iy, ipsi), its score, and valid = 0 for the padding
// of a list shorter than `keep`
struct PsEntry {
    int32_t L[3];
    int32_t valid;
    int64_t n_inl;
    double sum_sq;
};

// The ranking key: a ranks before b.  Valid entries first; then more inliers, smaller sum_sq, smaller |ipsi|, smaller ix^2 + iy^2,
// then (ipsi, ix, iy) lexicographic.  Total on distinct lattice points.
KICP_PS_HD inline bool ps_key_less(const PsEntry &a, const PsEntry &b) {
    if (a.valid != b.valid) return a.valid > b.valid;
    if (a.n_inl != b.n_inl) return a.n_inl > b.n_inl;
    if (a.sum_sq != b.sum_sq) return a.sum_sq < b.sum_sq;
    const int64_t pa = a.L[2] < 0 ? -(int64_t)a.L[2] : (int64_t)a.L[2], pb = b.L[2] < 0 ? -(int64_t)b.L[2] : (int64_t)b.L[2];
    if (pa != pb) return pa < pb;
    const uint64_t ra = (uint64_t)((int64_t)a.L[0] * a.L[0]) + (uint64_t)((int64_t)a.L[1] * a.L[1]);
    const uint64_t rb = (uint64_t)((int64_t)b.L[0] * b.L[0]) + (uint64_t)((int64_t)b.L[1] * b.L[1]);
    if (ra != rb) return ra < rb;
    if (a.L[2] != b.L[2]) return a.L[2] < b.L[2];
    if (a.L[0] != b.L[0]) return a.L[0] < b.L[0];
    return a.L[1] < b.L[1];
}

// Level 0 as a product: k[a] = floor(half_extent[a] / step[a]) level-0 steps each side, `scale` = 2^(levels-1) finest steps per
// level-0 step.  Hypothesis h = r * nt + t: rotation r (ipsi = (r - k[2]) * scale), translation t (ix = (t / ny - k[0]) * scale,
// iy = (t % ny - k[1]) * scale) with ny = 2 k[1] + 1, nt = (2 k[0] + 1) ny.
struct PsGrid {
    int32_t k[3];
    int32_t scale;
};

struct PsPlan {
    PsGrid g;
    int levels, keep;
    double u[3];  // the finest steps: step / scale (exact)
    double tau;
    int64_t nr0, nt0, n0;  // level-0 rotations, translations, hypotheses
};

// "" when the parameters are valid (params non-null), else "argument: why"
inline std::string ps_plan(const kicp_pose_search_params *p, int32_t cap, PsPlan *out) {
    for (int a = 0; a < 3; ++a) {
        if (!isfinite(p->half_extent[a])) return "params->half_extent: not finite";
        if (!isfinite(p->step[a])) return "params->step: not finite";
    }
    if (!isfinite(p->tau)) return "params->tau: not finite";
    for (int a = 0; a < 3; ++a)
        if (p->half_extent[a] < 0.0) return "params->half_extent: negative";
    if (p->half_extent[2] > M_PI) return "params->half_extent[2]: yaw above pi";
    for (int a = 0; a < 3; ++a)
        if (!(p->step[a] > 0.0)) return "params->step: not > 0";
    if (!(p->tau > 0.0)) return "params->tau: not > 0";
    if (p->levels < 1 || p->levels > kPsMaxLevels) return "params->levels: not in 1..8";
    if (p->keep < 1 || p->keep > kPsMaxKeep) return "params->keep: not in 1..64";
    if (cap < p->keep) return "cap: below params->keep";
    PsPlan P;
    P.levels = p->levels, P.keep = p->keep, P.tau = p->tau;
    P.g.scale = 1 << (p->levels - 1);
    double n0 = 1.0;
    for (int a = 0; a < 3; ++a) {
        const double q = floor(p->half_extent[a] / p->step[a]);  // >= 0; +inf for a subnormal step
        if (!(q <= (double)kPsMaxLevel0)) return "params: more than 4194304 level-0 hypotheses";
        P.g.k[a] = (int32_t)q;
        n0 *= 2.0 * q + 1.0;
        P.u[a] = p->step[a] / P.g.scale;
    }
    if (n0 > (double)kPsMaxLevel0) return "params: more than 4194304 level-0 hypotheses";
    for (int a = 0; a < 3; ++a)  // children reach one level-0 step beyond the box at most
        if (((int64_t)P.g.k[a] + 1) * P.g.scale > INT32_MAX) return "params: lattice coordinates overflow int32";
    P.nr0 = 2 * (int64_t)P.g.k[2] + 1;
    P.nt0 = (2 * (int64_t)P.g.k[0] + 1) * (2 * (int64_t)P.g.k[1] + 1);
    P.n0 = P.nr0 * P.nt0;
    *out = P;
    return "";
}

inline std::array<int32_t, 3> ps_level0_lattice(const PsGrid &g, int64_t h) {
    const int64_t ny = 2 * (int64_t)g.k[1] + 1, nt = (2 * (int64_t)g.k[0] + 1) * ny;
    const int64_t r = h / nt, t = h % nt;
    return {(int32_t)((t / ny - g.k[0]) * g.scale), (int32_t)((t % ny - g.k[1]) * g.scale), (int32_t)((r - g.k[2]) * g.scale)};
}

// The rotation of a hypothesis of yaw offset psi: normalize(q_prior * (0, 0, sin(psi/2), cos(psi/2))), the Quaternion product and
// SO3::normalize of the facade's compat Eigen / Sophus (cpp/compat) in their operation order; q = (x, y, z, w)
inline void ps_rotation(const double prior[7], double psi, double q[4]) {
    const double ax = prior[0], ay = prior[1], az = prior[2], aw = prior[3];
    const double bx = 0.0, by = 0.0, bz = sin(psi / 2.0), bw = cos(psi / 2.0);
    const double w = aw * bw - ax * bx - ay * by - az * bz;
    const double x = aw * bx + ax * bw + ay * bz - az * by;
    const double y = aw * by + ay * bw + az * bx - ax * bz;
    const double z = aw * bz + az * bw + ax * by - ay * bx;
    double n2 = x * x;
    n2 += y * y;
    n2 += z * z;
    n2 += w * w;
    const double len = sqrt(n2);
    q[0] = x / len, q[1] = y / len, q[2] = z / len, q[3] = w / len;
}

// The translation of a hypothesis of planar offset (x, y): t_prior + q_prior * (x, y, 0), quat_rotate's operation order
inline void ps_translation(const double prior[7], double x, double y, double t[3]) {
    const double qx = prior[0], qy = prior[1], qz = prior[2], qw = prior[3], px = x, py = y, pz = 0.0;
    double ux = qy * pz - qz * py, uy = qz * px - qx * pz, uz = qx * py - qy * px;
    ux = ux + ux, uy = uy + uy, uz = uz + uz;
    const double ox = px + qw * ux + (qy * uz - qz * uy);
    const double oy = py + qw * uy + (qz * ux - qx * uz);
    const double oz = pz + qw * uz + (qx * uy - qy * ux);
    t[0] = prior[4] + ox, t[1] = prior[5] + oy, t[2] = prior[6] + oz;
}

inline void ps_offset(const PsPlan &P, const int32_t L[3], double off[3]) {
    off[0] = L[0] * P.u[0], off[1] = L[1] * P.u[1], off[2] = L[2] * P.u[2];
}

inline void ps_pose(const PsPlan &P, const double prior[7], const int32_t L[3], double pose[7], double off[3]) {
    ps_offset(P, L, off);
    ps_rotation(prior, off[2], pose);
    ps_translation(prior, off[0], off[1], pose + 4);
}

// The lattice points scored so far in a call: level 0's box (implicitly) and those of the refinement levels
struct PsScored {
    const PsPlan *P;
    std::set<std::array<int32_t, 3>> refined;
    int64_t count = 0;
    bool contains(const std::array<int32_t, 3> &L) const {
        bool in0 = true;
        for (int a = 0; a < 3; ++a) {
            const int64_t c = L[a], s = P->g.scale;
            in0 = in0 && c % s == 0 && (c < 0 ? -c : c) <= (int64_t)P->g.k[a] * s;
        }
        return in0 || refined.count(L) != 0;
    }
};

// Level l >= 1: the 26 neighbours c + d * 2^(levels-1-l), d in {-1,0,1}^3 \ {0} (d over (yaw, x, y), lexicographic), of each kept
// hypothesis in rank order, without the points already scored and without repeats; they are marked scored
inline std::vector<std::array<int32_t, 3>> ps_children(const PsPlan &P, int level, const std::vector<PsEntry> &kept, PsScored &scored) {
    std::vector<std::array<int32_t, 3>> out;
    const int32_t s = 1 << (P.levels - 1 - level);
    for (const PsEntry &e : kept)
        for (int dp = -1; dp <= 1; ++dp)
            for (int dx = -1; dx <= 1; ++dx)
                for (int dy = -1; dy <= 1; ++dy) {
                    if (!dp && !dx && !dy) continue;
                    const std::array<int32_t, 3> L{e.L[0] + dx * s, e.L[1] + dy * s, e.L[2] + dp * s};
                    if (scored.contains(L)) continue;
                    scored.refined.insert(L);
                    out.push_back(L);
                }
    scored.count += (int64_t)out.size();
    return out;
}

// The device tables of a refinement level: its points sorted by (ipsi, ix, iy), one rotation per distinct ipsi, one translation per
// distinct (ix, iy); pair_t[h] = the translation of hypothesis h, lat[3h..3h+2] = its lattice point; tiles of k_pose_score as
// (first hypothesis, count <= kPsTile, rotation) triples over runs of one rotation
struct PsTables {
    std::vector<double> rot, trans;
    std::vector<int32_t> pair_t, lat, tiles;
};
inline void ps_tables(const PsPlan &P, const double prior[7], std::vector<std::array<int32_t, 3>> pts, PsTables &T) {
    std::sort(pts.begin(), pts.end(), [](const std::array<int32_t, 3> &a, const std::array<int32_t, 3> &b) {
        return a[2] != b[2] ? a[2] < b[2] : a[0] != b[0] ? a[0] < b[0] : a[1] < b[1];
    });
    T.rot.clear(), T.trans.clear(), T.pair_t.clear(), T.lat.clear(), T.tiles.clear();
    std::map<std::pair<int32_t, int32_t>, int32_t> tix;
    int32_t r = -1, run = 0;
    for (size_t h = 0; h < pts.size(); ++h) {
        const std::array<int32_t, 3> &L = pts[h];
        if (h == 0 || L[2] != pts[h - 1][2]) {
            double q[4];
            ps_rotation(prior, L[2] * P.u[2], q);
            T.rot.insert(T.rot.end(), q, q + 4);
            ++r, run = 0;
        }
        auto it = tix.find({L[0], L[1]});
        if (it == tix.end()) {
            double t[3];
            ps_translation(prior, L[0] * P.u[0], L[1] * P.u[1], t);
            it = tix.emplace(std::make_pair(L[0], L[1]), (int32_t)(T.trans.size() / 3)).first;
            T.trans.insert(T.trans.end(), t, t + 3);
        }
        T.pair_t.push_back(it->second);
        T.lat.insert(T.lat.end(), L.begin(), L.end());
        if (run % kPsTile == 0) T.tiles.insert(T.tiles.end(), {(int32_t)h, 0, r});
        ++T.tiles[T.tiles.size() - 2];
        ++run;
    }
}

// Level 0's tables: rotation r at yaw (r - k[2]) * scale finest steps, translation t at (t / ny - k[0], t % ny - k[1]) * scale
inline void ps_tables0(const PsPlan &P, const double prior[7], PsTables &T) {
    T.rot.resize(4 * P.nr0), T.trans.resize(3 * P.nt0);
    for (int64_t r = 0; r < P.nr0; ++r) ps_rotation(prior, (int32_t)((r - P.g.k[2]) * P.g.scale) * P.u[2], &T.rot[4 * r]);
    const int64_t ny = 2 * (int64_t)P.g.k[1] + 1;
    for (int64_t t = 0; t < P.nt0; ++t)
        ps_translation(prior, (int32_t)((t / ny - P.g.k[0]) * P.g.scale) * P.u[0], (int32_t)((t % ny - P.g.k[1]) * P.g.scale) * P.u[1],
                       &T.trans[3 * t]);
}

// A kept hypothesis with the level that scored it
struct PsKept {
    PsEntry e;
    int32_t level;
};

// The best `keep` of the kept hypotheses and a level's new ones (disjoint sets) by the key
inline void ps_merge(std::vector<PsKept> &kept, const std::vector<PsEntry> &fresh, int level, int keep) {
    for (const PsEntry &e : fresh)
        if (e.valid) kept.push_back(PsKept{e, level});
    std::sort(kept.begin(), kept.end(), [](const PsKept &a, const PsKept &b) { return ps_key_less(a.e, b.e); });
    if ((int)kept.size() > keep) kept.resize(keep);
}

// The caller's record of a kept hypothesis; n = the points scored
inline void ps_output(const PsPlan &P, const double prior[7], const PsKept &k, int64_t n, kicp_pose_hypothesis *o) {
    ps_pose(P, prior, k.e.L, o->pose, o->offset);
    for (int a = 0; a < 3; ++a) o->lattice[a] = k.e.L[a];
    o->level = k.level;
    o->n_inliers = k.e.n_inl;
    o->fitness = n > 0 ? (double)k.e.n_inl / (double)n : 0.0;
    o->inlier_rmse = k.e.n_inl > 0 ? sqrt(k.e.sum_sq / (double)k.e.n_inl) : 0.0;
    o->sum_sq = k.e.sum_sq;
}
