// Reader and writer of a voxel map file: the arrays of kicp_map_export_voxels, loaded back with kicp_map_load_voxels, so that a map
// built on one run (kicp_replay --save-map) serves as the prior map of another (--load-map with --map-update never).  Little-endian:
//   char magic[8] = "KICPMAP1"; double voxel_size; uint32 max_points_per_voxel; uint32 0; int64 V; int64 P;
//   int32 keys[3V]; int32 counts[V]; double points[3P]
// The reader validates the whole file before it returns (std::runtime_error naming what is wrong): the magic and the reserved word,
// the length against V and P, every count in [1, max_points_per_voxel] and their sum against P.  Host-only: no Eigen, Sophus or CUDA
// headers.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace kicp {

struct MapFile {
    double voxel_size = 0.0;
    uint32_t max_points_per_voxel = 0;
    std::vector<int32_t> keys;    // 3 per voxel
    std::vector<int32_t> counts;  // 1 per voxel
    std::vector<double> points;   // 3 per point, voxel by voxel in insertion order
    int64_t num_voxels() const { return static_cast<int64_t>(counts.size()); }
    int64_t num_points() const { return static_cast<int64_t>(points.size() / 3); }
};

inline constexpr char kMapFileMagic[8] = {'K', 'I', 'C', 'P', 'M', 'A', 'P', '1'};
inline constexpr int64_t kMapFileHeaderBytes = 8 + 8 + 4 + 4 + 8 + 8;

inline void write_map_file(const std::string &path, const MapFile &m) {
    const int64_t V = m.num_voxels(), P = m.num_points();
    if (m.keys.size() != 3 * m.counts.size() || m.points.size() != 3 * static_cast<size_t>(P))
        throw std::runtime_error(path + ": inconsistent map arrays");
    std::FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("cannot write " + path);
    const uint32_t reserved = 0;
    bool ok = std::fwrite(kMapFileMagic, 1, 8, f) == 8 && std::fwrite(&m.voxel_size, 8, 1, f) == 1 &&
              std::fwrite(&m.max_points_per_voxel, 4, 1, f) == 1 && std::fwrite(&reserved, 4, 1, f) == 1 && std::fwrite(&V, 8, 1, f) == 1 &&
              std::fwrite(&P, 8, 1, f) == 1;
    ok = ok && std::fwrite(m.keys.data(), 4, m.keys.size(), f) == m.keys.size();
    ok = ok && std::fwrite(m.counts.data(), 4, m.counts.size(), f) == m.counts.size();
    ok = ok && std::fwrite(m.points.data(), 8, m.points.size(), f) == m.points.size();
    if (std::fclose(f) != 0 || !ok) throw std::runtime_error("cannot write " + path);
}

inline MapFile read_map_file(const std::string &path) {
    std::FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error("cannot read " + path);
    std::vector<uint8_t> b;
    uint8_t chunk[1 << 16];
    for (size_t r; (r = std::fread(chunk, 1, sizeof(chunk), f)) > 0;) b.insert(b.end(), chunk, chunk + r);
    std::fclose(f);
    const auto bad = [&](const std::string &why) { return std::runtime_error(path + ": " + why); };
    if (b.size() < static_cast<size_t>(kMapFileHeaderBytes)) throw bad("shorter than the header");
    if (std::memcmp(b.data(), kMapFileMagic, 8) != 0) throw bad("not a KICPMAP1 file");
    MapFile m;
    uint32_t reserved;
    int64_t V, P;
    std::memcpy(&m.voxel_size, b.data() + 8, 8);
    std::memcpy(&m.max_points_per_voxel, b.data() + 16, 4);
    std::memcpy(&reserved, b.data() + 20, 4);
    std::memcpy(&V, b.data() + 24, 8);
    std::memcpy(&P, b.data() + 32, 8);
    if (reserved != 0) throw bad("reserved word not 0");
    if (!(m.voxel_size > 0.0)) throw bad("voxel_size not > 0");
    if (V < 0 || P < 0 || V > (int64_t)1 << 40 || P > (int64_t)1 << 40) throw bad("voxel or point count out of range");
    if (static_cast<int64_t>(b.size()) != kMapFileHeaderBytes + 16 * V + 24 * P) throw bad("length does not match V and P");
    const uint8_t *p = b.data() + kMapFileHeaderBytes;
    m.keys.resize(3 * static_cast<size_t>(V)), m.counts.resize(static_cast<size_t>(V)), m.points.resize(3 * static_cast<size_t>(P));
    std::memcpy(m.keys.data(), p, 12 * V);
    std::memcpy(m.counts.data(), p + 12 * V, 4 * V);
    std::memcpy(m.points.data(), p + 16 * V, 24 * P);
    int64_t total = 0;
    for (const int32_t c : m.counts) {
        if (c < 1 || static_cast<uint32_t>(c) > m.max_points_per_voxel) throw bad("a voxel count outside [1, max_points_per_voxel]");
        total += c;
    }
    if (total != P) throw bad("the voxel counts do not sum to P");
    return m;
}

}  // namespace kicp
