// extern "C" test hooks over the version-3 .kseq reader (kinematic-icp_b200/cpp/kicp/kseq.hpp): read a file and write back what the
// reader returned in the same format, so that a test can compare the bytes, and report the time offsets of the views.  Test
// infrastructure: built as tests/hooks/_build/libkicp_kseq_hooks.so by kinematic-icp_b200/cpp/Makefile; host-only, it links no library.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "kicp/kseq.hpp"

namespace {
// the drive in `path`, its buffers owned by `owned`; the error into err (err_cap bytes) when it throws
bool read(const char *path, kicp::Kseq3Drive &d, std::vector<std::unique_ptr<uint8_t[]>> &owned, char *err, int32_t err_cap) {
    try {
        d = kicp::read_kseq3(path, [&](size_t bytes) {
            owned.emplace_back(new uint8_t[bytes]);
            return static_cast<void *>(owned.back().get());
        });
        return true;
    } catch (const std::exception &e) {
        if (err && err_cap > 0) std::snprintf(err, static_cast<size_t>(err_cap), "%s", e.what());
        return false;
    }
}

template <class T>
void put(std::FILE *f, const T *p, size_t n) {
    std::fwrite(p, sizeof(T), n, f);
}

const kicp::PointFieldView *field(const kicp::PointCloud2View &m, const char *name) {
    for (const auto &x : m.fields)
        if (x.name == name) return &x;
    return nullptr;
}
}  // namespace

extern "C" {
// read_kseq3(in_path), then the drive it returned written to out_path in the version-3 layout (reserved fields 0); 0, or -1 with the
// reader's message in err
int32_t kseq3_rewrite(const char *in_path, const char *out_path, char *err, int32_t err_cap) {
    kicp::Kseq3Drive d;
    std::vector<std::unique_ptr<uint8_t[]>> owned;
    if (!read(in_path, d, owned, err, err_cap)) return -1;
    std::FILE *f = std::fopen(out_path, "wb");
    if (!f) return -2;
    const int32_t zero = 0, head[2] = {static_cast<int32_t>(d.frames.size()), static_cast<int32_t>(d.slots.size())};
    std::fwrite("KSEQ3\0\0\0", 1, 8, f);
    put(f, head, 2), put(f, d.start_pose, 7);
    for (const auto &s : d.slots) put(f, &s.kind, 1), put(f, &s.stamps_relative, 1), put(f, s.lidar_to_base, 7);
    for (const auto &fr : d.frames) {
        const int32_t n_samples = static_cast<int32_t>(fr.samples.size());
        put(f, fr.relative_odometry, 7), put(f, &n_samples, 1), put(f, &zero, 1);
        for (const auto &s : fr.samples) put(f, &s.stamp, 1), put(f, s.pose, 7);
        for (const auto &s : fr.sensors) {
            if (s.kind == kicp::SensorFrame::Kind::LaserScan) {
                const int32_t h[2] = {static_cast<int32_t>(s.scan.n), 0};
                const float p[6] = {s.scan.angle_min, s.scan.angle_max, s.scan.angle_increment, s.scan.time_increment, s.scan.range_min,
                                    s.scan.range_max};
                put(f, h, 2), put(f, &s.header_stamp, 1), put(f, p, 6), put(f, s.scan.ranges, s.scan.n);
                continue;
            }
            const kicp::PointFieldView *t = field(s.cloud, "t");
            const int32_t h[8] = {static_cast<int32_t>(s.cloud.num_points()), static_cast<int32_t>(s.cloud.point_step),
                                  static_cast<int32_t>(field(s.cloud, "x")->offset), static_cast<int32_t>(field(s.cloud, "y")->offset),
                                  static_cast<int32_t>(field(s.cloud, "z")->offset), t ? t->datatype : 0, t ? static_cast<int32_t>(t->offset) : 0, 0};
            put(f, h, 8), put(f, &s.header_stamp, 1), put(f, s.cloud.data, s.cloud.num_points() * s.cloud.point_step);
        }
    }
    return std::fclose(f) == 0 ? 0 : -2;
}
// per frame and slot (frame-major) the seconds the views add to the message's stamps (kicp::SensorFrame::offset()) and whether the
// message is a LaserScan, into offsets / is_scan (room for cap entries); the number of messages, or -1 with the message in err
int64_t kseq3_offsets(const char *path, double *offsets, int32_t *is_scan, int64_t cap, char *err, int32_t err_cap) {
    kicp::Kseq3Drive d;
    std::vector<std::unique_ptr<uint8_t[]>> owned;
    if (!read(path, d, owned, err, err_cap)) return -1;
    int64_t n = 0;
    for (const auto &fr : d.frames)
        for (const auto &s : fr.sensors) {
            if (n < cap) offsets[n] = s.offset(), is_scan[n] = s.kind == kicp::SensorFrame::Kind::LaserScan;
            ++n;
        }
    return n;
}
}
