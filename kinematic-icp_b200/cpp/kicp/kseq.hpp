// Reader of version-3 .kseq drives (the format is documented in tools/kicp_replay.cpp): a table of message streams ("slots", one
// PointCloud2 or LaserScan sensor each, with its extrinsic) and per frame one message per slot plus the wheel odometry, as one relative
// motion and optionally as poses sampled during the sweep.  The messages come back as the views KinematicICP's staging calls take
// (kicp::SensorFrame over a PointCloud2View or a LaserScanView); the records and ranges live in buffers of the caller's allocator, one per
// message, so that a replay can read them from page-locked memory.
// Everything in the file is validated here, before any library call: a malformed file throws std::runtime_error naming the frame and
// the slot.  Host-only: no Eigen, Sophus or CUDA headers.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "kicp.h"
#include "kicp/laser_scan.hpp"
#include "kicp/pointcloud2.hpp"
#include "kicp/sensor_frame.hpp"

namespace kicp {

struct KseqSlot {
    enum Kind : int32_t { Records = 0, LaserScan = 1 };
    int32_t kind = Records;
    int32_t stamps_relative = 0;  // records: 1 = the time field counts from the header stamp (time_offset = header_stamp)
    double lidar_to_base[7] = {0, 0, 0, 1, 0, 0, 0};
};

struct KseqSample {
    double stamp = 0.0;  // odometry clock
    double pose[7] = {0, 0, 0, 1, 0, 0, 0};  // the base pose in the odometry frame
};

struct KseqFrame {
    double relative_odometry[7] = {0, 0, 0, 1, 0, 0, 0};
    std::vector<KseqSample> samples;  // empty: one motion over the sweep
    std::vector<SensorFrame> sensors;  // one per slot, in slot order
};

struct Kseq3Drive {
    double start_pose[7] = {0, 0, 0, 1, 0, 0, 0};
    std::vector<KseqSlot> slots;
    std::vector<KseqFrame> frames;
};

// the version of a .kseq magic ("KSEQ1\0\0\0" .. "KSEQ3\0\0\0"), 0 for anything else
inline int kseq_version(const char magic[8]) {
    for (int v = 1; v <= 3; ++v) {
        const char m[8] = {'K', 'S', 'E', 'Q', static_cast<char>('0' + v), 0, 0, 0};
        if (std::memcmp(magic, m, 8) == 0) return v;
    }
    return 0;
}

namespace detail {
class KseqFile {
public:
    KseqFile(std::FILE *f, long size) : f_(f), left_(size) {}
    // where the next read is, for messages: "frame 3, slot 1"
    std::string where;
    template <class T>
    void read(T *dst, size_t count, const char *what) {
        const size_t bytes = sizeof(T) * count;
        if (bytes > left_ || std::fread(dst, 1, bytes, f_) != bytes) fail(std::string("truncated while reading ") + what);
        left_ -= bytes;
    }
    // true when `count` items of `item_bytes` each cannot fit in what is left of the file (checked before allocating for them)
    bool exceeds(uint64_t count, uint64_t item_bytes) const { return item_bytes && count > left_ / item_bytes; }
    uint64_t left() const { return left_; }
    [[noreturn]] void fail(const std::string &what) const { throw std::runtime_error(where.empty() ? what : where + ": " + what); }

private:
    std::FILE *f_;
    uint64_t left_;
};

inline bool finite7(const double *p) {
    for (int i = 0; i < 7; ++i)
        if (!std::isfinite(p[i])) return false;
    return true;
}
}  // namespace detail

// The drive in `path`, a version-3 .kseq file.  alloc(bytes) returns a buffer for one message's records or ranges (at least 1 byte is
// asked for an empty message); the caller owns what it returns.
inline Kseq3Drive read_kseq3(const std::string &path, const std::function<void *(size_t)> &alloc) {
    std::FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error("cannot open " + path);
    struct Closer {
        std::FILE *f;
        ~Closer() { std::fclose(f); }
    } closer{f};
    long size = -1;
    if (std::fseek(f, 0, SEEK_END) == 0) size = std::ftell(f);
    if (size < 0 || std::fseek(f, 0, SEEK_SET) != 0) throw std::runtime_error("cannot read " + path);
    detail::KseqFile in(f, size);
    char magic[8];
    in.read(magic, 8, "the magic");
    const int version = kseq_version(magic);
    if (version == 0) in.fail("not a .kseq file (bad magic)");
    if (version != 3) in.fail("a version-" + std::to_string(version) + " .kseq file, not version 3");
    Kseq3Drive d;
    int32_t n_frames = 0, n_slots = 0;
    in.read(&n_frames, 1, "the header"), in.read(&n_slots, 1, "the header");
    in.read(d.start_pose, 7, "the start pose");
    if (!detail::finite7(d.start_pose)) in.fail("non-finite start pose");
    if (n_slots < 1 || n_slots > KICP_MAX_SENSORS)
        in.fail("slot count " + std::to_string(n_slots) + " outside [1, " + std::to_string(KICP_MAX_SENSORS) + "]");
    d.slots.resize(static_cast<size_t>(n_slots));
    for (int32_t s = 0; s < n_slots; ++s) {
        KseqSlot &slot = d.slots[static_cast<size_t>(s)];
        in.where = "slot " + std::to_string(s);
        in.read(&slot.kind, 1, "the slot table"), in.read(&slot.stamps_relative, 1, "the slot table");
        in.read(slot.lidar_to_base, 7, "the slot table");
        if (slot.kind != KseqSlot::Records && slot.kind != KseqSlot::LaserScan)
            in.fail("kind " + std::to_string(slot.kind) + " is neither 0 (PointCloud2 records) nor 1 (LaserScan)");
        if (slot.stamps_relative != 0 && slot.stamps_relative != 1) in.fail("stamps_relative " + std::to_string(slot.stamps_relative) + " is neither 0 nor 1");
        if (!detail::finite7(slot.lidar_to_base)) in.fail("non-finite lidar_to_base");
    }
    in.where.clear();
    // a frame takes 64 bytes and at least 40 per slot: a count the file cannot hold is not allocated for
    if (n_frames < 0 || n_frames > (1 << 24) || in.exceeds(static_cast<uint64_t>(n_frames), 64 + 40 * static_cast<uint64_t>(n_slots)))
        in.fail("implausible frame count " + std::to_string(n_frames));
    d.frames.resize(static_cast<size_t>(n_frames));
    for (int32_t k = 0; k < n_frames; ++k) {
        KseqFrame &fr = d.frames[static_cast<size_t>(k)];
        in.where = "frame " + std::to_string(k);
        int32_t n_samples = 0, reserved = 0;
        in.read(fr.relative_odometry, 7, "the frame header");
        in.read(&n_samples, 1, "the frame header"), in.read(&reserved, 1, "the frame header");
        if (!detail::finite7(fr.relative_odometry)) in.fail("non-finite relative_odometry");
        if (n_samples < 0 || n_samples > (1 << 20)) in.fail("implausible sample count " + std::to_string(n_samples));
        if (in.exceeds(static_cast<uint64_t>(n_samples), sizeof(KseqSample))) in.fail("truncated while reading the odometry samples");
        fr.samples.resize(static_cast<size_t>(n_samples));
        for (int32_t i = 0; i < n_samples; ++i) {
            KseqSample &s = fr.samples[static_cast<size_t>(i)];
            in.read(&s.stamp, 1, "the odometry samples"), in.read(s.pose, 7, "the odometry samples");
            if (!std::isfinite(s.stamp)) in.fail("sample " + std::to_string(i) + ": non-finite stamp");
            if (!detail::finite7(s.pose)) in.fail("sample " + std::to_string(i) + ": non-finite pose");
            if (i > 0 && !(fr.samples[static_cast<size_t>(i) - 1].stamp < s.stamp))
                in.fail("sample " + std::to_string(i) + ": stamps do not increase");
        }
        for (int32_t s = 0; s < n_slots; ++s) {
            const KseqSlot &slot = d.slots[static_cast<size_t>(s)];
            in.where = "frame " + std::to_string(k) + ", slot " + std::to_string(s);
            double header = 0.0;
            if (slot.kind == KseqSlot::Records) {
                int32_t h[8];  // n_points, point_step, offset_x, offset_y, offset_z, stamp_datatype, stamp_offset, reserved
                in.read(h, 8, "the message header"), in.read(&header, 1, "the message header");
                if (!std::isfinite(header)) in.fail("non-finite header stamp");
                if (h[0] < 0) in.fail("negative point count " + std::to_string(h[0]));
                if (h[1] <= 0) in.fail("point_step " + std::to_string(h[1]) + " is not positive");
                for (int a = 0; a < 3; ++a)
                    if (h[2 + a] < 0 || static_cast<int64_t>(h[2 + a]) + 4 > h[1]) in.fail(std::string(1, "xyz"[a]) + " outside point_step");
                if (h[5] != 0 && h[5] != PF_UINT32 && h[5] != PF_FLOAT32 && h[5] != PF_FLOAT64)
                    in.fail("stamp_datatype " + std::to_string(h[5]) + " is none of 0, 6 (UINT32), 7 (FLOAT32), 8 (FLOAT64)");
                if (h[5] != 0 && (h[6] < 0 || static_cast<int64_t>(h[6]) + (h[5] == PF_FLOAT64 ? 8 : 4) > h[1]))
                    in.fail("time field outside point_step");
                if (in.exceeds(static_cast<uint64_t>(h[0]), static_cast<uint64_t>(h[1]))) in.fail("truncated while reading the records");
                const size_t bytes = static_cast<size_t>(h[0]) * static_cast<size_t>(h[1]);
                uint8_t *raw = static_cast<uint8_t *>(alloc(bytes ? bytes : 1));
                in.read(raw, bytes, "the records");
                PointCloud2View m;
                m.data = raw, m.width = static_cast<uint32_t>(h[0]), m.height = 1, m.point_step = static_cast<uint32_t>(h[1]);
                m.fields = {{"x", static_cast<uint32_t>(h[2]), PF_FLOAT32, 1}, {"y", static_cast<uint32_t>(h[3]), PF_FLOAT32, 1},
                            {"z", static_cast<uint32_t>(h[4]), PF_FLOAT32, 1}};
                if (h[5] != 0) m.fields.push_back({"t", static_cast<uint32_t>(h[6]), static_cast<uint8_t>(h[5]), 1});
                fr.sensors.push_back(SensorFrame::FromPointCloud2(m, header, slot.stamps_relative ? header : 0.0));
            } else {
                int32_t h[2];  // n_beams, reserved
                float p[6];    // angle_min, angle_max, angle_increment, time_increment, range_min, range_max
                in.read(h, 2, "the message header"), in.read(&header, 1, "the message header"), in.read(p, 6, "the message header");
                if (!std::isfinite(header)) in.fail("non-finite header stamp");
                if (h[0] < 0) in.fail("negative beam count " + std::to_string(h[0]));
                if (in.exceeds(static_cast<uint64_t>(h[0]), sizeof(float))) in.fail("truncated while reading the ranges");
                float *ranges = static_cast<float *>(alloc(h[0] ? sizeof(float) * static_cast<size_t>(h[0]) : 1));
                in.read(ranges, static_cast<size_t>(h[0]), "the ranges");
                LaserScanView v;
                v.ranges = ranges, v.n = static_cast<size_t>(h[0]);
                v.angle_min = p[0], v.angle_max = p[1], v.angle_increment = p[2], v.time_increment = p[3], v.range_min = p[4], v.range_max = p[5];
                fr.sensors.push_back(SensorFrame::FromLaserScan(v, header));
            }
        }
    }
    in.where.clear();
    if (in.left() != 0) in.fail(std::to_string(in.left()) + " bytes after the last frame");
    return d;
}

}  // namespace kicp
