// kicp_replay — offline replay of a recorded drive through kinematic_icp::pipeline::KinematicICP, the way
// ros/src/kinematic_icp_ros/nodes/offline_node.cpp:99-149 replays a bag: for every frame RegisterFrame(cloud, stamps,
// lidar_to_base, relative wheel odometry), collect the poses, write them in TUM format (offline_node.cpp:76-97).
// There is no ROS here, so the input is a flat ".kseq" file (below) instead of a bag: float32 x,y,z per point exactly as a
// PointCloud2 message carries them (ros/.../utils/RosUtils.cpp:30-39), handed to the facade without widening on the host.
//
//   kicp_replay drive.kseq out.tum [--deskew 0|1] [--voxel-size v] [--max-range r] [--min-range r] [--repeat k] [--pageable]
//               [--host-stamps] [--device-input] [--publish host|device|live] [--publish-digest FILE] [--downsample-order 0|1]
//               [--correspondences FILE] [--map-update always|never|gated] [--min-inliers k] [--min-fitness f]
//               [--max-inlier-rmse r] [--load-map FILE] [--freeze-prior] [--save-map FILE]
//
// .kseq, little endian:  char magic[8] = "KSEQ1\0\0\0"; int32 n_frames; int32 reserved; double lidar_to_base[7]; double start_pose[7];
//   per frame: int32 n_points; int32 has_stamps; double header_stamp; double relative_odometry[7]; float xyz[3 n]; double stamps[n] (if has_stamps)
// (poses are {qx, qy, qz, qw, tx, ty, tz}).
// Version 2, magic "KSEQ2\0\0\0", same header, carries the raw records the online node receives:
//   per frame: int32 n_points; int32 point_step; int32 offset_x, offset_y, offset_z (FLOAT32 fields); int32 stamp_datatype (PointField
//   UINT32 6 / FLOAT32 7 / FLOAT64 8, 0 = no time field); int32 stamp_offset; int32 reserved; double header_stamp;
//   double relative_odometry[7]; uint8 records[n * point_step]
// and is replayed as the online node runs a frame: KinematicICP::StageFrame (the stamps decoded on the device, the sweep interval
// back to the host), then RegisterStagedFrame.  --host-stamps replays it the host-decoding way instead: extract_timestamps +
// process_timestamps + RegisterFrame.  Both write the same poses.
// --device-input (KSEQ2 and KSEQ3, staged) replays a drive whose records a GPU producer left in device memory: every frame's records are copied
// to device memory once, before the repetitions, and each frame is staged from there with KinematicICP::StageDeviceFrame, then
// registered with RegisterStagedFrame as above.  Same poses again.  Not with --host-stamps or --pageable.
// --publish (KSEQ2 and KSEQ3, staged) also builds, for every frame, the three clouds an online node publishes when it has subscribers
// (LidarOdometryServer::PublishClouds, LidarOdometryServer.cpp:240-263: frame, keypoints, local map, each as EigenToPointCloud2's
// float32 records): `host` the reference's way, RegisterStagedFrame + LocalMap() + the narrowing loop of EigenToPointCloud2
// (RosUtils.cpp:41-63) restated below; `device` with RegisterStagedFramePointCloud2 + LocalMapPointCloud2, narrowed on the device;
// `live` as `device` for the frame and keypoints, and the local map through LocalMapPointCloud2Live, which writes only the records
// that changed since the previous frame into the map's own buffer (the JSON line then reports the records written per frame).  The
// JSON line reports the wall time of the local map's publication alone (the map step of the three, inside the frame loop) per frame.
// --publish-digest FILE writes one line per frame: a 64-bit FNV-1a hash over the bytes of the three clouds' data, in that order; the
// local map's records are hashed in sorted order, because the map's Pointcloud() order (its voxels' creation order on the device)
// may differ from run to run while its content does not.  The hashing is host work inside the timed loop: time without it.
// --downsample-order 1 sets the default context's option "downsample_order" (kicp.h): both down-samples of every frame emit the
// KISS-ICP robin_map order instead of the order of first occurrence (as KICP_DOWNSAMPLE_ORDER does for any facade program).
// --correspondences FILE switches on the default context's option "correspondences" (kicp.h; KinematicICP::SetCorrespondences) and
// writes one CSV line per frame of the last repetition, how well that frame registered (KinematicICP::LastCorrespondenceStats: its
// registration source at the returned pose against the local map before the frame's update):
//   stamp, n_points, n_inliers, fitness, inlier_rmse, JTJ00, JTJ01, JTJ11, JTr0, JTr1
// the stamp as in the TUM file, the doubles with 17 significant digits (they read back to the same bits), no header line.
// --map-update sets the default context's map-update policy (kicp.h kicp_ctx_set_map_update; KinematicICP::SetMapUpdate): always (the
// reference's Update after every frame, default), never (register every frame against the map as it is) or gated (update only when
// the frame's correspondence report passes --min-inliers k (default 0), --min-fitness f (default 0) and --max-inlier-rmse r (default
// inf), which are accepted only with gated).  --load-map FILE loads a map file (kicp/map_file.hpp, written by --save-map) into the
// pipeline's map before the first frame of every repetition; its voxel size and max_points_per_voxel must be the replay's.  The drive
// must start where the map's run started: the pipeline's start pose is the drive's.  --save-map FILE writes the map after the last
// repetition.  "Map once, localise later" is a --save-map run, then --load-map with --map-update never.  With any of these options
// the JSON line also reports the policy ("map_update") and how many frames of the last repetition had each outcome
// ("map_update_outcomes", KinematicICP::LastMapUpdate); without them the line is as before.  --freeze-prior (only with --load-map)
// freezes the loaded map (kicp_map_freeze): its voxels are never evicted or written into, and the frames' Updates build a live layer
// beside it.  "Localise on a prior map that keeps learning" is --load-map FILE --freeze-prior --map-update always (or gated).  The JSON
// line then also reports the prior's and the live layer's voxel and point counts at the end of the last repetition ("prior_voxels",
// "prior_points", "live_voxels", "live_points").
// --free-space M[,E] switches on free-space clearing in the frame path of the default context (kicp.h kicp_ctx_set_free_space;
// KinematicICP::SetFreeSpace) with min_misses M (>= 1) and end_margin E metres (default 0.5): after every applied Update the frame's
// down-sampled points clear the live voxels their rays pass through.  The JSON line then reports "free_space" {min_misses,
// end_margin} and the statistics summed over the last repetition's frames ("free_space_stats": rays, visits, cleared_voxels,
// cleared_points, prior_contradicted).  A multi-sensor (KSEQ3 with several slots) drive is refused with it.
// --occupancy I,G,L,M (needs --free-space) keeps occupancy evidence in the pipeline's map (kicp.h kicp_map_set_occupancy, set through
// KinematicICP::VoxelMap() after the map is loaded): initial I, hit_gain G, miss_loss L, max_evidence M.  The JSON line then reports
// "occupancy" {initial, hit_gain, miss_loss, max_evidence, voxels, evidence_sum}: the setting, and the map's voxel count and summed
// evidence at the end of the last repetition.
//
// Version 3, magic "KSEQ3\0\0\0", carries several message streams ("slots", 1..KICP_MAX_SENSORS: PointCloud2 records or 2D LaserScans,
// each with its extrinsic) and the wheel odometry either as one relative motion or as poses sampled during the sweep:
//   char magic[8]; int32 n_frames; int32 n_slots; double start_pose[7];
//   per slot:  int32 kind (0 = PointCloud2 records, 1 = LaserScan); int32 stamps_relative; double lidar_to_base[7]
//   per frame: double relative_odometry[7]; int32 n_samples; int32 reserved;
//              n_samples x { double stamp; double pose[7] }   (the base pose in the odometry frame, on the odometry clock)
//              per slot, in slot order, one message (it may be empty):
//                kind 0: int32 n_points, point_step, offset_x, offset_y, offset_z, stamp_datatype, stamp_offset, reserved;
//                        double header_stamp; uint8 records[n_points * point_step]          (the fields as in version 2)
//                kind 1: int32 n_beams, reserved; double header_stamp;
//                        float angle_min, angle_max, angle_increment, time_increment, range_min, range_max; float ranges[n_beams]
// A records slot with stamps_relative 0 has absolute stamps (time_offset 0), with 1 stamps relative to its header (an Ouster `t`,
// time_offset header_stamp); a LaserScan's offset is always its header stamp (kicp::SensorFrame).  Two slots may share an extrinsic
// (two scans of a 25 Hz scanner against one 10 Hz sweep).  A frame is replayed as an online node runs one: one slot through
// StageFrame / StageLaserScan (StageDevice* with --device-input) and RegisterStagedFrame, so that a one-slot drive is bit for bit the
// version-2 drive of the same records; several through StageSensors and RegisterStagedSensors with the slots' extrinsics.
// relative_odometry is T(begin)^-1 T(end) over the frame's sweep and keeps its role in the motion model and the threshold; n_samples 0
// de-skews with it as one motion, otherwise the frame is de-skewed along the samples (the overloads taking kicp::OdometrySample), which
// must cover the sweep the staging call returns (kicp/deskew_segments.hpp); a frame whose samples do not is an error.  The first sweep
// begins at the earliest header stamp of the first frame, where the online node starts (LidarOdometryServer.cpp:182), and each TUM
// line carries the end of its frame's sweep (offline_node.cpp:143-145), where versions 1 and 2 write the header stamp.  The file is
// validated as a whole before the replay starts (kicp/kseq.hpp).  --host-stamps does not apply (there is no host-stamp call for
// several sensors); the JSON line adds the slot kinds and the odometry samples per frame.
//
// Prints one JSON line with the frame rate; exits non-zero on any error (no CUDA
// device included: there is no CPU fallback).
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

#include "kicp/facade_pipeline.hpp"
#include "kicp/kseq.hpp"
#include "kicp/map_file.hpp"
#include "kicp/runtime.hpp"
#include "kicp/tum.hpp"

namespace {
struct Frame {
    int32_t n = 0, has_stamps = 0;
    double header_stamp = 0.0;
    double odom[7];
    float *xyz = nullptr;      // n * 3, page-locked unless --pageable
    double *stamps = nullptr;  // n
    kicp::PointCloud2View msg;  // KSEQ2: the records (page-locked unless --pageable) and their fields
    kicp::PointCloud2View device_msg;  // --device-input: msg with its records in device memory
};

void cuda_check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void *host_alloc(size_t bytes, bool pinned) {
    if (bytes == 0) bytes = 8;
    void *p = nullptr;
    if (pinned) {
        kicp::check(kicp_host_alloc((uint64_t)bytes, &p), "kicp_host_alloc");
    } else {
        p = std::malloc(bytes);
        if (!p) throw std::runtime_error("out of host memory");
    }
    return p;
}

// EigenToPointCloud2's loop (RosUtils.cpp:41-63): every coordinate narrowed with static_cast<float> into x/y/z at 0/4/8, point_step 12
kicp::PointCloud2Data eigen_to_pointcloud2(const std::vector<Eigen::Vector3d> &points) {
    kicp::PointCloud2Data m;
    m.resize(points.size());
    uint8_t *d = m.data.data();
    for (const Eigen::Vector3d &p : points) {
        const float xyz[3] = {static_cast<float>(p.x()), static_cast<float>(p.y()), static_cast<float>(p.z())};
        std::memcpy(d, xyz, 12);
        d += 12;
    }
    return m;
}

// 64-bit FNV-1a, continued from `h`
uint64_t fnv1a(const std::vector<uint8_t> &bytes, uint64_t h) {
    for (const uint8_t b : bytes) h = (h ^ b) * 0x100000001B3ull;
    return h;
}
// the 12-byte records of a message in lexicographic byte order
std::vector<uint8_t> sorted_records(const std::vector<uint8_t> &bytes) {
    std::vector<std::array<uint8_t, 12>> r(bytes.size() / 12);
    if (!r.empty()) std::memcpy(r.data(), bytes.data(), r.size() * 12);
    std::sort(r.begin(), r.end());
    std::vector<uint8_t> out(r.size() * 12);
    if (!r.empty()) std::memcpy(out.data(), r.data(), out.size());
    return out;
}

template <class T>
void read_exact(std::FILE *f, T *dst, size_t count, const char *what) {
    if (std::fread(dst, sizeof(T), count, f) != count) throw std::runtime_error(std::string("truncated .kseq file while reading ") + what);
}

// a version-1 or version-2 drive: the frames into buffers of host_alloc; returns true for version 2
bool read_kseq12(const char *path, bool pinned, double l2b[7], double start[7], std::vector<Frame> &frames, int64_t &total_points) {
    std::FILE *f = std::fopen(path, "rb");
    if (!f) throw std::runtime_error(std::string("cannot open ") + path);
    char magic[8];
    read_exact(f, magic, 8, "the header");
    const bool v2 = std::memcmp(magic, "KSEQ2\0\0\0", 8) == 0;
    if (!v2 && std::memcmp(magic, "KSEQ1\0\0\0", 8) != 0) throw std::runtime_error("not a .kseq file (bad magic)");
    int32_t n_frames = 0, reserved = 0;
    read_exact(f, &n_frames, 1, "the header"), read_exact(f, &reserved, 1, "the header");
    read_exact(f, l2b, 7, "lidar_to_base"), read_exact(f, start, 7, "the start pose");
    if (n_frames < 0 || n_frames > (1 << 24)) throw std::runtime_error("implausible frame count");
    frames.resize((size_t)n_frames);
    for (auto &fr : frames) {
        if (v2) {
            int32_t h[8];  // n, point_step, offset_x, offset_y, offset_z, stamp_datatype, stamp_offset, reserved
            read_exact(f, h, 8, "a frame header");
            read_exact(f, &fr.header_stamp, 1, "a frame header"), read_exact(f, fr.odom, 7, "a frame header");
            if (h[0] < 0 || h[1] <= 0) throw std::runtime_error("bad point count or point_step");
            fr.n = h[0];
            const size_t bytes = (size_t)h[0] * (size_t)h[1];
            uint8_t *raw = static_cast<uint8_t *>(host_alloc(bytes, pinned));
            read_exact(f, raw, bytes, "records");
            fr.msg.data = raw, fr.msg.width = (uint32_t)h[0], fr.msg.height = 1, fr.msg.point_step = (uint32_t)h[1];
            fr.msg.fields = {{"x", (uint32_t)h[2], kicp::PF_FLOAT32, 1}, {"y", (uint32_t)h[3], kicp::PF_FLOAT32, 1},
                             {"z", (uint32_t)h[4], kicp::PF_FLOAT32, 1}};
            if (h[5] != 0) fr.msg.fields.push_back({"t", (uint32_t)h[6], (uint8_t)h[5], 1});
            total_points += fr.n;
            continue;
        }
        read_exact(f, &fr.n, 1, "a frame header"), read_exact(f, &fr.has_stamps, 1, "a frame header");
        read_exact(f, &fr.header_stamp, 1, "a frame header"), read_exact(f, fr.odom, 7, "a frame header");
        if (fr.n < 0) throw std::runtime_error("negative point count");
        fr.xyz = static_cast<float *>(host_alloc((size_t)fr.n * 3 * sizeof(float), pinned));
        read_exact(f, fr.xyz, (size_t)fr.n * 3, "points");
        if (fr.has_stamps) {
            fr.stamps = static_cast<double *>(host_alloc((size_t)fr.n * sizeof(double), pinned));
            read_exact(f, fr.stamps, (size_t)fr.n, "stamps");
        }
        total_points += fr.n;
    }
    std::fclose(f);
    return v2;
}

// the .kseq version of the file at `path` (kicp::kseq_version), 0 when it cannot be read
int peek_version(const char *path) {
    char magic[8];
    std::FILE *f = std::fopen(path, "rb");
    if (!f) return 0;
    const bool ok = std::fread(magic, 1, 8, f) == 8;
    std::fclose(f);
    return ok ? kicp::kseq_version(magic) : 0;
}

// the points a staging call stages for a message: every record, or the beams projectLaser keeps (range_min <= r < range_max)
int64_t staged_points(const kicp::SensorFrame &s) {
    if (s.kind == kicp::SensorFrame::Kind::PointCloud2) return static_cast<int64_t>(s.cloud.num_points());
    int64_t n = 0;
    for (size_t i = 0; i < s.scan.n; ++i) n += s.scan.ranges[i] < s.scan.range_max && s.scan.ranges[i] >= s.scan.range_min;
    return n;
}
}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) {
        std::fprintf(stderr, "usage: %s drive.kseq out.tum [--deskew 0|1] [--voxel-size v] [--max-range r] [--min-range r] [--repeat k] [--pageable] "
                     "[--host-stamps] [--device-input] [--publish host|device|live] [--publish-digest FILE] [--downsample-order 0|1] "
                     "[--correspondences FILE] [--map-update always|never|gated] [--min-inliers k] [--min-fitness f] [--max-inlier-rmse r] "
                     "[--load-map FILE] [--freeze-prior] [--save-map FILE] [--free-space M[,E]] [--occupancy I,G,L,M]\n", argv[0]);
        return 2;
    }
    kinematic_icp::pipeline::Config config;  // the reference's defaults (pipeline/KinematicICP.hpp:38-60)
    config.deskew = true;
    int repeat = 1;
    bool pinned = true, host_stamps = false, device_input = false;
    std::string publish = "none", digest_path, corr_path;
    int downsample_order = -1;  // -1: leave the default context's option as it is
    std::string map_update = "always", load_map_path, save_map_path;
    kicp_map_update_policy policy{KICP_MAP_UPDATE_ALWAYS, 0, 0.0, HUGE_VAL};
    bool freeze_prior = false;  // --freeze-prior: freeze the map --load-map loaded
    kicp_free_space_params free_space{0.5, 0};  // --free-space M[,E]; min_misses 0: off
    bool occupancy = false;  // --occupancy I,G,L,M
    kicp_occupancy_params occ{0, 0, 0, 0};
    bool thresholds = false;  // a --min-* / --max-inlier-rmse option was given (only with --map-update gated)
    bool map_options = false;  // any of --map-update, the thresholds, --load-map, --save-map: the JSON line reports the outcomes
    for (int i = 3; i < argc; ++i) {
        const std::string a = argv[i];
        auto value = [&](const char *name) -> const char * {
            if (i + 1 >= argc) throw std::runtime_error(std::string("missing value for ") + name);
            return argv[++i];
        };
        try {
            if (a == "--deskew") config.deskew = std::atoi(value("--deskew")) != 0;
            else if (a == "--voxel-size") config.voxel_size = std::atof(value("--voxel-size"));
            else if (a == "--max-range") config.max_range = std::atof(value("--max-range"));
            else if (a == "--min-range") config.min_range = std::atof(value("--min-range"));
            else if (a == "--repeat") repeat = std::max(1, std::atoi(value("--repeat")));
            else if (a == "--pageable") pinned = false;
            else if (a == "--host-stamps") host_stamps = true;
            else if (a == "--device-input") device_input = true;
            else if (a == "--publish") publish = value("--publish");
            else if (a == "--publish-digest") digest_path = value("--publish-digest");
            else if (a == "--correspondences") corr_path = value("--correspondences");
            else if (a == "--map-update") map_update = value("--map-update"), map_options = true;
            else if (a == "--min-inliers") policy.min_inliers = std::atoll(value("--min-inliers")), thresholds = true;
            else if (a == "--min-fitness") policy.min_fitness = std::atof(value("--min-fitness")), thresholds = true;
            else if (a == "--max-inlier-rmse") policy.max_inlier_rmse = std::atof(value("--max-inlier-rmse")), thresholds = true;
            else if (a == "--load-map") load_map_path = value("--load-map"), map_options = true;
            else if (a == "--save-map") save_map_path = value("--save-map"), map_options = true;
            else if (a == "--freeze-prior") freeze_prior = true, map_options = true;
            else if (a == "--free-space") {
                const std::string v = value("--free-space");
                const size_t comma = v.find(',');
                char *end = nullptr;
                const long mm = std::strtol(v.c_str(), &end, 10);
                if (end == v.c_str() || (comma == std::string::npos ? *end != '\0' : end != v.c_str() + comma) || mm < 1 || mm > INT32_MAX)
                    throw std::runtime_error("--free-space takes M[,E]: min_misses M >= 1, end_margin E >= 0 metres");
                free_space.min_misses = (int32_t)mm;
                if (comma != std::string::npos) {
                    const std::string e = v.substr(comma + 1);
                    free_space.end_margin = std::strtod(e.c_str(), &end);
                    if (e.empty() || *end != '\0' || !(free_space.end_margin >= 0.0) || std::isinf(free_space.end_margin))
                        throw std::runtime_error("--free-space takes M[,E]: min_misses M >= 1, end_margin E >= 0 metres");
                }
            }
            else if (a == "--occupancy") {
                const std::string v = value("--occupancy");
                int32_t f[4];
                const char *q = v.c_str();
                for (int k = 0; k < 4; ++k) {
                    char *end = nullptr;
                    const long x = std::strtol(q, &end, 10);
                    if (end == q || x < INT32_MIN || x > INT32_MAX || *end != (k < 3 ? ',' : '\0'))
                        throw std::runtime_error("--occupancy takes I,G,L,M: initial, hit_gain, miss_loss, max_evidence (integers)");
                    f[k] = (int32_t)x, q = end + 1;
                }
                occ = kicp_occupancy_params{f[0], f[1], f[2], f[3]}, occupancy = true;
            }
            else if (a == "--downsample-order") {
                const std::string v = value("--downsample-order");
                if (v != "0" && v != "1") throw std::runtime_error("--downsample-order takes 0 or 1");
                downsample_order = v == "1" ? 1 : 0;
            }
            else throw std::runtime_error("unknown option " + a);
        } catch (const std::exception &e) {
            std::fprintf(stderr, "kicp_replay: %s\n", e.what());
            return 2;
        }
    }
    if (map_update != "always" && map_update != "never" && map_update != "gated") {
        std::fprintf(stderr, "kicp_replay: --map-update takes always, never or gated\n");
        return 2;
    }
    if (thresholds && map_update != "gated") {
        std::fprintf(stderr, "kicp_replay: --min-inliers, --min-fitness and --max-inlier-rmse need --map-update gated\n");
        return 2;
    }
    if (freeze_prior && load_map_path.empty()) {
        std::fprintf(stderr, "kicp_replay: --freeze-prior freezes the map --load-map loads: it needs --load-map\n");
        return 2;
    }
    if (occupancy && free_space.min_misses == 0) {
        std::fprintf(stderr, "kicp_replay: --occupancy keeps evidence across the frames' free-space clearing: it needs --free-space\n");
        return 2;
    }
    map_options = map_options || thresholds;
    policy.mode = map_update == "never" ? KICP_MAP_UPDATE_NEVER : map_update == "gated" ? KICP_MAP_UPDATE_GATED : KICP_MAP_UPDATE_ALWAYS;
    if (publish != "none" && publish != "host" && publish != "device" && publish != "live") {
        std::fprintf(stderr, "kicp_replay: --publish takes host, device or live\n");
        return 2;
    }
    if (device_input && (host_stamps || !pinned)) {
        std::fprintf(stderr, "kicp_replay: --device-input stages from device memory: not with --host-stamps or --pageable\n");
        return 2;
    }
    if (!digest_path.empty() && publish == "none") {
        std::fprintf(stderr, "kicp_replay: --publish-digest needs --publish\n");
        return 2;
    }
    const bool v3 = peek_version(argv[1]) == 3;  // other files: read (and refused) below
    if (v3 && host_stamps) {
        std::fprintf(stderr, "kicp_replay: --host-stamps replays a KSEQ2 drive; a KSEQ3 drive is always staged (there is no host-stamp "
                     "call for several sensors)\n");
        return 2;
    }
    try {
        kicp::default_context();  // fails here, loudly, without a CUDA device
        if (downsample_order >= 0)
            kicp::check(kicp_ctx_set_option(kicp::default_context(), "downsample_order", downsample_order), "--downsample-order");
        if (!corr_path.empty()) kinematic_icp::pipeline::KinematicICP::SetCorrespondences(true);
        if (map_options) kinematic_icp::pipeline::KinematicICP::SetMapUpdate(policy);  // a threshold out of range throws, naming the field
        if (free_space.min_misses > 0) kinematic_icp::pipeline::KinematicICP::SetFreeSpace(free_space.min_misses, free_space.end_margin);
        kicp::MapFile prior;  // --load-map
        if (!load_map_path.empty()) {
            prior = kicp::read_map_file(load_map_path);
            if (prior.voxel_size != config.voxel_size || prior.max_points_per_voxel != config.max_points_per_voxel)
                throw std::runtime_error(load_map_path + ": voxel size " + std::to_string(prior.voxel_size) + " and max_points_per_voxel " +
                                         std::to_string(prior.max_points_per_voxel) + " differ from the replay's " +
                                         std::to_string(config.voxel_size) + " and " + std::to_string(config.max_points_per_voxel));
        }
        bool v2 = false;
        double l2b[7], start[7];
        std::vector<Frame> frames;  // KSEQ1 / KSEQ2
        kicp::Kseq3Drive drive;     // KSEQ3
        int64_t total_points = 0;
        if (v3) {
            drive = kicp::read_kseq3(argv[1], [&](size_t bytes) { return host_alloc(bytes, pinned); });
            std::memcpy(start, drive.start_pose, sizeof(start));
            for (const auto &fr : drive.frames)
                for (const auto &s : fr.sensors) total_points += staged_points(s);
        } else {
            v2 = read_kseq12(argv[1], pinned, l2b, start, frames, total_points);
        }
        const int32_t n_frames = static_cast<int32_t>(v3 ? drive.frames.size() : frames.size());
        if (publish != "none" && ((!v2 && !v3) || host_stamps))
            throw std::runtime_error("--publish replays a KSEQ2 or KSEQ3 drive staged (without --host-stamps)");
        if (device_input && !v2 && !v3) throw std::runtime_error("--device-input replays a KSEQ2 or KSEQ3 drive");
        // --device-input: every frame's records (KSEQ3: every message's records or ranges), as a GPU producer would leave them, on the
        // default context's device (current since kicp::default_context() created it)
        std::vector<void *> device_records;
        auto to_device = [&](const void *src, size_t bytes) {
            void *d = nullptr;
            cuda_check(cudaMalloc(&d, std::max<size_t>(bytes, 1)), "cudaMalloc");
            device_records.push_back(d);
            cuda_check(cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice), "cudaMemcpy");
            return d;
        };
        for (auto &fr : frames) {
            if (!device_input) break;
            fr.device_msg = fr.msg;
            fr.device_msg.data = static_cast<const uint8_t *>(to_device(fr.msg.data, fr.msg.num_points() * fr.msg.point_step));
        }
        std::vector<std::vector<kicp::SensorFrame>> device_sensors;  // KSEQ3 --device-input: per frame, the messages in device memory
        for (const auto &fr : drive.frames) {
            if (!device_input) break;
            device_sensors.push_back(fr.sensors);
            for (auto &s : device_sensors.back()) {
                s.device = true;
                if (s.kind == kicp::SensorFrame::Kind::LaserScan)
                    s.scan.ranges = static_cast<const float *>(to_device(s.scan.ranges, s.scan.n * sizeof(float)));
                else
                    s.cloud.data = static_cast<const uint8_t *>(to_device(s.cloud.data, s.cloud.num_points() * s.cloud.point_step));
            }
        }
        // KSEQ3: the slots' extrinsics, every frame's odometry and samples, as the facade takes them
        std::vector<Sophus::SE3d> lidar_to_bases;
        for (const auto &slot : drive.slots) lidar_to_bases.push_back(kicp::from_pose7(slot.lidar_to_base));
        std::vector<Sophus::SE3d> odoms;
        std::vector<std::vector<kicp::OdometrySample>> samples(drive.frames.size());
        int64_t total_samples = 0;
        for (size_t k = 0; k < drive.frames.size(); ++k) {
            odoms.push_back(kicp::from_pose7(drive.frames[k].relative_odometry));
            for (const auto &s : drive.frames[k].samples) samples[k].push_back({s.stamp, kicp::from_pose7(s.pose)});
            total_samples += static_cast<int64_t>(samples[k].size());
        }
        double first_header = 0.0;  // KSEQ3: where the first sweep begins, the earliest header stamp of the first frame
        for (size_t s = 0; !drive.frames.empty() && s < drive.slots.size(); ++s)
            first_header = s ? std::min(first_header, drive.frames[0].sensors[s].header_stamp) : drive.frames[0].sensors[0].header_stamp;

        const Sophus::SE3d lidar_to_base = v3 ? Sophus::SE3d() : kicp::from_pose7(l2b);
        std::vector<std::pair<double, Sophus::SE3d>> poses;
        double seconds = 0.0;
        std::vector<uint64_t> digests;
        std::vector<kicp_corr_stats> corr;  // --correspondences: every frame's report, in frame order (last repetition)
        int64_t map_points = 0;  // the local map's size after the last frame
        int64_t map_voxels = 0, prior_voxels = 0, prior_points = 0;  // --freeze-prior: the layers after the last repetition
        int64_t live_written = 0, live_records = 0;  // --publish live, last repetition: records written, and published, over all frames
        double map_seconds = 0.0;  // --publish, last repetition: time spent publishing the local map
        int64_t outcomes[KICP_FRAME_UPDATE_NONE + 1] = {};  // frames of the last repetition per KICP_FRAME_UPDATE_* outcome
        kicp_free_space_stats free_sum{};  // --free-space: the statistics summed over the last repetition's frames
        int64_t occ_voxels = 0, occ_sum = 0;  // --occupancy: the map's voxels and summed evidence after the last repetition
        std::vector<double> rep_seconds;  // every repetition's wall time (a 24-frame drive lasts milliseconds: one hiccup halves a single figure)
        for (int rep = 0; rep < repeat; ++rep) {  // --repeat: the same drive again on a fresh pipeline (the last run is the one written)
            kinematic_icp::pipeline::KinematicICP pipeline(config);
            pipeline.SetPose(kicp::from_pose7(start));  // (clears the map: the prior map is loaded after it)
            if (!load_map_path.empty())
                kicp::check(kicp_map_load_voxels(pipeline.VoxelMap().handle_, prior.keys.data(), prior.counts.data(), prior.points.data(),
                                                 prior.num_voxels()),
                            "kicp_map_load_voxels");
            if (freeze_prior) kicp::check(kicp_map_freeze(pipeline.VoxelMap().handle_), "kicp_map_freeze");
            if (occupancy) pipeline.VoxelMap().SetOccupancy(&occ);  // a field out of range throws, naming it
            for (int64_t &o : outcomes) o = 0;
            free_sum = kicp_free_space_stats{};
            poses.clear();
            poses.reserve((size_t)n_frames);
            digests.clear();
            corr.clear();
            // after every frame: its pose with the stamp the TUM file carries, and with --correspondences its report
            auto frame_done = [&](double stamp) {
                poses.emplace_back(stamp, pipeline.pose());
                if (!corr_path.empty()) corr.push_back(pipeline.LastCorrespondenceStats());
                ++outcomes[pipeline.LastMapUpdate()];
                if (free_space.min_misses > 0) {
                    const kicp_free_space_stats f = pipeline.LastFreeSpace();
                    free_sum.rays += f.rays, free_sum.visits += f.visits, free_sum.cleared_voxels += f.cleared_voxels;
                    free_sum.cleared_points += f.cleared_points, free_sum.prior_contradicted += f.prior_contradicted;
                }
            };
            live_written = live_records = 0;
            map_seconds = 0.0;
            double last_processed = v3 ? first_header : 0.0;  // end of the previous sweep (TimeStampHandler's state)
            // the staged frame's registration and, with --publish, the three clouds an online node publishes: reg() registers it as
            // RegisterStagedFrame* does, reg_pc2() as RegisterStagedFramePointCloud2 does
            auto register_staged = [&](auto &&reg, auto &&reg_pc2) {
                if (publish == "none") {
                    reg();
                    return;
                }
                kicp::PointCloud2Data frame_msg, keypoints_msg, map_msg;
                if (publish == "host") {
                    const auto [frame, keypoints] = reg();
                    frame_msg = eigen_to_pointcloud2(frame), keypoints_msg = eigen_to_pointcloud2(keypoints);
                    const auto m0 = std::chrono::steady_clock::now();
                    map_msg = eigen_to_pointcloud2(pipeline.LocalMap());
                    map_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - m0).count();
                } else if (publish == "device") {
                    std::tie(frame_msg, keypoints_msg) = reg_pc2();
                    const auto m0 = std::chrono::steady_clock::now();
                    map_msg = pipeline.LocalMapPointCloud2();
                    map_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - m0).count();
                } else {
                    std::tie(frame_msg, keypoints_msg) = reg_pc2();
                    const auto m0 = std::chrono::steady_clock::now();
                    const auto [view, stats] = pipeline.LocalMapPointCloud2Live();
                    map_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - m0).count();
                    live_written += stats.written, live_records += view.width;
                    if (!digest_path.empty()) map_msg.data.assign(view.data, view.data + 12 * (size_t)view.width);  // hashing only
                }
                if (!digest_path.empty())
                    digests.push_back(fnv1a(sorted_records(map_msg.data), fnv1a(keypoints_msg.data, fnv1a(frame_msg.data, 0xCBF29CE484222325ull))));
            };
            const auto t0 = std::chrono::steady_clock::now();
            for (size_t k = 0; v3 && k < drive.frames.size(); ++k) {
                const std::vector<kicp::SensorFrame> &sensors = device_input ? device_sensors[k] : drive.frames[k].sensors;
                const std::vector<kicp::OdometrySample> &smp = samples[k];
                const Sophus::SE3d &odom = odoms[k];
                try {
                    if (sensors.size() == 1) {  // the single-sensor calls: bit for bit the KSEQ2 replay of the same records
                        const kicp::SensorFrame &s = sensors[0];
                        if (s.kind == kicp::SensorFrame::Kind::LaserScan)
                            device_input ? pipeline.StageDeviceLaserScan(s.scan, s.header_stamp, last_processed)
                                         : pipeline.StageLaserScan(s.scan, s.header_stamp, last_processed);
                        else
                            device_input ? pipeline.StageDeviceFrame(s.cloud, s.header_stamp, last_processed)
                                         : pipeline.StageFrame(s.cloud, s.header_stamp, last_processed);
                        register_staged(
                            [&] { return smp.empty() ? pipeline.RegisterStagedFrame(lidar_to_bases[0], odom)
                                                     : pipeline.RegisterStagedFrame(lidar_to_bases[0], odom, smp); },
                            [&] { return smp.empty() ? pipeline.RegisterStagedFramePointCloud2(lidar_to_bases[0], odom)
                                                     : pipeline.RegisterStagedFramePointCloud2(lidar_to_bases[0], odom, smp); });
                    } else {
                        pipeline.StageSensors(sensors, last_processed);
                        register_staged(
                            [&] { return smp.empty() ? pipeline.RegisterStagedSensors(lidar_to_bases, odom)
                                                     : pipeline.RegisterStagedSensors(lidar_to_bases, odom, smp); },
                            [&] { return smp.empty() ? pipeline.RegisterStagedSensorsPointCloud2(lidar_to_bases, odom)
                                                     : pipeline.RegisterStagedSensorsPointCloud2(lidar_to_bases, odom, smp); });
                    }
                } catch (const std::exception &e) {
                    throw std::runtime_error("frame " + std::to_string(k) + ": " + e.what());
                }
                frame_done(last_processed);  // the end of the sweep, as the offline node stamps its poses
            }
            for (const auto &fr : frames) {
                if (v2 && host_stamps) {
                    std::vector<double> stamps = kicp::extract_timestamps(fr.msg);
                    kicp::process_timestamps(stamps, fr.header_stamp, last_processed);
                    kicp_frame_input in = kicp::make_frame_input(fr.msg);
                    in.stamps = stamps.empty() ? nullptr : stamps.data(), in.n_stamps = (int64_t)stamps.size();
                    pipeline.RegisterFrame(in, lidar_to_base, kicp::from_pose7(fr.odom));
                    frame_done(fr.header_stamp);
                    continue;
                }
                if (v2) {
                    if (device_input)
                        pipeline.StageDeviceFrame(fr.device_msg, fr.header_stamp, last_processed);
                    else
                        pipeline.StageFrame(fr.msg, fr.header_stamp, last_processed);  // the interval an online node looks the odometry up for
                    const Sophus::SE3d odom = kicp::from_pose7(fr.odom);
                    register_staged([&] { return pipeline.RegisterStagedFrame(lidar_to_base, odom); },
                                    [&] { return pipeline.RegisterStagedFramePointCloud2(lidar_to_base, odom); });
                    frame_done(fr.header_stamp);
                    continue;
                }
                kicp_frame_input in{};
                in.data = fr.xyz, in.n = fr.n, in.dtype = KICP_DTYPE_F32, in.point_step = 0;
                in.stamps = fr.has_stamps ? fr.stamps : nullptr, in.n_stamps = fr.has_stamps ? fr.n : 0;
                pipeline.RegisterFrame(in, lidar_to_base, kicp::from_pose7(fr.odom));
                frame_done(fr.header_stamp);
            }
            seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            rep_seconds.push_back(seconds);
            kicp::check(kicp_map_num_points(pipeline.VoxelMap().handle_, &map_points), "kicp_map_num_points");
            if (occupancy) {
                const std::vector<int32_t> ev = pipeline.VoxelMap().Occupancy();
                occ_voxels = (int64_t)ev.size(), occ_sum = 0;
                for (const int32_t e : ev) occ_sum += e;
            }
            if (freeze_prior) {
                kicp::check(kicp_map_prior_size(pipeline.VoxelMap().handle_, &prior_voxels, &prior_points), "kicp_map_prior_size");
                kicp::check(kicp_map_num_voxels(pipeline.VoxelMap().handle_, &map_voxels), "kicp_map_num_voxels");
            }
            if (!save_map_path.empty() && rep == repeat - 1) {  // the map after the last repetition, as kicp_map_export_voxels gives it
                kicp_map *h = pipeline.VoxelMap().handle_;
                kicp::MapFile out;
                out.voxel_size = config.voxel_size, out.max_points_per_voxel = config.max_points_per_voxel;
                int64_t nv = 0, np = 0;
                kicp::check(kicp_map_num_voxels(h, &nv), "kicp_map_num_voxels");
                out.keys.resize(3 * (size_t)nv), out.counts.resize((size_t)nv), out.points.resize(3 * (size_t)map_points);
                kicp::check(kicp_map_export_voxels(h, out.keys.data(), out.counts.data(), out.points.data(), nv, map_points, &nv, &np),
                            "kicp_map_export_voxels");
                kicp::write_map_file(save_map_path, out);
            }
        }
        // the fastest repetition after the first (which also pays for allocations); the last one stays the headline of this line
        double best = seconds;
        for (size_t k = rep_seconds.size() > 1 ? 1 : 0; k < rep_seconds.size(); ++k) best = std::min(best, rep_seconds[k]);
        std::string reps = "[";
        for (size_t k = 0; k < rep_seconds.size(); ++k) {
            char buf[32];
            std::snprintf(buf, sizeof(buf), "%s%.6f", k ? ", " : "", rep_seconds[k]);
            reps += buf;
        }
        reps += "]";
        for (void *d : device_records) cuda_check(cudaFree(d), "cudaFree");
        if (!kicp::write_poses_tum(argv[2], poses)) throw std::runtime_error(std::string("cannot write ") + argv[2]);
        if (!digest_path.empty()) {
            std::FILE *d = std::fopen(digest_path.c_str(), "w");
            if (!d) throw std::runtime_error("cannot write " + digest_path);
            for (const uint64_t h : digests) std::fprintf(d, "%016llx\n", (unsigned long long)h);
            if (std::fclose(d) != 0) throw std::runtime_error("cannot write " + digest_path);
        }
        if (!corr_path.empty()) {
            std::FILE *c = std::fopen(corr_path.c_str(), "w");
            if (!c) throw std::runtime_error("cannot write " + corr_path);
            for (size_t k = 0; k < corr.size(); ++k) {
                const kicp_corr_stats &st = corr[k];
                std::fprintf(c, "%.17g,%lld,%lld,%.17g,%.17g,%.17g,%.17g,%.17g,%.17g,%.17g\n", poses[k].first, (long long)st.n_points,
                             (long long)st.n_inliers, st.fitness, st.inlier_rmse, st.jtj[0], st.jtj[1], st.jtj[2], st.jtr[0], st.jtr[1]);
            }
            if (std::fclose(c) != 0) throw std::runtime_error("cannot write " + corr_path);
        }
        std::string live;
        if (publish != "none") {
            char buf[64];
            std::snprintf(buf, sizeof(buf), ", \"map_publish_ms_per_frame\": %.4f", n_frames ? 1e3 * map_seconds / n_frames : 0.0);
            live = buf;
        }
        if (publish == "live") {
            char buf[128];
            std::snprintf(buf, sizeof(buf), ", \"live_written_per_frame\": %.1f, \"live_map_records_per_frame\": %.1f",
                          n_frames ? (double)live_written / n_frames : 0.0, n_frames ? (double)live_records / n_frames : 0.0);
            live += buf;
        }
        if (map_options) {  // the map-update policy and the outcomes of the last repetition's frames
            char buf[256];
            std::snprintf(buf, sizeof(buf), ", \"map_update\": \"%s\", \"map_update_outcomes\": {\"applied\": %lld, \"no_correspondences\": %lld, "
                          "\"rejected\": %lld, \"skipped\": %lld, \"none\": %lld}", map_update.c_str(),
                          (long long)outcomes[KICP_FRAME_UPDATE_APPLIED], (long long)outcomes[KICP_FRAME_UPDATE_NO_CORRESPONDENCES],
                          (long long)outcomes[KICP_FRAME_UPDATE_REJECTED], (long long)outcomes[KICP_FRAME_UPDATE_SKIPPED],
                          (long long)outcomes[KICP_FRAME_UPDATE_NONE]);
            live += buf;
            if (freeze_prior) {
                std::snprintf(buf, sizeof(buf), ", \"prior_voxels\": %lld, \"prior_points\": %lld, \"live_voxels\": %lld, \"live_points\": %lld",
                              (long long)prior_voxels, (long long)prior_points, (long long)(map_voxels - prior_voxels),
                              (long long)(map_points - prior_points));
                live += buf;
            }
        }
        if (free_space.min_misses > 0) {  // the free-space setting and its statistics over the last repetition's frames
            char buf[384];
            std::snprintf(buf, sizeof(buf), ", \"free_space\": {\"min_misses\": %d, \"end_margin\": %.17g}, \"free_space_stats\": {\"rays\": %lld, "
                          "\"visits\": %lld, \"cleared_voxels\": %lld, \"cleared_points\": %lld, \"prior_contradicted\": %lld}",
                          (int)free_space.min_misses, free_space.end_margin, (long long)free_sum.rays, (long long)free_sum.visits,
                          (long long)free_sum.cleared_voxels, (long long)free_sum.cleared_points, (long long)free_sum.prior_contradicted);
            live += buf;
        }
        if (occupancy) {
            char buf[256];
            std::snprintf(buf, sizeof(buf), ", \"occupancy\": {\"initial\": %d, \"hit_gain\": %d, \"miss_loss\": %d, \"max_evidence\": %d, "
                          "\"voxels\": %lld, \"evidence_sum\": %lld}", (int)occ.initial, (int)occ.hit_gain, (int)occ.miss_loss,
                          (int)occ.max_evidence, (long long)occ_voxels, (long long)occ_sum);
            live += buf;
        }
        if (v3) {  // the slots, their kinds, and the odometry samples per frame (0: one motion per frame)
            live += ", \"slots\": " + std::to_string(drive.slots.size()) + ", \"slot_kinds\": [";
            for (size_t s = 0; s < drive.slots.size(); ++s)
                live += std::string(s ? ", " : "") + (drive.slots[s].kind == kicp::KseqSlot::LaserScan ? "\"laser_scan\"" : "\"records\"");
            char buf[64];
            std::snprintf(buf, sizeof(buf), "], \"odometry_samples_per_frame\": %.2f", n_frames ? (double)total_samples / n_frames : 0.0);
            live += buf;
        }
        std::printf("{\"harness\": \"kicp_replay\", \"frames\": %d, \"points_per_frame\": %.0f, \"seconds\": %.6f, \"frames_per_s\": %.2f, "
                    "\"ms_per_frame\": %.4f, \"frames_per_s_best\": %.2f, \"repetition_seconds\": %s, \"host_buffers\": \"%s %s\", "
                    "\"deskew\": %s, \"publish\": \"%s\"%s, \"map_points\": %lld, \"tum_file\": \"%s\"}\n",
                    n_frames, n_frames ? (double)total_points / n_frames : 0.0, seconds, seconds > 0 ? n_frames / seconds : 0.0,
                    n_frames ? 1e3 * seconds / n_frames : 0.0, best > 0 ? n_frames / best : 0.0, reps.c_str(), pinned ? "pinned" : "pageable",
                    !v2 && !v3 ? "float32" : host_stamps ? "records, host-decoded stamps" : device_input ? "records, staged from device memory" : "records, staged",
                    config.deskew ? "true" : "false", publish.c_str(), live.c_str(), (long long)map_points, argv[2]);
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "kicp_replay: %s\n", e.what());
        return 1;
    }
}
