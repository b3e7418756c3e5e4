// Device-side front end of KinematicICP::RegisterFrame (SURVEY.md §8(f)#2): the two operations the reference runs
// immediately before the hot path (pipeline/KinematicICP.cpp:38-44, 54-59), both from KISS-ICP v1.2.0:
//   kiss_icp::VoxelDownsample(frame, voxel_size)          first point (input order) of every voxel
//   kiss_icp::Preprocessor::Preprocess(frame, stamps, T)  de-skew p <- exp((s-1) log T) p, then keep min < |p| < max
// followed by the transform to the robot base frame.  Output order is the input order of the survivors (stable stream
// compaction — the library's own single-pass scan, kicp_scan.cuh, fused into the kernels that decide what survives), which is what
// the CPU restatement produces.  Compiled with -fmad=false like kicp_map.cu: voxel floors and
// range tests are evaluated in plain IEEE order.
#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "kicp_device.cuh"

using namespace kicp_dev;

#include "kicp_frontend_kernels.cuh"  // struct P3, IngestArgs, PreArgs and the kernels of this file
#include "kicp_downsample_order_kernels.cuh"  // option "downsample_order" 1: the robin_map order of the down-sample
#include "kicp_sensors_kernels.cuh"  // the multi-sensor frame: the common sweep window and the segmented Preprocess
#include "kicp_segments_kernels.cuh"  // the piecewise de-skew: per-sensor tables of constant-velocity segments
#include "kicp_map_update_kernels.cuh"  // the map-update policy: the rule and the gate of KICP_MAP_UPDATE_GATED
static_assert(kMaxSensors == KICP_MAX_SENSORS, "kicp_sensors_kernels.cuh and kicp.h disagree");
static_assert(kMaxDeskewSegments == KICP_MAX_DESKEW_SEGMENTS, "kicp_segments_kernels.cuh and kicp.h disagree");

// ------------------------------------------------------------------------------------------------------------ host
namespace {
// laser_geometry's cos / sin table: LaserProjection keeps one per projector (here: per context) and recomputes it only when the beam
// count, angle_min or angle_max differ from the cached ones, compared with != (a NaN angle_min always recomputes); a changed
// angle_increment alone reuses the old table.  It lives beside the scratch, not in it: a regrown scratch leaves it alone, as the
// projector outlives the buffers of its messages.  The device copy (d_cap beams) is uploaded after each recompute.
struct LaserTable {
    bool valid = false;
    int64_t n = 0;
    float angle_min = 0.0f, angle_max = 0.0f;
    std::vector<double2> cs;  // {cos, sin} of angle_min + i * angle_increment: the C library's, as the reference's x86-64 build computes it
    double2 *d_cs = nullptr;
    int64_t d_cap = 0;
    bool uploaded = false;
    // no exception may cross the C ABI: without host memory for the table it is left invalid (the next scan recomputes)
    int refresh(const kicp_laser_scan *scan, const char *where) {
        if (valid && n == scan->n && angle_min == scan->angle_min && angle_max == scan->angle_max) return KICP_OK;
        try {
            cs.resize((size_t)scan->n);
        } catch (const std::exception &) {
            valid = false, cs.clear(), cs.shrink_to_fit();
            kicp_set_error(std::string(where) + ": no host memory for the cos / sin table");
            return KICP_ERR_CAPACITY;
        }
        valid = true, n = scan->n, angle_min = scan->angle_min, angle_max = scan->angle_max;
        for (int64_t i = 0; i < n; ++i) {
            const double angle = (double)scan->angle_min + (double)i * (double)scan->angle_increment;
            cs[(size_t)i] = make_double2(std::cos(angle), std::sin(angle));
        }
        uploaded = false;
        return KICP_OK;
    }
    int upload(cudaStream_t stream) {
        if (uploaded) return KICP_OK;
        if (d_cap < n) {
            KICP_CUDA(cudaStreamSynchronize(stream));
            cudaFree(d_cs);
            d_cs = nullptr, d_cap = 0;
            KICP_CUDA(cudaMalloc(&d_cs, (size_t)n * sizeof(double2)));
            d_cap = n;
        }
        KICP_CUDA(cudaMemcpyAsync(d_cs, cs.data(), (size_t)n * sizeof(double2), cudaMemcpyHostToDevice, stream));
        uploaded = true;
        return KICP_OK;
    }
};

// The two clouds RegisterFrame returns (frame and source), staged in pinned host memory for cap points each: as doubles, and with
// KICP_STAGE_F32 as float32 records encoded on the device into d_rec (frame at 0, source at 3 cap; allocated on first use).  The
// counts are what kicp_frame_clouds / kicp_frame_clouds_f32 return.
struct Staging {
    P3 *frame = nullptr, *source = nullptr;
    float *d_rec = nullptr, *frame32 = nullptr, *source32 = nullptr;
    int64_t cap = 0;
    int64_t n_frame = 0, n_source = 0, n_frame32 = 0, n_source32 = 0;
    int reserve(int64_t points, bool records) {
        cap = points;
        if (!frame) KICP_CUDA(cudaMallocHost(&frame, cap * sizeof(P3)));
        if (!source) KICP_CUDA(cudaMallocHost(&source, cap * sizeof(P3)));
        if (!records) return KICP_OK;
        if (!d_rec) KICP_CUDA(cudaMalloc(&d_rec, (size_t)cap * 6 * sizeof(float)));
        if (!frame32) KICP_CUDA(cudaMallocHost(&frame32, (size_t)cap * 3 * sizeof(float)));
        if (!source32) KICP_CUDA(cudaMallocHost(&source32, (size_t)cap * 3 * sizeof(float)));
        return KICP_OK;
    }
    void release() { cudaFreeHost(frame), cudaFreeHost(source), cudaFree(d_rec), cudaFreeHost(frame32), cudaFreeHost(source32); }
    float *d_source_rec() const { return d_rec + 3 * cap; }
    // copies on `copy` of frame[0, frame_n) and source[src_lo, src_hi) from the device clouds, as doubles (f64) and records (f32)
    int fetch(cudaStream_t copy, const P3 *d_frame, const P3 *d_source, bool f64, bool f32, int64_t frame_n, int64_t src_lo,
              int64_t src_hi) {
        const size_t nf = (size_t)frame_n, lo = (size_t)src_lo, ns = (size_t)(src_hi - src_lo);
        if (f64 && nf) KICP_CUDA(cudaMemcpyAsync(frame, d_frame, nf * sizeof(P3), cudaMemcpyDeviceToHost, copy));
        if (f64 && ns) KICP_CUDA(cudaMemcpyAsync(source + lo, d_source + lo, ns * sizeof(P3), cudaMemcpyDeviceToHost, copy));
        if (f32 && nf) KICP_CUDA(cudaMemcpyAsync(frame32, d_rec, nf * 3 * sizeof(float), cudaMemcpyDeviceToHost, copy));
        if (f32 && ns)
            KICP_CUDA(cudaMemcpyAsync(source32 + 3 * lo, d_source_rec() + 3 * lo, ns * 3 * sizeof(float), cudaMemcpyDeviceToHost, copy));
        return KICP_OK;
    }
    // after the copy stream has drained: the staged counts, and the doubles to the caller's buffers (either may be null)
    void publish(bool f64, bool f32, int64_t nf, int64_t ns, double *out_frame, double *out_source) {
        if (f64) n_frame = nf, n_source = ns;
        if (f32) n_frame32 = nf, n_source32 = ns;
        if (out_frame && nf) memcpy(out_frame, frame, (size_t)nf * sizeof(P3));
        if (out_source && ns) memcpy(out_source, source, (size_t)ns * sizeof(P3));
    }
};

struct Scratch {
    P3 *in = nullptr, *out = nullptr, *out2 = nullptr, *out3 = nullptr;
    double *stamps = nullptr, *d_mm = nullptr;  // d_mm: {min, max} of the stamps, then the per-CTA partials of their reduction
    unsigned int *d_mm_ticket = nullptr;
    unsigned char *raw = nullptr;
    size_t raw_cap = 0;
    int *h_count = nullptr;  // pinned, 4 ints
    double *h_range = nullptr;  // pinned, 2 doubles: the stamps' {min, max} kicp_frame_stage returns
    // kicp_frame_stage_sensors: per sensor the {min, max} of its stamps (device, then pinned), followed on the device by the partials of
    // their reduction, and the kept beam count of each LaserScan (device, then pinned)
    double *d_seg_mm = nullptr, *h_seg_mm = nullptr;
    int *d_seg_count = nullptr, *h_seg_count = nullptr;
    uint32_t *h_mapctr = nullptr;  // pinned, 8 words: the map's counters after an asynchronous update
    cudaEvent_t ev_front = nullptr;  // front end finished (the copy stream waits for it before staging the clouds)
    int64_t last_source = 0;       // registration-source points of the previous frame (sizes this frame's grid and staging copy)
    Staging staged;
    // the frame kicp_frame_stage left in s.in (points) and s.stamps / s.d_mm (stamps and their {min, max}) for
    // kicp_register_staged_frame: its point count, -1 when there is none (consumed, or discarded by another front-end call)
    int64_t held_n = -1, held_n_stamps = 0;
    // its sensors (1 for a frame of kicp_frame_stage / kicp_frame_stage_laser_scan): where each one's points are in s.in, how many, and
    // whether they have stamps; held_extent is the end of the last sensor's place (holes included).  Meaningful while held_n >= 0.
    struct HeldSensor {
        int base, count;
        bool stamped;
    };
    int held_k = 1;
    HeldSensor held[kMaxSensors] = {};
    int64_t held_extent = 0;
    double held_range[2] = {0.0, 0.0};  // the staged frame's window {T0, T1} (meaningful when held_n_stamps > 0)
    // the segment tables of kicp_register_staged_*_segments (KICP_MAX_SENSORS x KICP_MAX_DESKEW_SEGMENTS entries, allocated on first
    // use): packed in pinned memory, copied on the context stream; ev_segs marks the end of the last copy, which the next packing waits
    // for (complete already after a frame's synchronisation, so it only orders a frame that failed before its end)
    DeskewSeg *d_segs = nullptr, *h_segs = nullptr;
    cudaEvent_t ev_segs = nullptr;
    bool segs_pending = false;
    // the clouds of the last frame as kicp_frame_clouds_device returns them (s.out, s.out3 and, with f32, staged.d_rec): 0 after any
    // other front-end call and after a frame that failed
    int64_t dev_n_frame = 0, dev_n_source = 0;
    bool dev_f32 = false;
    // option "correspondences": the per-point results of the last frame's evaluation (allocated on first use for corr_cap points) and
    // its statistics (pinned, copied on the stream); corr_n source points and `corr` as kicp_frame_correspondences returns them, 0 after
    // any other front-end call, a frame that failed or one without the option
    P3 *corr_pts = nullptr;
    double *corr_dist = nullptr;
    uint8_t *corr_inl = nullptr;
    kicp_corr_stats *h_corr = nullptr;
    int64_t corr_cap = 0, corr_n = 0;
    kicp_corr_stats corr = {};
    // the map-update policy: the last frame's outcome as kicp_frame_map_update returns it (the report's lifetime: NONE after any other
    // front-end call and a frame that failed), and for GATED in the single-synchronisation order the gate's shadow result block and
    // outcome word (device, allocated on the first such frame) and the outcome's pinned copy
    int32_t map_update = KICP_FRAME_UPDATE_NONE;
    kicp_reg_result *d_shadow = nullptr;
    int32_t *d_gate = nullptr, *h_gate = nullptr;
    // free-space clearing (kicp_ctx_set_free_space): the last frame's statistics as kicp_frame_free_space returns them (the report's
    // lifetime) and their pinned copy (allocated on the first frame with the option)
    kicp_free_space_stats free_space = {};
    kicp_free_space_stats *h_free = nullptr;
    double timing[8] = {0};  // host-side stage times of the last kicp_register_frame, milliseconds (debug export)
    int *first_idx = nullptr, *slot_of = nullptr, *d_count = nullptr;
    int4 *slots = nullptr;
    int64_t cap = 0;
    uint32_t nslots = 0;
    // option "downsample_order" 1 (kicp_downsample_order_kernels.cuh), allocated on its first use for cap points and
    // robin_buckets(cap) buckets: the survivors in first-occurrence order, the bucket histogram (zero between calls), its exclusive
    // sum and prefix max, and per survivor its home, ticket, place in bucket order, bucket and replayed cluster slot
    P3 *ro_pts = nullptr;
    uint32_t *ro_cnt = nullptr, *ro_start = nullptr, *ro_home = nullptr, *ro_ticket = nullptr, *ro_bucket = nullptr;
    int *ro_q = nullptr, *ro_slot = nullptr, *ro_table = nullptr;
    int64_t ro_cap = 0;
};
void release(Scratch &s) {
    cudaFree(s.ro_pts), cudaFree(s.ro_cnt), cudaFree(s.ro_start), cudaFree(s.ro_home), cudaFree(s.ro_ticket), cudaFree(s.ro_bucket);
    cudaFree(s.ro_q), cudaFree(s.ro_slot), cudaFree(s.ro_table);
    cudaFree(s.in), cudaFree(s.out), cudaFree(s.out2), cudaFree(s.out3), cudaFree(s.stamps), cudaFree(s.d_mm_ticket);
    cudaFree(s.first_idx), cudaFree(s.slot_of), cudaFree(s.slots), cudaFree(s.d_count), cudaFree(s.d_mm);
    cudaFree(s.raw), cudaFreeHost(s.h_count), cudaFreeHost(s.h_mapctr), cudaFreeHost(s.h_range);
    cudaFree(s.d_seg_mm), cudaFree(s.d_seg_count), cudaFreeHost(s.h_seg_mm), cudaFreeHost(s.h_seg_count);
    cudaFree(s.d_segs), cudaFreeHost(s.h_segs);
    cudaFree(s.corr_pts), cudaFree(s.corr_dist), cudaFree(s.corr_inl), cudaFreeHost(s.h_corr);
    cudaFree(s.d_shadow), cudaFree(s.d_gate), cudaFreeHost(s.h_gate), cudaFreeHost(s.h_free);
    if (s.ev_segs) cudaEventDestroy(s.ev_segs);
    s.staged.release();
    if (s.ev_front) cudaEventDestroy(s.ev_front);
    s = Scratch();
}
// what the context's front end owns: the scratch and, beside it, the LaserScan tables, one per sensor index of
// kicp_frame_stage_sensors (a robot's scanners each keep their own, as each would have its own projector); the single-sensor calls use
// the first
struct Frontend {
    Scratch s;
    LaserTable laser[kMaxSensors];
};
void free_scratch(kicp_ctx *c) {
    if (!c->frontend) return;
    Frontend *f = static_cast<Frontend *>(c->frontend);
    release(f->s);
    for (LaserTable &t : f->laser) cudaFree(t.d_cs);
    delete f;
    c->frontend = nullptr;
}
// the front end belongs to the context (created on first use, freed by kicp_ctx_destroy); like every other object of the
// library it is not thread-safe
Frontend &frontend(kicp_ctx *c) {
    if (!c->frontend) {
        c->frontend = new Frontend();
        c->frontend_free = free_scratch;
    }
    return *static_cast<Frontend *>(c->frontend);
}
Scratch &scratch(kicp_ctx *c) { return frontend(c).s; }

int reserve(kicp_ctx *c, Scratch &s, int64_t n) {
    if (n <= s.cap) return KICP_OK;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->copy_stream));
    release(s);
    const int64_t cap = std::max<int64_t>(n + n / 4, 4096);
    uint32_t nslots = 1;
    while (nslots < (uint64_t)cap * 2) nslots <<= 1;
    KICP_CUDA(cudaMalloc(&s.in, cap * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.out, cap * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.out2, cap * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.out3, cap * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.d_mm, (2 + 2 * kMinMaxMaxGrid) * sizeof(double)));
    KICP_CUDA(cudaMalloc(&s.d_mm_ticket, sizeof(unsigned int)));
    KICP_CUDA(cudaMemsetAsync(s.d_mm_ticket, 0, sizeof(unsigned int), c->stream));
    KICP_CUDA(cudaMallocHost(&s.h_count, 4 * sizeof(int)));
    KICP_CUDA(cudaMallocHost(&s.h_mapctr, 8 * sizeof(uint32_t)));
    KICP_CUDA(cudaMallocHost(&s.h_range, 2 * sizeof(double)));
    KICP_CUDA(cudaEventCreateWithFlags(&s.ev_front, cudaEventDisableTiming));
    KICP_TRY(s.staged.reserve(cap, false));
    KICP_CUDA(cudaMalloc(&s.stamps, cap * sizeof(double)));
    KICP_CUDA(cudaMalloc(&s.first_idx, (size_t)nslots * sizeof(int)));
    KICP_CUDA(cudaMalloc(&s.slot_of, cap * sizeof(int)));
    KICP_CUDA(cudaMalloc(&s.slots, (size_t)nslots * sizeof(int4)));
    KICP_CUDA(cudaMalloc(&s.d_count, 4 * sizeof(int)));
    KICP_CUDA(cudaMalloc(&s.d_seg_mm, 2 * kMaxSensors * (1 + kSensorMinMaxMaxGrid) * sizeof(double)));
    KICP_CUDA(cudaMalloc(&s.d_seg_count, kMaxSensors * sizeof(int)));
    KICP_CUDA(cudaMallocHost(&s.h_seg_mm, 2 * kMaxSensors * sizeof(double)));
    KICP_CUDA(cudaMallocHost(&s.h_seg_count, kMaxSensors * sizeof(int)));
    s.cap = cap, s.nslots = nslots;
    return KICP_OK;
}

// Sophus SE3::log of a pose7 (host, once per frame)
void se3_log_host(const double p[7], double out[6]) {
    const double eps = 1e-10;
    const double qx = p[0], qy = p[1], qz = p[2], qw = p[3];
    const double squared_n = qx * qx + qy * qy + qz * qz;
    double two_atan_nbyw_by_n, theta;
    if (squared_n < eps * eps) {
        two_atan_nbyw_by_n = 2.0 / qw - (2.0 / 3.0) * squared_n / (qw * qw * qw);
        theta = 2.0 * squared_n / qw;
    } else {
        const double nn = std::sqrt(squared_n);
        const double at = qw < 0.0 ? std::atan2(-nn, -qw) : std::atan2(nn, qw);
        two_atan_nbyw_by_n = 2.0 * at / nn;
        theta = two_atan_nbyw_by_n * nn;
    }
    const double w[3] = {two_atan_nbyw_by_n * qx, two_atan_nbyw_by_n * qy, two_atan_nbyw_by_n * qz};
    const double O[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    double O2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O2[3 * i + j] = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
    double cc;
    if (std::abs(theta) < eps) {
        cc = 1.0 / 12.0;
    } else {
        const double half = 0.5 * theta;
        cc = (1.0 - theta * std::cos(half) / (2.0 * std::sin(half))) / (theta * theta);
    }
    double Vinv[9];
    for (int i = 0; i < 9; ++i) Vinv[i] = ((i % 4 == 0) ? 1.0 : 0.0) - 0.5 * O[i] + cc * O2[i];
    for (int i = 0; i < 3; ++i) out[i] = Vinv[3 * i] * p[4] + Vinv[3 * i + 1] * p[5] + Vinv[3 * i + 2] * p[6];
    out[3] = w[0], out[4] = w[1], out[5] = w[2];
}

// the scratch of option "downsample_order" 1 for s.cap points (allocated once per scratch size; the histogram starts at zero)
constexpr int64_t kRobinMaxPoints = 1 << 28;  // robin_buckets(2^28) = 2^29 buckets: below the single-pass scan's 2^30 items
int reserve_robin(kicp_ctx *c, Scratch &s) {
    if (s.ro_cap == s.cap) return KICP_OK;
    const size_t nb = robin_buckets(s.cap, s.cap), n = (size_t)s.cap;
    KICP_CUDA(cudaMalloc(&s.ro_pts, n * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.ro_cnt, nb * sizeof(uint32_t)));
    KICP_CUDA(cudaMalloc(&s.ro_start, (nb + 1) * sizeof(uint32_t)));
    KICP_CUDA(cudaMalloc(&s.ro_home, n * sizeof(uint32_t)));
    KICP_CUDA(cudaMalloc(&s.ro_ticket, n * sizeof(uint32_t)));
    KICP_CUDA(cudaMalloc(&s.ro_bucket, n * sizeof(uint32_t)));
    KICP_CUDA(cudaMalloc(&s.ro_q, nb * sizeof(int)));
    KICP_CUDA(cudaMalloc(&s.ro_slot, n * sizeof(int)));
    KICP_CUDA(cudaMalloc(&s.ro_table, n * sizeof(int)));
    KICP_CUDA(cudaMemsetAsync(s.ro_cnt, 0, nb * sizeof(uint32_t), c->stream));
    s.ro_cap = s.cap;
    return KICP_OK;
}

// the buffers of option "correspondences" for s.cap points (allocated on the first frame with the option, and after the scratch grew)
int reserve_corr(Scratch &s) {
    if (!s.h_corr) KICP_CUDA(cudaMallocHost(&s.h_corr, sizeof(kicp_corr_stats)));
    if (s.corr_cap == s.cap) return KICP_OK;
    cudaFree(s.corr_pts), cudaFree(s.corr_dist), cudaFree(s.corr_inl);
    s.corr_pts = nullptr, s.corr_dist = nullptr, s.corr_inl = nullptr, s.corr_cap = 0;
    KICP_CUDA(cudaMalloc(&s.corr_pts, (size_t)s.cap * sizeof(P3)));
    KICP_CUDA(cudaMalloc(&s.corr_dist, (size_t)s.cap * sizeof(double)));
    KICP_CUDA(cudaMalloc(&s.corr_inl, (size_t)s.cap));
    s.corr_cap = s.cap;
    return KICP_OK;
}

// the gate's buffers (KICP_MAP_UPDATE_GATED, allocated on the first gated frame of the single-synchronisation order); the shadow block
// starts zeroed, and the gate writes its pose and status before every use
int reserve_gate(Scratch &s) {
    if (s.d_shadow) return KICP_OK;
    KICP_CUDA(cudaMalloc(&s.d_shadow, sizeof(kicp_reg_result)));
    KICP_CUDA(cudaMemset(s.d_shadow, 0, sizeof(kicp_reg_result)));
    KICP_CUDA(cudaMalloc(&s.d_gate, sizeof(int32_t)));
    KICP_CUDA(cudaMallocHost(&s.h_gate, sizeof(int32_t)));
    return KICP_OK;
}

// VoxelDownsample of src[0, n) (n = *d_n when given, else n_max) into dst, survivor count to d_count_out; all on the stream:
// clear the scratch hash, claim a slot per voxel with the smallest input index, select the points that hold their voxel's index.
// With option "downsample_order" 1 the select writes to s.ro_pts and five more launches put the survivors into the robin_map's bucket
// order in dst (kicp_downsample_order_kernels.cuh); the counts stay on the device.
int enqueue_downsample(kicp_ctx *c, Scratch &s, const P3 *src, int n_max, const int *d_n, double voxel_size, P3 *dst, int *d_count_out) {
    const bool robin = c->downsample_order == 1;
    if (robin) {
        if (n_max > kRobinMaxPoints) {
            kicp_set_error("VoxelDownsample: option downsample_order 1 takes at most 2^28 points");
            return KICP_ERR_INVALID;
        }
        KICP_TRY(reserve_robin(c, s));
    }
    const int threads = 256, blocks = (n_max + threads - 1) / threads;
    k_ds_clear<<<(s.nslots + 255) / 256, 256, 0, c->stream>>>(s.slots, s.first_idx, (int)s.nslots);
    KICP_CHECK_LAUNCH(c);
    k_ds_insert<<<blocks, threads, 0, c->stream>>>(src, n_max, d_n, voxel_size, s.slots, s.nslots - 1, s.first_idx, s.slot_of);
    KICP_CHECK_LAUNCH(c);
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n_max, &sa));
    k_ds_select<<<(n_max + kScanTile - 1) / kScanTile, kScanThreads, 0, c->stream>>>(src, n_max, d_n, s.first_idx, s.slot_of,
                                                                                    robin ? s.ro_pts : dst, d_count_out, sa);
    KICP_CHECK_LAUNCH(c);
    if (!robin) return KICP_OK;
    const uint32_t nb_max = robin_buckets(n_max, n_max);
    const RobinArgs a{s.ro_pts, dst, d_n, d_count_out, n_max, nb_max, voxel_size, s.ro_cnt, s.ro_start, s.ro_q, s.ro_home, s.ro_ticket,
                      s.ro_slot, s.ro_bucket, s.ro_table};
    const unsigned scan_grid = (nb_max + kScanTile - 1) / kScanTile;
    k_robin_hist<<<blocks, threads, 0, c->stream>>>(a);
    KICP_CHECK_LAUNCH(c);
    KICP_TRY(kicp_scan_next(c, nb_max, &sa));
    k_robin_scan<<<scan_grid, kScanThreads, 0, c->stream>>>(a, sa);
    KICP_CHECK_LAUNCH(c);
    KICP_TRY(kicp_scan_next(c, nb_max, &sa));
    k_robin_qmax<<<scan_grid, kScanThreads, 0, c->stream>>>(a, sa);
    KICP_CHECK_LAUNCH(c);
    k_robin_place<<<blocks, threads, 0, c->stream>>>(a);
    KICP_CHECK_LAUNCH(c);
    k_robin_cluster<<<blocks, threads, 0, c->stream>>>(a);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// {min, max} of v[0, n) (s.stamps, or the beam-indexed stamps of a LaserScan) into s.d_mm
int enqueue_stamp_minmax(kicp_ctx *c, Scratch &s, const double *v, int n) {
    const int grid = std::min(kMinMaxMaxGrid, (n + 2047) / 2048);
    k_stamp_minmax<<<grid, 256, 0, c->stream>>>(v, n, s.d_mm + 2, s.d_mm_ticket, s.d_mm);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// Preprocess of s.in[0, n) + transform to the base frame, compacted into dst.  The stamps are on the host, or, with
// `stamps_held`, already in s.stamps with their {min, max} in s.d_mm (a frame of kicp_frame_stage).
int enqueue_preprocess(kicp_ctx *c, Scratch &s, int n, const double *stamps, int64_t n_stamps, bool stamps_held,
                       const double relative_motion[7], const double lidar_to_base[7], double max_range, double min_range, int deskew,
                       P3 *dst, int *d_count_out) {
    PreArgs a;
    a.deskew = (deskew && n_stamps > 0) ? 1 : 0;  // Preprocessing.cpp: `!deskew_ || timestamps.empty()` returns the frame as is
    a.max_range = max_range, a.min_range = min_range;
    a.lidar_to_base = Pose{lidar_to_base[0], lidar_to_base[1], lidar_to_base[2], lidar_to_base[3], lidar_to_base[4], lidar_to_base[5],
                           lidar_to_base[6]};
    for (int k = 0; k < 6; ++k) a.omega[k] = 0.0;
    if (a.deskew) {
        if (!stamps_held) {
            KICP_CUDA(cudaMemcpyAsync(s.stamps, stamps, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->stream));
            KICP_TRY(enqueue_stamp_minmax(c, s, s.stamps, n));
        }
        se3_log_host(relative_motion, a.omega);
    }
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n, &sa));
    k_preprocess_select<<<(n + kScanTile - 1) / kScanTile, kScanThreads, 0, c->stream>>>(s.in, s.stamps, s.d_mm, n, a, dst, d_count_out, sa);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// Preprocess of the staged frame's sensors (s.held) + the transform of each to the base frame, compacted into dst in sensor order.  The
// stamps are in s.stamps on the common clock, the window in s.d_mm (kicp_frame_stage_sensors, or kicp_frame_stage for one sensor).
int enqueue_preprocess_sensors(kicp_ctx *c, Scratch &s, const double (*deskew_motions)[7], const double (*lidar_to_bases)[7],
                               double max_range, double min_range, int deskew, P3 *dst, int *d_count_out) {
    SensorPreArgs a;
    a.k = s.held_k;
    for (int k = 0; k < kMaxSensors; ++k) {
        SensorPreSeg &g = a.seg[k];
        const bool used = k < s.held_k;
        g.base = used ? s.held[k].base : 0, g.count = used ? s.held[k].count : 0;
        PreArgs &p = g.pre;
        p.deskew = used && deskew && s.held[k].stamped ? 1 : 0;
        p.max_range = max_range, p.min_range = min_range;
        const double *l2b = used ? lidar_to_bases[k] : nullptr;
        p.lidar_to_base = l2b ? Pose{l2b[0], l2b[1], l2b[2], l2b[3], l2b[4], l2b[5], l2b[6]} : Pose{0, 0, 0, 1, 0, 0, 0};
        for (int j = 0; j < 6; ++j) p.omega[j] = 0.0;
        if (p.deskew) se3_log_host(deskew_motions[k], p.omega);
    }
    const int n = (int)s.held_extent;
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n, &sa));
    k_preprocess_select_sensors<<<(n + kScanTile - 1) / kScanTile, kScanThreads, 0, c->stream>>>(s.in, s.stamps, s.d_mm, n, a, dst,
                                                                                                  d_count_out, sa);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// Preprocess of the staged frame's sensors with their segment tables (packed in s.d_segs by the caller), compacted into dst in sensor
// order: one launch, as enqueue_preprocess_sensors
int enqueue_preprocess_segments(kicp_ctx *c, Scratch &s, const SegmentPreArgs &a, P3 *dst, int *d_count_out) {
    const int n = (int)s.held_extent;
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n, &sa));
    k_preprocess_select_segments<<<(n + kScanTile - 1) / kScanTile, kScanThreads, 0, c->stream>>>(s.in, s.stamps, n, a, s.d_segs, dst,
                                                                                                   d_count_out, sa);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// The opening of every front-end entry point: a frame staged by kicp_frame_stage is discarded — by a call that fails its validation
// (`status`) too — then the device is set and the scratch reserved for n points.
int open_frontend(kicp_ctx *c, int status, int64_t n) {
    if (c) {
        Scratch &s = scratch(c);
        s.held_n = -1, s.dev_n_frame = s.dev_n_source = 0;
        s.corr_n = 0, s.corr = kicp_corr_stats{}, s.map_update = KICP_FRAME_UPDATE_NONE, s.free_space = kicp_free_space_stats{};
    }
    if (status != KICP_OK) return status;
    KICP_CUDA(cudaSetDevice(c->device));
    return reserve(c, scratch(c), n);
}

// the survivor count in s.d_count, then the survivors in `src` when out_xyz holds them (kicp_voxel_downsample, kicp_preprocess and
// their _device variants: host or `device` out_xyz; nothing to copy when the select wrote into out_xyz itself)
int read_back(kicp_ctx *c, Scratch &s, const P3 *src, double *out_xyz, int64_t cap, int64_t *m, bool device = false) {
    int count = 0;
    KICP_CUDA(cudaMemcpyAsync(&count, s.d_count, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    *m = count;
    if (count > cap) return KICP_ERR_CAPACITY;
    if (src == reinterpret_cast<const P3 *>(out_xyz)) return KICP_OK;
    // on the context stream, and waited for: out_xyz is complete when the call returns (a device-to-device cudaMemcpy would not be),
    // and the next front-end call cannot overwrite src while the copy still reads it
    KICP_CUDA(cudaMemcpyAsync(out_xyz, src, (size_t)count * sizeof(P3), device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                              c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}
}  // namespace

extern "C" int kicp_voxel_downsample(kicp_ctx *c, const double *xyz, int64_t n, double voxel_size, double *out_xyz, int64_t cap,
                                     int64_t *m) {
    const bool valid = c && m && n >= 0 && (n == 0 || (xyz && out_xyz)) && voxel_size > 0.0 && n <= 0x3FFFFFFF;
    KICP_TRY(open_frontend(c, valid ? KICP_OK : KICP_ERR_INVALID, n));
    *m = 0;
    if (n == 0) return KICP_OK;
    Scratch &s = scratch(c);
    KICP_CUDA(cudaMemcpyAsync(s.in, xyz, (size_t)n * sizeof(P3), cudaMemcpyHostToDevice, c->stream));
    KICP_TRY(enqueue_downsample(c, s, s.in, (int)n, nullptr, voxel_size, s.out, s.d_count));
    return read_back(c, s, s.out, out_xyz, cap, m);
}

extern "C" int kicp_preprocess(kicp_ctx *c, const double *xyz, int64_t n, const double *stamps, int64_t n_stamps,
                               const double relative_motion[7], const double lidar_to_base[7], double max_range, double min_range,
                               int deskew, double *out_xyz, int64_t cap, int64_t *m) {
    const bool valid = c && m && n >= 0 && (n == 0 || (xyz && out_xyz)) && relative_motion && lidar_to_base && n <= 0x3FFFFFFF &&
                       !(deskew && n_stamps > 0 && (n_stamps != n || !stamps));
    KICP_TRY(open_frontend(c, valid ? KICP_OK : KICP_ERR_INVALID, n));
    *m = 0;
    if (n == 0) return KICP_OK;
    Scratch &s = scratch(c);
    KICP_CUDA(cudaMemcpyAsync(s.in, xyz, (size_t)n * sizeof(P3), cudaMemcpyHostToDevice, c->stream));
    KICP_TRY(enqueue_preprocess(c, s, (int)n, stamps, n_stamps, false, relative_motion, lidar_to_base, max_range, min_range, deskew, s.out,
                                s.d_count));
    return read_back(c, s, s.out, out_xyz, cap, m);
}

// ------------------------------------------------------------------------------------------- fused RegisterFrame
namespace {
// byte layout of a kicp_frame_input's records: stride and x/y/z offsets (the tightly packed defaults when point_step == 0)
struct Layout {
    int elem, step, ox, oy, oz;
};
int frame_layout(const kicp_frame_input *in, Layout &l) {
    const int64_t n = in->n;
    if (n < 0 || n > 0x3FFFFFFF || (n > 0 && !in->data)) return KICP_ERR_INVALID;
    if (in->dtype != KICP_DTYPE_F64 && in->dtype != KICP_DTYPE_F32) return KICP_ERR_INVALID;
    l.elem = in->dtype == KICP_DTYPE_F32 ? 4 : 8;
    l.step = in->point_step > 0 ? in->point_step : 3 * l.elem;
    l.ox = in->point_step > 0 ? in->offset_x : 0, l.oy = in->point_step > 0 ? in->offset_y : l.elem;
    l.oz = in->point_step > 0 ? in->offset_z : 2 * l.elem;
    if (l.ox < 0 || l.oy < 0 || l.oz < 0 || l.ox + l.elem > l.step || l.oy + l.elem > l.step || l.oz + l.elem > l.step)
        return KICP_ERR_INVALID;
    return KICP_OK;
}
// packed float64 x,y,z: the layout the kernels read, so that the records are copied, or read in place, rather than widened
bool packed_f64(const kicp_frame_input *in, const Layout &l) {
    return in->dtype == KICP_DTYPE_F64 && l.step == 24 && l.ox == 0 && l.oy == 8 && l.oz == 16;
}
// k_ingest of n > 0 records at `raw` (device memory) into packed doubles at dst
int launch_ingest(kicp_ctx *c, const kicp_frame_input *in, const Layout &l, const unsigned char *raw, P3 *dst) {
    const IngestArgs a{in->dtype == KICP_DTYPE_F32, l.step, l.ox, l.oy, l.oz};
    k_ingest<<<(unsigned)((in->n + 255) / 256), 256, 0, c->stream>>>(raw, (int)in->n, a, dst);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// the device buffer the raw input bytes are uploaded to, grown to at least `bytes`
int reserve_raw(kicp_ctx *c, Scratch &s, size_t bytes) {
    if (bytes > s.raw_cap) {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        cudaFree(s.raw);
        s.raw = nullptr, s.raw_cap = 0;
        KICP_CUDA(cudaMalloc(&s.raw, bytes + bytes / 4));
        s.raw_cap = bytes + bytes / 4;
    }
    return KICP_OK;
}

// upload of the frame's n > 0 records (once) and their widening into s.in + base; with `t`, the time field is decoded into
// s.stamps + base in the same pass.  Packed float64 x,y,z without a time field are copied straight into s.in + base.  `device` records
// are read in place (the packed float64 ones copied device to device); host records are uploaded to s.raw + raw_off.
int enqueue_ingest(kicp_ctx *c, Scratch &s, const kicp_frame_input *in, const Layout &l, const StampArgs *t, bool device, int64_t base = 0,
                   size_t raw_off = 0) {
    const int64_t n = in->n;
    if (!t && packed_f64(in, l)) {
        KICP_CUDA(cudaMemcpyAsync(s.in + base, in->data, (size_t)n * sizeof(P3),
                                  device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
        return KICP_OK;
    }
    const unsigned char *raw = static_cast<const unsigned char *>(in->data);
    if (!device) {
        const size_t raw_bytes = (size_t)n * l.step;
        KICP_TRY(reserve_raw(c, s, raw_off + raw_bytes));
        KICP_CUDA(cudaMemcpyAsync(s.raw + raw_off, in->data, raw_bytes, cudaMemcpyHostToDevice, c->stream));
        raw = s.raw + raw_off;
    }
    if (!t) return launch_ingest(c, in, l, raw, s.in + base);
    const IngestArgs a{in->dtype == KICP_DTYPE_F32, l.step, l.ox, l.oy, l.oz};
    k_ingest_stamped<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(raw, (int)n, a, *t, s.in + base, s.stamps + base);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// kicp_frame_stage's checks of a record set (`where` names it in the errors of the device-range checks); fills its layout.
// *range_error (optional) tells whether a failure came from a device-range check, which has set the error text.
int check_frame_stage(kicp_ctx *c, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset, bool device, Layout &l,
                      const std::string &where, bool *range_error = nullptr) {
    if (!in || frame_layout(in, l) != KICP_OK) return KICP_ERR_INVALID;
    if (stamp_datatype == 0) {
        if (in->n_stamps > 0 && (in->n_stamps != in->n || !in->stamps)) return KICP_ERR_INVALID;
    } else {
        if (stamp_datatype != 6 && stamp_datatype != 7 && stamp_datatype != 8) return KICP_ERR_UNSUPPORTED;
        const int width = stamp_datatype == 8 ? 8 : 4;
        if (in->point_step <= 0 || stamp_offset < 0 || stamp_offset + width > in->point_step || in->n_stamps > 0) return KICP_ERR_INVALID;
    }
    if (!device || in->n == 0) return KICP_OK;
    if (range_error) *range_error = true;
    // the bytes the ingest reads: up to the last field of the last record
    const int end = std::max({l.ox, l.oy, l.oz}) + l.elem, t_end = stamp_datatype == 0 ? 0 : stamp_offset + (stamp_datatype == 8 ? 8 : 4);
    KICP_TRY(kicp_check_device_range(c, in->data, (size_t)(in->n - 1) * l.step + std::max(end, t_end), 1, (where + "data").c_str()));
    if (in->n_stamps > 0)
        KICP_TRY(kicp_check_device_range(c, in->stamps, (size_t)in->n_stamps * sizeof(double), sizeof(double), (where + "stamps").c_str()));
    if (range_error) *range_error = false;
    return KICP_OK;
}

// kicp_frame_stage_laser_scan's checks of a scan (`where` names its ranges in the error of the device-range check; *range_error as
// check_frame_stage's)
int check_laser_scan(kicp_ctx *c, const kicp_laser_scan *scan, bool device, const std::string &where, bool *range_error = nullptr) {
    if (!scan || scan->n < 0 || scan->n > 0x3FFFFFFF || (scan->n > 0 && !scan->ranges)) return KICP_ERR_INVALID;
    if (!device || scan->n == 0) return KICP_OK;
    const int st = kicp_check_device_range(c, scan->ranges, (size_t)scan->n * sizeof(float), sizeof(float), where.c_str());
    if (range_error) *range_error = st != KICP_OK;
    return st;
}

// k_laser_project_select of a scan of n > 0 beams into s.in / s.stamps + base (table refreshed by the caller), its kept count to
// *d_count_out and its beam-indexed stamps to beam_stamps; host ranges are uploaded to s.raw + raw_off
int enqueue_laser(kicp_ctx *c, Scratch &s, LaserTable &lt, const kicp_laser_scan *scan, bool device, int64_t base, size_t raw_off,
                  double *beam_stamps, int *d_count_out) {
    const int64_t n = scan->n;
    KICP_TRY(lt.upload(c->stream));
    const float *ranges = scan->ranges;
    if (!device) {
        KICP_TRY(reserve_raw(c, s, raw_off + (size_t)n * sizeof(float)));
        KICP_CUDA(cudaMemcpyAsync(s.raw + raw_off, scan->ranges, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        ranges = reinterpret_cast<const float *>(s.raw + raw_off);
    }
    kicp_scan_args sa;
    KICP_TRY(kicp_scan_next(c, n, &sa));
    const LaserArgs a{scan->range_min, scan->range_max, scan->time_increment};
    k_laser_project_select<<<(unsigned)((n + kScanTile - 1) / kScanTile), kScanThreads, 0, c->stream>>>(
        ranges, lt.d_cs, (int)n, a, s.in + base, s.stamps + base, beam_stamps, d_count_out, sa);
    KICP_CHECK_LAUNCH(c);
    return KICP_OK;
}

// The arguments of kicp_register_frame / kicp_register_staged_frame, for the frame they leave in s.in[0, n) with its stamps as
// enqueue_preprocess takes them
struct FrameArgs {
    int64_t n;
    const double *stamps;
    int64_t n_stamps;
    bool stamps_held;
    const double *deskew_motion, *lidar_to_base, *last_pose, *relative_odometry;
    double tau;
    const kicp_frame_params *fp;
    double *out_pose, *out_frame;
    int64_t cap_frame, *n_frame;
    double *out_source;
    int64_t cap_source, *n_source;
    kicp_reg_result *result;
    std::chrono::steady_clock::time_point t0;  // the call's start (timing[] is measured from it)
    // kicp_register_staged_sensors: per sensor of the staged frame (s.held) its deskew motion and extrinsic; null for the single-sensor
    // calls (deskew_motion / lidar_to_base)
    const double (*deskew_motions)[7] = nullptr, (*lidar_to_bases)[7] = nullptr;
    // kicp_register_staged_*_segments: the Preprocess arguments of every sensor, whose segment tables are in s.d_segs already
    const SegmentPreArgs *segments = nullptr;
    bool valid() const {
        return deskew_motion && lidar_to_base && last_pose && relative_odometry && fp && out_pose && fp->voxel_size > 0.0;
    }
};

// KinematicICP::RegisterFrame from the frame in s.in[0, n) on: Preprocess, both down-samples, registration, map update (as the
// context's map-update policy decides, kicp_map_update.h), the two clouds.  A frame is ONE host synchronisation (at its end): every later stage reads the survivor counts and the pose from device
// memory, and the registration and the staging copies are sized by upper bounds.  The read-back order (read the counts back, size
// everything exactly) remains for callers whose output buffers might be too small for the worst case — they are owed
// KICP_ERR_CAPACITY before the map changes — and as option "frame_sync" for A/B measurements.
int register_ingested(kicp_map *map, Scratch &s, const FrameArgs &a) {
    auto ms_since = [&a]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a.t0).count(); };
    kicp_ctx *c = map->ctx;
    const kicp_frame_params *fp = a.fp;
    const int64_t n = a.n;
    // KICP_STAGE_F64 (and any other nonzero value but KICP_STAGE_F32 alone, as before the flag had two bits): the clouds as doubles
    const bool stage = (fp->stage_clouds & ~KICP_STAGE_F32) != 0 || a.out_frame || a.out_source;
    const bool stage32 = (fp->stage_clouds & KICP_STAGE_F32) != 0;
    const bool one_sync = n > 0 && !c->frame_sync && (!a.out_frame || a.cap_frame >= n) && (!a.out_source || a.cap_source >= n);
    // the policy: NEVER enqueues no Update; GATED decides on the report, which it evaluates whatever option "correspondences" says,
    // and on whether the map held points before the frame (the host mirror is current: every frame call ends with it up to date)
    const kicp_map_update_policy policy = c->map_update;
    const bool never = policy.mode == KICP_MAP_UPDATE_NEVER, gated = policy.mode == KICP_MAP_UPDATE_GATED;
    const bool map_was_empty = map->num_points == 0;
    const bool corr = c->correspondences != 0 || gated;
    // free-space clearing after an applied Update: the frame's rays from the sensor origin in the base frame (lidar_to_base's translation)
    const kicp_free_space_params fs = c->free_space;
    const bool clear = fs.min_misses > 0 && !never;
    const double fs_origin[3] = {a.lidar_to_base[4], a.lidar_to_base[5], a.lidar_to_base[6]};
    kicp_free_space_stats free_st{};
    s.corr_n = 0, s.corr = kicp_corr_stats{}, s.map_update = KICP_FRAME_UPDATE_NONE, s.free_space = kicp_free_space_stats{};
    // the report's buffers are sized before anything of this frame is enqueued: a growth (cudaFree / cudaMalloc) waits for the device
    if (corr) KICP_TRY(reserve_corr(s));
    if (clear && !s.h_free) KICP_CUDA(cudaMallocHost(&s.h_free, sizeof(kicp_free_space_stats)));
    if (gated && one_sync) KICP_TRY(reserve_gate(s));
    // the survivor counts of the three stages (12 bytes back, one synchronisation of the stream)
    int counts[3] = {0, 0, 0};
    auto read_counts = [&]() -> int {
        KICP_CUDA(cudaMemcpyAsync(s.h_count, s.d_count, 3 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        for (int k = 0; k < 3; ++k) counts[k] = s.h_count[k];
        s.last_source = counts[2];
        if (a.n_frame) *a.n_frame = counts[0];
        if (a.n_source) *a.n_source = counts[2];
        return KICP_OK;
    };
    if (n > 0) {
        // s.out = preprocessed frame in base, s.out2 = frame_downsample (0.5 vs), s.out3 = source (1.5 vs); each stage reads
        // the previous stage's survivor count from device memory (KinematicICP.cpp:38-44, 54-62)
        if (a.segments)
            KICP_TRY(enqueue_preprocess_segments(c, s, *a.segments, s.out, s.d_count));
        else if (a.deskew_motions)
            KICP_TRY(enqueue_preprocess_sensors(c, s, a.deskew_motions, a.lidar_to_bases, fp->max_range, fp->min_range,
                                                fp->deskew && a.n_stamps > 0, s.out, s.d_count));
        else
            KICP_TRY(enqueue_preprocess(c, s, (int)n, a.stamps, a.n_stamps, a.stamps_held, a.deskew_motion, a.lidar_to_base,
                                        fp->max_range, fp->min_range, fp->deskew, s.out, s.d_count));
        KICP_TRY(enqueue_downsample(c, s, s.out, (int)n, s.d_count, fp->voxel_size * 0.5, s.out2, s.d_count + 1));
        KICP_TRY(enqueue_downsample(c, s, s.out2, (int)n, s.d_count + 1, fp->voxel_size * 1.5, s.out3, s.d_count + 2));
        if (stage32) {  // the published records, encoded before the registration so that they never share the SMs with its grid
            KICP_TRY(s.staged.reserve(s.cap, true));
            k_encode_clouds<<<(unsigned)((3 * n + 255) / 256), 256, 0, c->stream>>>(s.out, s.out3, (int)n, s.d_count, s.staged.d_rec,
                                                                                  s.staged.d_source_rec());
            KICP_CHECK_LAUNCH(c);
        }
        if (!one_sync) KICP_TRY(read_counts());
    }
    s.timing[0] = ms_since();  // upload + front end (ingest, de-skew, filter, transform, both down-samples)
    // (in the single-synchronisation order the counts are still 0 and the caller's buffers hold n points)
    if ((a.out_frame && counts[0] > a.cap_frame) || (a.out_source && counts[2] > a.cap_source)) return KICP_ERR_CAPACITY;
    if (one_sync && (stage || stage32)) KICP_CUDA(cudaEventRecord(s.ev_front, c->stream));
    // registration of the source against the local map, enqueued first so that the staging copies overlap it; in the
    // single-synchronisation order its grid is planned from the previous source
    const int64_t reg_n = one_sync ? n : counts[2];
    const int64_t reg_hint = one_sync && s.last_source > 0 ? s.last_source + s.last_source / 4 + 256 : 0;
    KICP_TRY(kicp_enqueue_registration_device(map, reg_n ? reinterpret_cast<const double *>(s.out3) : nullptr, reg_n,
                                              one_sync ? s.d_count + 2 : nullptr, a.last_pose, a.relative_odometry, a.tau, &fp->reg,
                                              reg_hint));
    s.timing[1] = ms_since();  // + registration enqueued
    // the two clouds go to pinned staging on the copy stream while the registration runs; in the single-synchronisation order the
    // frame is copied for n points and the source for the previous frame's twofold (the rest follows below)
    s.staged.n_frame = s.staged.n_source = s.staged.n_frame32 = s.staged.n_source32 = 0;
    const int64_t src_copy = one_sync ? std::min<int64_t>(n, std::max<int64_t>(2 * s.last_source, 32768)) : counts[2];
    if (one_sync && (stage || stage32)) KICP_CUDA(cudaStreamWaitEvent(c->copy_stream, s.ev_front, 0));
    KICP_TRY(s.staged.fetch(c->copy_stream, s.out, s.out3, stage, stage32, one_sync ? n : counts[0], 0, src_copy));
    if (corr) {
        // the source at the pose the registration returns (read from its result block) against the map before this frame's Update,
        // the source count read from the device in the single-synchronisation order; the statistics come back with the frame's
        // synchronisation
        KICP_TRY(kicp_map_enqueue_correspondences(map, reinterpret_cast<const double *>(s.out3), reg_n, one_sync ? s.d_count + 2 : nullptr,
                                                  nullptr, kicp_device_result(c), a.tau, reinterpret_cast<double *>(s.corr_pts),
                                                  s.corr_dist, s.corr_inl, s.h_corr));
    }
    if (one_sync) {
        if (!never) {
            // local_map_.Update(frame_downsample, new_pose) (KinematicICP.cpp:79), pose and count still on the device.  Under GATED the
            // gate reads the result block and the report's statistics (the bytes copied to s.h_corr above) and hands the map's kernels
            // a shadow block whose status is KICP_OK only when the update is applied; they leave the map untouched otherwise.
            const kicp_reg_result *d_res = kicp_device_result(c);
            if (gated) {
                k_map_update_gate<<<1, 1, 0, c->stream>>>(d_res, map->d_corr_stats, policy, map_was_empty ? 1 : 0, s.d_shadow, s.d_gate);
                KICP_CHECK_LAUNCH(c);
                KICP_CUDA(cudaMemcpyAsync(s.h_gate, s.d_gate, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
                d_res = s.d_shadow;
            }
            KICP_TRY(kicp_map_update_pose_async(map, reinterpret_cast<const double *>(s.out2), n, s.d_count + 1, d_res, s.h_mapctr,
                                                clear ? &fs : nullptr, fs_origin, s.h_free));
        }
        KICP_TRY(read_counts());  // THE synchronisation of the frame
    } else {
        KICP_CUDA(cudaStreamSynchronize(c->stream));
    }
    s.timing[2] = ms_since();  // + registration finished
    const kicp_reg_result &r = *c->h_result;
    for (int k = 0; k < 7; ++k) a.out_pose[k] = r.pose[k];
    if (a.result) *a.result = r;
    int status = r.status;
    // a NaN pose (zero correspondences, which the reference does not defend against) is reported and leaves the map untouched; in the
    // read-back order the host applies the gate's rule to the statistics it has read back
    const int32_t outcome = one_sync && gated ? *s.h_gate
                                              : map_update_outcome(policy, r.status, map_was_empty, corr ? *s.h_corr : kicp_corr_stats{});
    if (one_sync) {
        const int mst = never ? KICP_OK : kicp_map_finish_update(map, s.h_mapctr, false);
        if (mst != KICP_OK) status = mst;
        if (clear) free_st = *s.h_free;
    } else if (outcome == KICP_FRAME_UPDATE_APPLIED && counts[1] > 0) {
        status = kicp_map_update_pose_packed(map, reinterpret_cast<const double *>(s.out2), counts[1], r.pose);
        if (status == KICP_OK && clear)
            status = kicp_map_clear_free_space_packed(map, reinterpret_cast<const double *>(s.out2), counts[1], r.pose, fs_origin, &fs,
                                                      &free_st);
    }
    s.timing[3] = ms_since();  // + map update
    if (counts[2] > src_copy) KICP_TRY(s.staged.fetch(c->copy_stream, s.out, s.out3, stage, stage32, 0, src_copy, counts[2]));
    if (stage || stage32 || !one_sync) KICP_CUDA(cudaStreamSynchronize(c->copy_stream));
    s.staged.publish(stage, stage32, counts[0], counts[2], a.out_frame, a.out_source);
    if (status == KICP_OK || status == KICP_WARN_NO_CORRESPONDENCES) {
        s.dev_n_frame = counts[0], s.dev_n_source = counts[2], s.dev_f32 = stage32;
        if (corr) s.corr_n = counts[2], s.corr = *s.h_corr;
        s.map_update = outcome;
        s.free_space = free_st;
    }
    s.timing[4] = ms_since();  // + clouds delivered
    return status;
}
}  // namespace

// KinematicICP::RegisterFrame (pipeline/KinematicICP.cpp:48-85) with every per-point stage on the device and the frame
// resident in HBM from ingest to map update: one upload of the raw scan, one pose-sized download, plus the two point
// clouds the reference returns by value.  The scalar threshold model (CorrespondenceThreshold) stays with the caller:
// it needs tau before and the pose after, both of which cross this boundary anyway.
extern "C" int kicp_register_frame(kicp_map *map, const kicp_frame_input *in, const double deskew_motion[7], const double lidar_to_base[7],
                                   const double last_pose[7], const double relative_odometry[7], double tau, const kicp_frame_params *fp,
                                   double out_pose[7], double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source,
                                   int64_t cap_source, int64_t *n_source, kicp_reg_result *result) {
    const FrameArgs a{in ? in->n : 0, in ? in->stamps : nullptr, in ? in->n_stamps : 0, false, deskew_motion, lidar_to_base, last_pose,
                      relative_odometry, tau, fp, out_pose, out_frame, cap_frame, n_frame, out_source, cap_source, n_source, result,
                      std::chrono::steady_clock::now()};
    Layout l;
    const bool valid = map && in && a.valid() && frame_layout(in, l) == KICP_OK &&
                       !(fp->deskew && a.n_stamps > 0 && (a.n_stamps != a.n || !a.stamps));
    KICP_TRY(open_frontend(map ? map->ctx : nullptr, valid ? KICP_OK : KICP_ERR_INVALID, a.n));
    if (n_frame) *n_frame = 0;
    if (n_source) *n_source = 0;
    Scratch &s = scratch(map->ctx);
    if (a.n > 0) KICP_TRY(enqueue_ingest(map->ctx, s, in, l, nullptr, false));
    return register_ingested(map, s, a);
}

// The first half of an online node's frame (LidarOdometryServer.cpp:186-210 needs the sweep's stamps before it can look up the
// wheel odometry): the records cross PCIe once, the device decodes x, y, z and the time field and reduces the stamps' {min, max};
// 16 bytes come back.  The frame stays in HBM for kicp_register_staged_frame.  With `device`, the records and host stamps are the
// caller's device memory, read in place.
static int frame_stage(kicp_ctx *c, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset, double stamp_range[2],
                       int64_t *n_stamps, bool device) {
    Layout l;
    auto validate = [&]() -> int {
        if (!c || !stamp_range || !n_stamps) return KICP_ERR_INVALID;
        return check_frame_stage(c, in, stamp_datatype, stamp_offset, device, l, "kicp_frame_stage_device: in->");
    };
    KICP_TRY(open_frontend(c, validate(), in ? in->n : 0));
    const int64_t n = in->n;
    const StampArgs t{stamp_datatype, stamp_offset};
    Scratch &s = scratch(c);
    stamp_range[0] = stamp_range[1] = 0.0;
    *n_stamps = 0;
    const int64_t stamps = n > 0 && (stamp_datatype != 0 || in->n_stamps > 0) ? n : 0;
    if (n > 0) {
        KICP_TRY(enqueue_ingest(c, s, in, l, stamp_datatype != 0 ? &t : nullptr, device));
        if (stamps) {
            if (stamp_datatype == 0)
                KICP_CUDA(cudaMemcpyAsync(s.stamps, in->stamps, (size_t)n * sizeof(double),
                                          device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
            KICP_TRY(enqueue_stamp_minmax(c, s, s.stamps, (int)n));
            KICP_CUDA(cudaMemcpyAsync(s.h_range, s.d_mm, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        }
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        if (stamps) stamp_range[0] = s.h_range[0], stamp_range[1] = s.h_range[1];
    }
    *n_stamps = stamps;
    s.held_n = n, s.held_n_stamps = stamps;
    s.held_k = 1, s.held[0] = {0, (int)n, stamps > 0}, s.held_extent = n;
    s.held_range[0] = stamp_range[0], s.held_range[1] = stamp_range[1];
    return KICP_OK;
}
extern "C" int kicp_frame_stage(kicp_ctx *c, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset,
                                double stamp_range[2], int64_t *n_stamps) {
    return frame_stage(c, in, stamp_datatype, stamp_offset, stamp_range, n_stamps, false);
}
extern "C" int kicp_frame_stage_device(kicp_ctx *c, const kicp_frame_input *in, int32_t stamp_datatype, int32_t stamp_offset,
                                       double stamp_range[2], int64_t *n_stamps) {
    return frame_stage(c, in, stamp_datatype, stamp_offset, stamp_range, n_stamps, true);
}

// ------------------------------------------------------------------------------------------- device clouds (kicp_*_device)
int kicp_check_cloud_args(const kicp_frame_input *in, const char *fn) {
    Layout l;
    if (in->n < 0) return kicp_invalid(fn, "n < 0");
    if (in->n > 0x3FFFFFFF) return kicp_invalid(fn, "n >= 2^30");
    if (in->n > 0 && !in->data) return kicp_invalid(fn, "data: null pointer");
    if (in->dtype != KICP_DTYPE_F64 && in->dtype != KICP_DTYPE_F32) return kicp_invalid(fn, "dtype: neither KICP_DTYPE_F64 nor KICP_DTYPE_F32");
    if (frame_layout(in, l) != KICP_OK) return kicp_invalid(fn, "point_step / offset: a field outside the point");
    return KICP_OK;
}
int kicp_check_device_cloud(kicp_ctx *c, const kicp_frame_input *in, const char *fn, bool *packed) {
    KICP_TRY(kicp_check_cloud_args(in, fn));
    Layout l;
    KICP_TRY(frame_layout(in, l));
    if (packed) *packed = packed_f64(in, l);
    return check_frame_stage(c, in, 0, 0, true, l, std::string(fn) + ": ");
}
int kicp_enqueue_widen(kicp_ctx *c, const kicp_frame_input *in, double *dst) {
    Layout l;
    KICP_TRY(frame_layout(in, l));
    return launch_ingest(c, in, l, static_cast<const unsigned char *>(in->data), reinterpret_cast<P3 *>(dst));
}

namespace {
// The opening of kicp_voxel_downsample_device / kicp_preprocess_device: the device ranges of the cloud and `out` checked (cap points,
// or n when fewer) after the call's own checks (`status`, which include kicp_check_cloud_args), the staged frame discarded whatever
// they find, and the cloud ingested into s.in (copied device to device when it is packed float64, else widened by k_ingest).  *dst:
// where the select writes, `out` itself when it holds n points, else s.out.
int open_device_frontend(kicp_ctx *c, int status, const kicp_frame_input &in, double *out, int64_t cap, const char *fn, P3 **dst) {
    Layout l;
    if (status == KICP_OK) status = kicp_check_device_cloud(c, &in, fn, nullptr);
    if (status == KICP_OK && in.n > 0)
        status = kicp_check_device_range(c, out, (size_t)std::max<int64_t>(1, std::min(cap, in.n)) * sizeof(P3), sizeof(double),
                                         (std::string(fn) + ": out").c_str());
    KICP_TRY(open_frontend(c, status, in.n));
    Scratch &s = scratch(c);
    *dst = cap >= in.n ? reinterpret_cast<P3 *>(out) : s.out;
    if (in.n == 0) return KICP_OK;
    KICP_TRY(frame_layout(&in, l));
    return enqueue_ingest(c, s, &in, l, nullptr, true);
}
}  // namespace

extern "C" int kicp_voxel_downsample_device(kicp_ctx *c, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                            int32_t offset_y, int32_t offset_z, double voxel_size, double *out, int64_t cap, int64_t *m) {
    static const char fn[] = "kicp_voxel_downsample_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    auto validate = [&]() -> int {
        KICP_TRY(kicp_check_cloud_args(&in, fn));
        if (n > 0 && !out) return kicp_invalid(fn, "out: null pointer");
        if (!m) return kicp_invalid(fn, "m: null pointer");
        if (!(voxel_size > 0.0)) return kicp_invalid(fn, "voxel_size is not > 0");
        if (!c) return kicp_invalid(fn, "null context");
        return KICP_OK;
    };
    P3 *dst = nullptr;
    KICP_TRY(open_device_frontend(c, validate(), in, out, cap, fn, &dst));
    *m = 0;
    if (n == 0) return KICP_OK;
    Scratch &s = scratch(c);
    KICP_TRY(enqueue_downsample(c, s, s.in, (int)n, nullptr, voxel_size, dst, s.d_count));
    return read_back(c, s, dst, out, cap, m, true);
}

extern "C" int kicp_preprocess_device(kicp_ctx *c, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                      int32_t offset_y, int32_t offset_z, const double *stamps, int64_t n_stamps,
                                      const double relative_motion[7], const double lidar_to_base[7], double max_range, double min_range,
                                      int32_t deskew, double *out, int64_t cap, int64_t *m) {
    static const char fn[] = "kicp_preprocess_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    const bool stamped = deskew && n_stamps > 0;  // kicp_preprocess's rule: otherwise the stamps are not read
    auto validate = [&]() -> int {
        KICP_TRY(kicp_check_cloud_args(&in, fn));
        if (n > 0 && !out) return kicp_invalid(fn, "out: null pointer");
        if (!m) return kicp_invalid(fn, "m: null pointer");
        if (!relative_motion) return kicp_invalid(fn, "relative_motion: null pointer");
        if (!lidar_to_base) return kicp_invalid(fn, "lidar_to_base: null pointer");
        if (stamped && n_stamps != n) return kicp_invalid(fn, "n_stamps != n with deskew");
        if (stamped && !stamps) return kicp_invalid(fn, "stamps: null pointer");
        if (!c) return kicp_invalid(fn, "null context");
        if (!stamped) return KICP_OK;
        return kicp_check_device_range(c, stamps, (size_t)n_stamps * sizeof(double), 1, (std::string(fn) + ": stamps").c_str());
    };
    P3 *dst = nullptr;
    KICP_TRY(open_device_frontend(c, validate(), in, out, cap, fn, &dst));
    *m = 0;
    if (n == 0) return KICP_OK;
    Scratch &s = scratch(c);
    if (stamped) {  // into the staged frame's stamp buffer, whose {min, max} enqueue_preprocess then takes as held
        KICP_CUDA(cudaMemcpyAsync(s.stamps, stamps, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        KICP_TRY(enqueue_stamp_minmax(c, s, s.stamps, (int)n));
    }
    KICP_TRY(enqueue_preprocess(c, s, (int)n, nullptr, stamped ? n : 0, true, relative_motion, lidar_to_base, max_range, min_range, deskew,
                                dst, s.d_count));
    return read_back(c, s, dst, out, cap, m, true);
}

// The first half for a 2D LiDAR: the LaserScan's ranges cross PCIe once, k_laser_project_select projects, range-tests, stamps and
// compacts them into the staged frame (s.in, s.stamps), k_stamp_minmax reduces the beam-indexed stamps it leaves in s.out; the range
// and the kept count come back with one host synchronisation.  `device` ranges are read in place.
static int stage_laser_scan(kicp_ctx *c, const kicp_laser_scan *scan, double stamp_range[2], int64_t *n_points, bool device) {
    const bool valid = c && stamp_range && n_points && check_laser_scan(c, scan, false, "") == KICP_OK;
    const int status = valid ? check_laser_scan(c, scan, device, "kicp_frame_stage_laser_scan_device: scan->ranges") : KICP_ERR_INVALID;
    KICP_TRY(open_frontend(c, status, valid ? scan->n : 0));
    const int64_t n = scan->n;
    Scratch &s = scratch(c);
    stamp_range[0] = stamp_range[1] = 0.0;
    *n_points = 0;
    LaserTable &lt = frontend(c).laser[0];
    KICP_TRY(lt.refresh(scan, "kicp_frame_stage_laser_scan"));
    int64_t kept = 0;
    if (n > 0) {
        double *beam_stamps = reinterpret_cast<double *>(s.out);  // n doubles; s.out is free until the registration's Preprocess
        KICP_TRY(enqueue_laser(c, s, lt, scan, device, 0, 0, beam_stamps, s.d_count));
        KICP_TRY(enqueue_stamp_minmax(c, s, beam_stamps, (int)n));
        KICP_CUDA(cudaMemcpyAsync(s.h_range, s.d_mm, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaMemcpyAsync(s.h_count, s.d_count, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        kept = s.h_count[0];
        if (kept > 0) stamp_range[0] = s.h_range[0], stamp_range[1] = s.h_range[1];
    }
    *n_points = kept;
    s.held_n = kept, s.held_n_stamps = kept;
    s.held_k = 1, s.held[0] = {0, (int)kept, kept > 0}, s.held_extent = kept;
    s.held_range[0] = stamp_range[0], s.held_range[1] = stamp_range[1];
    return KICP_OK;
}
extern "C" int kicp_frame_stage_laser_scan(kicp_ctx *c, const kicp_laser_scan *scan, double stamp_range[2], int64_t *n_points) {
    return stage_laser_scan(c, scan, stamp_range, n_points, false);
}
extern "C" int kicp_frame_stage_laser_scan_device(kicp_ctx *c, const kicp_laser_scan *scan, double stamp_range[2], int64_t *n_points) {
    return stage_laser_scan(c, scan, stamp_range, n_points, true);
}

// The second half: kicp_register_frame on the frame kicp_frame_stage left on the device.
extern "C" int kicp_register_staged_frame(kicp_map *map, const double deskew_motion[7], const double lidar_to_base[7], const double last_pose[7],
                                          const double relative_odometry[7], double tau, const kicp_frame_params *fp, double out_pose[7],
                                          double *out_frame, int64_t cap_frame, int64_t *n_frame, double *out_source, int64_t cap_source,
                                          int64_t *n_source, kicp_reg_result *result) {
    if (!map) return KICP_ERR_INVALID;
    Scratch &s = scratch(map->ctx);
    const FrameArgs a{s.held_n, nullptr, s.held_n_stamps, true, deskew_motion, lidar_to_base, last_pose, relative_odometry, tau, fp,
                      out_pose, out_frame, cap_frame, n_frame, out_source, cap_source, n_source, result, std::chrono::steady_clock::now()};
    // the staged frame is consumed, whatever the outcome (its points are in the scratch already)
    KICP_TRY(open_frontend(map->ctx, a.n >= 0 && s.held_k == 1 && a.valid() ? KICP_OK : KICP_ERR_INVALID, a.n));
    if (n_frame) *n_frame = 0;
    if (n_source) *n_source = 0;
    return register_ingested(map, s, a);
}

// The first half for K sensors: each sensor is ingested at its own place of the staged frame — sensor k owns [base_k, base_k + n_k)
// of s.in and s.stamps, n_k being its record or beam count, so a LaserScan's dropped beams leave a hole at the end of its place — with
// no host round trip in between; then k_stamp_minmax_sensors puts the stamps on the common clock and reduces the window.  The window,
// the per-sensor ranges and the kept beam counts come back with one host synchronisation.
extern "C" int kicp_frame_stage_sensors(kicp_ctx *c, const kicp_sensor_input *sensors, int32_t k, double stamp_range[2],
                                        kicp_sensor_stats *stats) {
    Layout layout[kMaxSensors];
    int64_t base[kMaxSensors + 1] = {0};
    size_t raw_off[kMaxSensors + 1] = {0};
    auto validate = [&]() -> int {
        if (!c || !sensors || !stamp_range || k < 1 || k > kMaxSensors) {
            kicp_set_error("kicp_frame_stage_sensors: a null argument, or k outside [1, KICP_MAX_SENSORS]");
            return KICP_ERR_INVALID;
        }
        for (int i = 0; i < k; ++i) {
            const kicp_sensor_input &in = sensors[i];
            const bool device = in.device != 0;
            const std::string where = "kicp_frame_stage_sensors: sensors[" + std::to_string(i) + "].";
            int st = KICP_OK;
            bool range_error = false;
            int64_t n = 0;
            size_t raw = 0;
            if (!std::isfinite(in.time_offset) || (in.kind != KICP_SENSOR_POINTS && in.kind != KICP_SENSOR_LASER_SCAN)) {
                st = KICP_ERR_INVALID;
            } else if (in.kind == KICP_SENSOR_POINTS) {
                st = check_frame_stage(c, &in.points, in.stamp_datatype, in.stamp_offset, device, layout[i], where + "points.",
                                       &range_error);
                n = in.points.n;
                raw = device ? 0 : (size_t)n * (st == KICP_OK ? layout[i].step : 0);
            } else {
                st = check_laser_scan(c, &in.scan, device, where + "scan.ranges", &range_error);
                n = in.scan.n, raw = device ? 0 : (size_t)n * sizeof(float);
            }
            if (st != KICP_OK) {
                // a device-range check has named the pointer; every other rejection names the sensor here
                if (!range_error) kicp_set_error(where.substr(0, where.size() - 1) + ": " + kicp_status_string(st));
                return st;
            }
            base[i + 1] = base[i] + n;
            raw_off[i + 1] = raw_off[i] + (raw + 15) / 16 * 16;
        }
        if (base[k] <= 0x3FFFFFFF) return KICP_OK;
        kicp_set_error("kicp_frame_stage_sensors: more than 2^30 - 1 points in all sensors");
        return KICP_ERR_INVALID;
    };
    const int status = validate();
    KICP_TRY(open_frontend(c, status, status == KICP_OK ? base[k] : 0));
    Scratch &s = scratch(c);
    Frontend &f = frontend(c);
    stamp_range[0] = stamp_range[1] = 0.0;
    if (stats)
        for (int i = 0; i < k; ++i) stats[i] = kicp_sensor_stats{0, 0, {0.0, 0.0}};
    // every table refreshed and the upload buffer sized before anything is enqueued (a regrown buffer drops what is in flight)
    for (int i = 0; i < k; ++i)
        if (sensors[i].kind == KICP_SENSOR_LASER_SCAN) KICP_TRY(f.laser[i].refresh(&sensors[i].scan, "kicp_frame_stage_sensors"));
    if (raw_off[k] > 0) KICP_TRY(reserve_raw(c, s, raw_off[k]));
    SensorStampArgs ma;
    ma.k = k;
    int64_t widest = 0;
    for (int i = 0; i < kMaxSensors; ++i) {
        const kicp_sensor_input *in = i < k ? &sensors[i] : nullptr;
        const bool laser = in && in->kind == KICP_SENSOR_LASER_SCAN;
        const int64_t n = in ? base[i + 1] - base[i] : 0;
        const bool stamped = laser || (in && (in->stamp_datatype != 0 || in->points.n_stamps > 0));
        ma.seg[i] = SensorStampSeg{(int)base[std::min(i, (int)k)], (int)n, laser ? i : -1, stamped && n > 0 ? 1 : 0, in ? in->time_offset : 0.0};
        widest = std::max(widest, n);
        if (n == 0) continue;
        const bool device = in->device != 0;
        if (laser) {
            KICP_TRY(enqueue_laser(c, s, f.laser[i], &in->scan, device, base[i], raw_off[i], reinterpret_cast<double *>(s.out) + base[i],
                                   s.d_seg_count + i));
            continue;
        }
        const StampArgs t{in->stamp_datatype, in->stamp_offset};
        KICP_TRY(enqueue_ingest(c, s, &in->points, layout[i], in->stamp_datatype != 0 ? &t : nullptr, device, base[i], raw_off[i]));
        if (in->stamp_datatype == 0 && in->points.n_stamps > 0)
            KICP_CUDA(cudaMemcpyAsync(s.stamps + base[i], in->points.stamps, (size_t)n * sizeof(double),
                                      device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
    }
    if (base[k] > 0) {
        ma.grid = (int)std::min<int64_t>(kSensorMinMaxMaxGrid, (widest + 2047) / 2048);
        k_stamp_minmax_sensors<<<(unsigned)(k * ma.grid), 256, 0, c->stream>>>(s.stamps, s.d_seg_count, ma,
                                                                                 s.d_seg_mm + 2 * kMaxSensors, s.d_mm_ticket, s.d_seg_mm, s.d_mm);
        KICP_CHECK_LAUNCH(c);
        KICP_CUDA(cudaMemcpyAsync(s.h_range, s.d_mm, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaMemcpyAsync(s.h_seg_mm, s.d_seg_mm, 2 * k * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaMemcpyAsync(s.h_seg_count, s.d_seg_count, k * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
    }
    int64_t kept = 0, n_stamps = 0;
    for (int i = 0; i < k; ++i) {
        const SensorStampSeg &g = ma.seg[i];
        const int count = g.count_slot >= 0 && g.n > 0 ? std::min(s.h_seg_count[i], g.n) : g.n;
        const bool stamped = g.stamped && count > 0;
        s.held[i] = {g.base, count, stamped};
        kept += count, n_stamps += stamped ? count : 0;
        if (stats) {
            stats[i].n_points = count, stats[i].n_stamps = stamped ? count : 0;
            if (stamped) stats[i].stamp_range[0] = s.h_seg_mm[2 * i], stats[i].stamp_range[1] = s.h_seg_mm[2 * i + 1];
        }
    }
    if (n_stamps > 0) stamp_range[0] = s.h_range[0], stamp_range[1] = s.h_range[1];
    s.held_n = kept, s.held_n_stamps = n_stamps, s.held_k = k, s.held_extent = base[k];
    s.held_range[0] = stamp_range[0], s.held_range[1] = stamp_range[1];
    return KICP_OK;
}

// The multi-sensor frame calls refuse free-space clearing: the down-sampled frame no longer knows which sensor a point came from
static const char kMultiSensorFree[] =
    "free-space clearing (kicp_ctx_set_free_space) needs a single-sensor frame: clear once per sensor with kicp_map_clear_free_space";

// The second half for K sensors: kicp_register_staged_frame with a de-skew motion and an extrinsic per sensor of the staged frame.
extern "C" int kicp_register_staged_sensors(kicp_map *map, int32_t k, const double deskew_motions[][7], const double lidar_to_bases[][7],
                                            const double last_pose[7], const double relative_odometry[7], double tau,
                                            const kicp_frame_params *fp, double out_pose[7], double *out_frame, int64_t cap_frame,
                                            int64_t *n_frame, double *out_source, int64_t cap_source, int64_t *n_source,
                                            kicp_reg_result *result) {
    if (!map) return KICP_ERR_INVALID;
    Scratch &s = scratch(map->ctx);
    const bool tables = deskew_motions && lidar_to_bases;
    FrameArgs a{s.held_n, nullptr, s.held_n_stamps, true, tables ? deskew_motions[0] : nullptr, tables ? lidar_to_bases[0] : nullptr,
                last_pose, relative_odometry, tau, fp, out_pose, out_frame, cap_frame, n_frame, out_source, cap_source, n_source, result,
                std::chrono::steady_clock::now()};
    a.deskew_motions = deskew_motions, a.lidar_to_bases = lidar_to_bases;
    // the staged frame is consumed, whatever the outcome (its points are in the scratch already)
    int valid = a.n >= 0 && k == s.held_k && a.valid() ? KICP_OK : KICP_ERR_INVALID;
    if (valid == KICP_OK && map->ctx->free_space.min_misses > 0) valid = kicp_invalid("kicp_register_staged_sensors", kMultiSensorFree);
    KICP_TRY(open_frontend(map->ctx, valid, a.n));
    if (n_frame) *n_frame = 0;
    if (n_source) *n_source = 0;
    return register_ingested(map, s, a);
}

namespace {
bool finite_pose(const double p[7]) {
    for (int k = 0; k < 7; ++k)
        if (!std::isfinite(p[k])) return false;
    return true;
}
// Sophus SE3::inverse of a pose7: conjugate rotation, t' = -(q^-1 t)
void pose_inverse_host(const double p[7], double out[7]) {
    const double qx = -p[0], qy = -p[1], qz = -p[2], qw = p[3];
    const double ux = 2.0 * (qy * p[6] - qz * p[5]), uy = 2.0 * (qz * p[4] - qx * p[6]), uz = 2.0 * (qx * p[5] - qy * p[4]);
    out[0] = qx, out[1] = qy, out[2] = qz, out[3] = qw;
    out[4] = -(p[4] + qw * ux + (qy * uz - qz * uy));
    out[5] = -(p[5] + qw * uy + (qz * ux - qx * uz));
    out[6] = -(p[6] + qw * uz + (qx * uy - qy * ux));
}
bool identity_pose(const double p[7]) {
    return p[0] == 0.0 && p[1] == 0.0 && p[2] == 0.0 && p[3] == 1.0 && p[4] == 0.0 && p[5] == 0.0 && p[6] == 0.0;
}
// the checks of one sensor's segment table; `cover`: the table must cover the window win = {T0, T1} (a stamped sensor, de-skew on)
int check_segments(const char *fn, const std::string &where, int32_t n, const kicp_deskew_segment *segs, bool cover, const double win[2]) {
    auto fail = [&](const std::string &why) { return kicp_invalid(fn, (where + why).c_str()); };
    if (n < 1 || n > KICP_MAX_DESKEW_SEGMENTS) return fail(" count outside [1, KICP_MAX_DESKEW_SEGMENTS]");
    if (!segs) return fail(": null pointer");
    for (int j = 0; j < n; ++j) {
        const kicp_deskew_segment &g = segs[j];
        const std::string at = "[" + std::to_string(j) + "]";
        if (!std::isfinite(g.t_begin) || !std::isfinite(g.t_end)) return fail(at + ": a non-finite time");
        if (!(g.t_begin < g.t_end)) return fail(at + ": t_begin >= t_end");
        if (!finite_pose(g.motion)) return fail(at + ".motion: not finite");
        if (!finite_pose(g.to_end)) return fail(at + ".to_end: not finite");
        if (j > 0 && segs[j - 1].t_end != g.t_begin) return fail(at + ".t_begin != [" + std::to_string(j - 1) + "].t_end (a gap or an overlap)");
    }
    if (cover && !(segs[0].t_begin <= win[0] && segs[n - 1].t_end >= win[1])) return fail(": does not cover the staged window [T0, T1]");
    return KICP_OK;
}

// kicp_register_staged_frame_segments (`single`: the staged frame must be of one sensor) and kicp_register_staged_sensors_segments:
// validation before any device work, the tables packed into pinned memory and copied on the context stream, then the frame.
int register_staged_segments(kicp_map *map, int32_t k, const int32_t *n_segments, const kicp_deskew_segment *const *segments,
                             const double (*lidar_to_bases)[7], bool single, const double last_pose[7], const double relative_odometry[7],
                             double tau, const kicp_frame_params *fp, double out_pose[7], double *out_frame, int64_t cap_frame,
                             int64_t *n_frame, double *out_source, int64_t cap_source, int64_t *n_source, kicp_reg_result *result,
                             const char *fn) {
    if (!map) return kicp_invalid(fn, "map: null pointer");
    kicp_ctx *c = map->ctx;
    Scratch &s = scratch(c);
    static const double kUnused[7] = {0, 0, 0, 1, 0, 0, 0};  // FrameArgs' deskew_motion: the segments de-skew instead
    FrameArgs a{s.held_n, nullptr, s.held_n_stamps, true, kUnused, lidar_to_bases ? lidar_to_bases[0] : nullptr, last_pose,
                relative_odometry, tau, fp, out_pose, out_frame, cap_frame, n_frame, out_source, cap_source, n_source, result,
                std::chrono::steady_clock::now()};
    const bool deskew = fp && fp->deskew && s.held_n_stamps > 0;
    auto validate = [&]() -> int {
        if (!lidar_to_bases) return kicp_invalid(fn, single ? "lidar_to_base: null pointer" : "lidar_to_bases: null pointer");
        if (!last_pose) return kicp_invalid(fn, "last_pose: null pointer");
        if (!relative_odometry) return kicp_invalid(fn, "relative_odometry: null pointer");
        if (!fp) return kicp_invalid(fn, "fp: null pointer");
        if (!out_pose) return kicp_invalid(fn, "out_pose: null pointer");
        if (!(fp->voxel_size > 0.0)) return kicp_invalid(fn, "fp->voxel_size is not > 0");
        if (!n_segments || !segments) return kicp_invalid(fn, single ? "segments: null pointer" : "n_segments / segments: null pointer");
        if (s.held_n < 0) return kicp_invalid(fn, "no staged frame");
        if (single && s.held_k != 1) return kicp_invalid(fn, "the staged frame has several sensors");
        if (k != s.held_k) return kicp_invalid(fn, "k differs from the staged frame's sensor count");
        if (!single && c->free_space.min_misses > 0) return kicp_invalid(fn, kMultiSensorFree);
        for (int i = 0; i < k; ++i) {
            const std::string where = single ? "segments" : "segments[" + std::to_string(i) + "]";
            KICP_TRY(check_segments(fn, where, n_segments[i], segments[i], deskew && s.held[i].stamped, s.held_range));
        }
        return KICP_OK;
    };
    // the staged frame is consumed, whatever the outcome (its points are in the scratch already)
    KICP_TRY(open_frontend(c, validate(), a.n));
    if (n_frame) *n_frame = 0;
    if (n_source) *n_source = 0;
    SegmentPreArgs pa;
    pa.k = k;
    int first = 0;
    bool any = false;
    for (int i = 0; i < kMaxSensors; ++i) {
        SegmentSensor &g = pa.seg[i];
        const bool used = i < k;
        g.base = used ? s.held[i].base : 0, g.count = used ? s.held[i].count : 0;
        g.deskew = used && deskew && s.held[i].stamped ? 1 : 0;
        g.first = first, g.n_seg = g.deskew ? n_segments[i] : 0;
        first += g.n_seg, any = any || g.deskew;
        PreArgs &p = g.pre;
        p.deskew = 0, p.max_range = fp->max_range, p.min_range = fp->min_range;
        const double *l2b = used ? lidar_to_bases[i] : nullptr;
        p.lidar_to_base = l2b ? Pose{l2b[0], l2b[1], l2b[2], l2b[3], l2b[4], l2b[5], l2b[6]} : Pose{0, 0, 0, 1, 0, 0, 0};
        for (int j = 0; j < 6; ++j) p.omega[j] = 0.0;
    }
    if (a.n > 0 && any) {
        if (!s.d_segs) {
            const size_t bytes = (size_t)kMaxSensors * kMaxDeskewSegments * sizeof(DeskewSeg);
            KICP_CUDA(cudaMalloc(&s.d_segs, bytes));
            KICP_CUDA(cudaMallocHost(&s.h_segs, bytes));
            KICP_CUDA(cudaEventCreateWithFlags(&s.ev_segs, cudaEventDisableTiming));
            s.segs_pending = false;
        }
        if (s.segs_pending) KICP_CUDA(cudaEventSynchronize(s.ev_segs));
        for (int i = 0; i < k; ++i)
            for (int j = 0; j < pa.seg[i].n_seg; ++j) {
                const kicp_deskew_segment &in = segments[i][j];
                DeskewSeg &d = s.h_segs[pa.seg[i].first + j];
                d.t_begin = in.t_begin, d.t_end = in.t_end;
                se3_log_host(in.motion, d.omega);
                double e[7];  // the kernel takes a point from the frame at t_end to the frame at T1: the inverse of that motion
                pose_inverse_host(in.to_end, e);
                d.to_end = Pose{e[0], e[1], e[2], e[3], e[4], e[5], e[6]};
                d.identity = identity_pose(in.to_end) ? 1 : 0;
            }
        KICP_CUDA(cudaMemcpyAsync(s.d_segs, s.h_segs, (size_t)first * sizeof(DeskewSeg), cudaMemcpyHostToDevice, c->stream));
        KICP_CUDA(cudaEventRecord(s.ev_segs, c->stream));
        s.segs_pending = true;
    }
    a.segments = &pa;
    return register_ingested(map, s, a);
}
}  // namespace

// kicp_register_staged_frame with the de-skew of a segment table (include/kicp.h)
extern "C" int kicp_register_staged_frame_segments(kicp_map *map, int32_t n_segments, const kicp_deskew_segment *segments,
                                                   const double lidar_to_base[7], const double last_pose[7], const double relative_odometry[7],
                                                   double tau, const kicp_frame_params *fp, double out_pose[7], double *out_frame,
                                                   int64_t cap_frame, int64_t *n_frame, double *out_source, int64_t cap_source,
                                                   int64_t *n_source, kicp_reg_result *result) {
    return register_staged_segments(map, 1, &n_segments, &segments, reinterpret_cast<const double(*)[7]>(lidar_to_base), true, last_pose,
                                    relative_odometry, tau, fp, out_pose, out_frame, cap_frame, n_frame, out_source, cap_source, n_source,
                                    result, "kicp_register_staged_frame_segments");
}

// kicp_register_staged_sensors with a segment table per sensor (include/kicp.h)
extern "C" int kicp_register_staged_sensors_segments(kicp_map *map, int32_t k, const int32_t n_segments[],
                                                     const kicp_deskew_segment *const segments[], const double lidar_to_bases[][7],
                                                     const double last_pose[7], const double relative_odometry[7], double tau,
                                                     const kicp_frame_params *fp, double out_pose[7], double *out_frame, int64_t cap_frame,
                                                     int64_t *n_frame, double *out_source, int64_t cap_source, int64_t *n_source,
                                                     kicp_reg_result *result) {
    return register_staged_segments(map, k, n_segments, segments, lidar_to_bases, false, last_pose, relative_odometry, tau, fp, out_pose,
                                    out_frame, cap_frame, n_frame, out_source, cap_source, n_source, result,
                                    "kicp_register_staged_sensors_segments");
}

/* The clouds of the last kicp_register_frame on this context (fp->stage_clouds), in context-owned pinned host memory, valid
 * until the next kicp_register_frame / kicp_preprocess / kicp_voxel_downsample call on the same context. */
extern "C" int kicp_frame_clouds(kicp_ctx *c, const double **frame, int64_t *n_frame, const double **source, int64_t *n_source) {
    if (!c || !frame || !n_frame || !source || !n_source) return KICP_ERR_INVALID;
    const Staging &st = scratch(c).staged;
    *frame = reinterpret_cast<const double *>(st.frame), *n_frame = st.n_frame;
    *source = reinterpret_cast<const double *>(st.source), *n_source = st.n_source;
    return KICP_OK;
}

// The same clouds as float32 records (fp->stage_clouds & KICP_STAGE_F32), encoded on the device; same lifetime
extern "C" int kicp_frame_clouds_f32(kicp_ctx *c, const float **frame, int64_t *n_frame, const float **source, int64_t *n_source) {
    if (!c || !frame || !n_frame || !source || !n_source) return KICP_ERR_INVALID;
    const Staging &st = scratch(c).staged;
    *frame = st.frame32, *n_frame = st.n_frame32;
    *source = st.source32, *n_source = st.n_source32;
    return KICP_OK;
}

// The same clouds in context-owned device memory: packed xyz doubles (F64, no staging flag needed) or the float32 records
// k_encode_clouds wrote (F32, frames with KICP_STAGE_F32); not a front-end call
extern "C" int kicp_frame_clouds_device(kicp_ctx *c, int32_t dtype, const void **frame, int64_t *n_frame, const void **source,
                                        int64_t *n_source) {
    if (!c || !frame || !n_frame || !source || !n_source || (dtype != KICP_DTYPE_F64 && dtype != KICP_DTYPE_F32)) return KICP_ERR_INVALID;
    const Scratch &s = scratch(c);
    const bool f64 = dtype == KICP_DTYPE_F64, ok = f64 || s.dev_f32;
    *frame = f64 ? static_cast<const void *>(s.out) : s.staged.d_rec;
    *source = f64 ? static_cast<const void *>(s.out3) : s.staged.d_rec ? s.staged.d_source_rec() : nullptr;
    *n_frame = ok ? s.dev_n_frame : 0, *n_source = ok ? s.dev_n_source : 0;
    return KICP_OK;
}

// The correspondence report of the last frame (option "correspondences"): its statistics, and the per-point results in context-owned
// device memory; not a front-end call
extern "C" int kicp_frame_correspondences(kicp_ctx *c, kicp_corr_stats *stats) {
    static const char fn[] = "kicp_frame_correspondences";
    if (!stats) return kicp_invalid(fn, "stats: null pointer");
    if (!c) return kicp_invalid(fn, "null context");
    *stats = scratch(c).corr;
    return KICP_OK;
}
extern "C" int kicp_frame_correspondences_device(kicp_ctx *c, const double **points, const double **dist, const uint8_t **inlier,
                                                 int64_t *n) {
    static const char fn[] = "kicp_frame_correspondences_device";
    if (!points) return kicp_invalid(fn, "points: null pointer");
    if (!dist) return kicp_invalid(fn, "dist: null pointer");
    if (!inlier) return kicp_invalid(fn, "inlier: null pointer");
    if (!n) return kicp_invalid(fn, "n: null pointer");
    if (!c) return kicp_invalid(fn, "null context");
    const Scratch &s = scratch(c);
    *points = reinterpret_cast<const double *>(s.corr_pts), *dist = s.corr_dist, *inlier = s.corr_inl;
    *n = s.corr_n;
    return KICP_OK;
}

// The map-update policy of the frame calls (kicp_map_update.h): checked field by field, the context last; a failing call keeps the
// previous policy
extern "C" int kicp_ctx_set_map_update(kicp_ctx *c, const kicp_map_update_policy *policy) {
    static const char fn[] = "kicp_ctx_set_map_update";
    if (!policy) return kicp_invalid(fn, "policy: null pointer");
    const kicp_map_update_policy &p = *policy;
    if (p.mode < KICP_MAP_UPDATE_ALWAYS || p.mode > KICP_MAP_UPDATE_GATED) return kicp_invalid(fn, "policy->mode: not in 0..2");
    if (p.min_inliers < 0) return kicp_invalid(fn, "policy->min_inliers: negative");
    if (!(p.min_fitness >= 0.0 && p.min_fitness <= 1.0)) return kicp_invalid(fn, "policy->min_fitness: not in [0, 1]");
    if (!(p.max_inlier_rmse > 0.0)) return kicp_invalid(fn, "policy->max_inlier_rmse: not > 0");
    if (!c) return kicp_invalid(fn, "null context");
    c->map_update = p;
    return KICP_OK;
}

// The free-space clearing of the frame calls: checked field by field, the context last; a failing call keeps the previous setting
extern "C" int kicp_ctx_set_free_space(kicp_ctx *c, const kicp_free_space_params *params) {
    static const char fn[] = "kicp_ctx_set_free_space";
    if (!params) return kicp_invalid(fn, "params: null pointer");
    KICP_TRY(kicp_check_free_space_params(fn, params, true));
    if (!c) return kicp_invalid(fn, "null context");
    c->free_space = *params;
    return KICP_OK;
}

// The free-space statistics of the last frame call; not a front-end call
extern "C" int kicp_frame_free_space(kicp_ctx *c, kicp_free_space_stats *stats) {
    static const char fn[] = "kicp_frame_free_space";
    if (!stats) return kicp_invalid(fn, "stats: null pointer");
    if (!c) return kicp_invalid(fn, "null context");
    *stats = scratch(c).free_space;
    return KICP_OK;
}

// The map-update outcome of the last frame call; not a front-end call
extern "C" int kicp_frame_map_update(kicp_ctx *c, int32_t *outcome) {
    static const char fn[] = "kicp_frame_map_update";
    if (!outcome) return kicp_invalid(fn, "outcome: null pointer");
    if (!c) return kicp_invalid(fn, "null context");
    *outcome = scratch(c).map_update;
    return KICP_OK;
}

// debugging aid (not part of the public header): cumulative host-side stage times of the last kicp_register_frame, ms
extern "C" int kicp_debug_frame_timing(kicp_ctx *c, double out[8]) {
    if (!c || !out) return KICP_ERR_INVALID;
    for (int k = 0; k < 8; ++k) out[k] = scratch(c).timing[k];
    return KICP_OK;
}
