// Host side of the registration path: options, scratch, the chunked upload, the launch sequence, profiling, and the C ABI
// entry points of include/kicp.h for KinematicRegistration::ComputeRobotMotion (registration/Registration.hpp:39-43).
// The kernels live in kicp_register.cu; this file reaches them through kicp_register.cuh.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "kicp_register.cuh"

// Per-context options (kicp_ctx_set_option): "persistent" 1 = one cooperative launch per registration (default), 0 = one
// launch per IRLS iteration; "stats" 1 = count probes / candidate points / lines on the device (kicp_debug_last_stats);
// "ctas_per_sm" caps the resident CTAs per SM the grid is sized for (0 = occupancy limit); "nn_cache" 0 / 1 / 2 = never / for scans of
// 49152 points or more (default) / always carry every point's neighbour and its certificate from pass to pass; "spin_timeout_ms" bounds every device-side wait.
extern "C" int kicp_ctx_set_option(kicp_ctx *c, const char *name, int32_t value) {
    if (!c || !name) return KICP_ERR_INVALID;
    if (!strcmp(name, "persistent")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->persistent = value;
    } else if (!strcmp(name, "stats")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->collect_stats = value;
    } else if (!strcmp(name, "ctas_per_sm")) {
        if (value < 0 || value > 16) return KICP_ERR_INVALID;
        c->ctas_per_sm_cap = value;
    } else if (!strcmp(name, "spin_timeout_ms")) {
        if (value < 1) return KICP_ERR_INVALID;
        c->spin_timeout_ms = value;
    } else if (!strcmp(name, "nn_cache")) {
        if (value < 0 || value > 2) return KICP_ERR_INVALID;
        c->nn_cache = value;
    } else if (!strcmp(name, "overlap_upload")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->overlap_upload = value;
    } else if (!strcmp(name, "frame_sync")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->frame_sync = value;
    } else if (!strcmp(name, "downsample_order")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->downsample_order = value;
    } else if (!strcmp(name, "correspondences")) {
        if (value != 0 && value != 1) return KICP_ERR_INVALID;
        c->correspondences = value;
    } else {
        kicp_set_error(std::string("kicp_ctx_set_option: unknown option ") + name);
        return KICP_ERR_INVALID;
    }
    return KICP_OK;
}

// Profiling record of one registration (kicp_ctx_profile_begin / end): CUDA events on the context stream.
struct EventPair {
    cudaEvent_t begin = nullptr, end = nullptr;
};
struct ProfReg {
    EventPair prep;              // the set-up: the stats reset and k_reg_init
    std::vector<EventPair> it;   // one per launch of k_register
    bool persistent = false;     // one launch covers every iteration
    int32_t *d_iters = nullptr;  // device word receiving the registration's iteration count
};
static constexpr int64_t kProfCap = 1 << 16;  // registrations recorded between kicp_ctx_profile_begin and _end

// The registration's scratch on one context (kicp_ctx::reg): the upload flags from kicp_ctx_create on, the rest from first use.
struct RegScratch {
    RegState *d_state = nullptr;
    double *d_partials = nullptr;    // per-CTA partial sums of the registration kernel [2][grid][8]
    int pruned_ctas_per_sm = 1;      // resident CTAs per SM of k_register<false> (occupancy query)
    int persistent_ctas_per_sm = 1;  // ... of k_register<true>
    // nearest-neighbour cache of the persistent kernel, one entry per scan point carried from pass to pass: the five 4-byte arrays
    // nn_g, nn_g2, nn_l, todo and todo2 of nn_cap entries each, every one starting on a multiple of 64 entries (256 bytes)
    unsigned int *d_nn = nullptr;
    int64_t nn_cap = 0;
    // chunked upload of the host-pointer entry points, overlapped with the first IRLS pass of the persistent kernel
    uint32_t *d_chunk_flags = nullptr;  // [KICP_UPLOAD_CHUNKS] raised (to the upload sequence number) chunk by chunk
    uint32_t *h_chunk_tags = nullptr;   // pinned source of the flag copies
    uint32_t upload_seq = 0;
    kicp_scan *upload_scan = nullptr;   // staging scan of the host-pointer entry points
    bool profiling = false;
    std::vector<ProfReg> prof;
    int32_t *d_prof_iters = nullptr;  // [kProfCap]
};

void kicp_reg_scratch_free(kicp_ctx *c) {
    RegScratch *s = c->reg;
    if (!s) return;
    if (s->upload_scan) kicp_scan_destroy(s->upload_scan);
    cudaFree(s->d_state), cudaFree(s->d_partials), cudaFree(s->d_nn), cudaFree(s->d_chunk_flags), cudaFree(s->d_prof_iters);
    cudaFreeHost(s->h_chunk_tags);
    delete s;
    c->reg = nullptr;
}

int kicp_reg_scratch_create(kicp_ctx *c) {
    RegScratch *s = c->reg = new RegScratch();
    KICP_CUDA(cudaMalloc(&s->d_chunk_flags, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    KICP_CUDA(cudaMemset(s->d_chunk_flags, 0, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    KICP_CUDA(cudaMallocHost(&s->h_chunk_tags, KICP_UPLOAD_CHUNKS * sizeof(uint32_t)));
    return kicp_scan_create(c, 0, &s->upload_scan);  // (no device memory until the first host frame)
}

// The kernel's state and partial sums, allocated by the first registration.  A device without cooperative launch runs one launch
// per pass.
static int reg_reserve(kicp_ctx *c) {
    RegScratch &s = *c->reg;
    if (s.d_state) return KICP_OK;
    KICP_CUDA(cudaMalloc((void **)&s.d_state, kr_state_bytes()));
    KICP_CUDA(cudaMemset(s.d_state, 0, kr_state_bytes()));
    int per_sm_p = 0, per_sm_m = 0;
    KICP_CUDA(kr_prepare(&per_sm_p, &per_sm_m));
    s.persistent_ctas_per_sm = std::max(per_sm_p, 1);
    s.pruned_ctas_per_sm = std::max(per_sm_m, 1);
    const int max_grid = c->sm_count * std::max(s.persistent_ctas_per_sm, s.pruned_ctas_per_sm);
    KICP_CUDA(cudaMalloc(&s.d_partials, (size_t)2 * max_grid * 8 * sizeof(double)));
    int coop = 0;
    KICP_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device));
    if (!coop) c->persistent = 0;
    return KICP_OK;
}

// Everything the arguments of a registration can get wrong, checked by every entry point before any device work.  `owner`: the
// context the n points at `points` live on.
static int check_registration(const kicp_map *m, const kicp_ctx *owner, int64_t n, const void *points, const double *last,
                              const double *odom, const kicp_reg_params *p, bool sharded) {
    if (!m || !owner || n < 0 || (n > 0 && !points) || !last || !odom || !p) return KICP_ERR_INVALID;
    if (p->max_num_iterations > KICP_MAX_ITERATIONS) {
        kicp_set_error("max_num_iterations exceeds KICP_MAX_ITERATIONS");
        return KICP_ERR_INVALID;
    }
    if (owner != m->ctx) return KICP_ERR_INVALID;
    if (n > 0x7FFFFFE0ll) return KICP_ERR_CAPACITY;
    if (sharded && !m->ctx->nccl_comm && !m->ctx->p2p_ready) {
        kicp_set_error("kicp_register_sharded: neither kicp_comm_p2p_init nor kicp_comm_init has been called on this context");
        return KICP_ERR_INVALID;
    }
    return KICP_OK;
}

// Host side of the chunked upload: the frame's bytes go out in KICP_UPLOAD_CHUNKS pieces on the copy stream, each followed
// by a 4-byte flag copy; the persistent kernel's first pass waits per chunk on the flag, so the association starts while
// later chunks are still on the bus.
static int issue_chunks(kicp_ctx *c, const void *host_src, const KernelArgs &ka) {
    const unsigned char *src = static_cast<const unsigned char *>(host_src);
    unsigned char *dst = const_cast<unsigned char *>(ka.scan.base);
    const int64_t n = ka.scan.n, stride = ka.scan.stride, wpc = ka.up.windows_per_chunk;
    // The kernel always sees KICP_UPLOAD_CHUNKS segments; the host groups them into copies of at least ~384 KB (a small frame is
    // ONE copy and one flag copy: every DMA operation costs microseconds, which a 24 KB scan cannot win back by overlapping).
    const int copies = (int)std::max<int64_t>(1, std::min<int64_t>(KICP_UPLOAD_CHUNKS, n * stride / (384 << 10)));
    for (int j = 0; j < copies; ++j) {
        const int k0 = j * KICP_UPLOAD_CHUNKS / copies, k1 = (j + 1) * KICP_UPLOAD_CHUNKS / copies;  // segments [k0, k1)
        const int64_t lo = std::min<int64_t>(n, k0 * wpc * 32), hi = std::min<int64_t>(n, k1 * wpc * 32);
        if (hi > lo)
            KICP_CUDA(cudaMemcpyAsync(dst + lo * stride, src + lo * stride, (size_t)((hi - lo) * stride), cudaMemcpyHostToDevice,
                                      c->copy_stream));
        KICP_CUDA(cudaMemcpyAsync(c->reg->d_chunk_flags + k0, c->reg->h_chunk_tags + k0, (size_t)(k1 - k0) * sizeof(uint32_t),
                                  cudaMemcpyHostToDevice, c->copy_stream));
    }
    return KICP_OK;
}

static ScanView scan_view(const kicp_scan *s) {
    ScanView v;
    v.base = (const unsigned char *)s->data(), v.n = (int)s->n, v.d_n = s->d_n;
    v.stride = s->stride, v.ox = s->ox, v.oy = s->oy, v.oz = s->oz, v.f32 = s->dtype == KICP_DTYPE_F32 ? 1 : 0;
    return v;
}

// Enqueues `work` on the context stream between the two events of `ev`, which it creates (ev == nullptr: not profiled).
template <class Work>
static int between_events(kicp_ctx *c, EventPair *ev, Work &&work) {
    if (ev) {
        KICP_CUDA(cudaEventCreate(&ev->begin));
        KICP_CUDA(cudaEventCreate(&ev->end));
        KICP_CUDA(cudaEventRecord(ev->begin, c->stream));
    }
    KICP_TRY(work());
    if (ev) KICP_CUDA(cudaEventRecord(ev->end, c->stream));
    return KICP_OK;
}

// Enqueue one registration on the context stream (check_registration has accepted the arguments).  `n_hint`: see
// kicp_enqueue_registration_device.  `host_src`: a host frame to copy into `scan`.  `sharded`: this rank holds a contiguous index
// range of the frame; the 8 sums of every iteration are exchanged (fused peer-memory exchange after kicp_comm_p2p_init, else NCCL).
static int enqueue_registration(kicp_map *m, const ScanView &scan, int64_t n_hint, const double last[7], const double odom[7],
                                double tau, const kicp_reg_params *p, kicp_reg_result *result, bool sharded,
                                const void *host_src = nullptr) {
    kicp_ctx *c = m->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(reg_reserve(c));
    RegScratch &s = *c->reg;
    // The plan.  An empty map returns the prediction (Registration.cpp:157).  A persistent launch with work in it runs the set-up and
    // every pass; otherwise k_reg_init runs first, then k_register and k_solve once per pass (which the NCCL exchange needs).
    const int max_iter = m->num_blocks == 0 ? 0 : p->max_num_iterations;
    const bool p2p = sharded && c->p2p_ready;
    const bool persistent = c->persistent && (!sharded || p2p) && max_iter > 0;
    // a frame whose exact count is still on the device is planned (grid, certificates) for the count its producer expects
    const int64_t n_plan = (scan.d_n && n_hint > 0) ? std::min<int64_t>(n_hint, scan.n) : scan.n;
    // every CTA is resident and pulls 32-point windows from a device-side counter; a small scan is spread one window per
    // CTA over the whole machine (a window is a chain of dependent memory round trips: latency, not throughput)
    // (the persistent kernel sizes its windows so that a phase that fits one round spreads evenly over the grid: a small scan
    // runs as many tiny windows on the whole machine)
    const int num_windows = persistent ? (int)((n_plan + 7) / 8) : (scan.n + 31) / 32;
    int per_sm = persistent ? s.persistent_ctas_per_sm : s.pruned_ctas_per_sm;
    if (c->ctas_per_sm_cap > 0) per_sm = std::min(per_sm, c->ctas_per_sm_cap);
    const int grid = std::max(1, std::min(num_windows, c->sm_count * per_sm));
    // (1 = automatic: a small scan is one tiny window per warp and gains nothing from the extra phase and its barrier)
    const bool nn_cache = (c->nn_cache == 2 || (c->nn_cache == 1 && n_plan >= 49152)) && scan.n > 0;
    // a host frame goes out in chunks right after the launch, overlapped with the first pass, or else in one copy before the set-up
    const bool overlap = persistent && host_src && scan.n > 0 && c->overlap_upload;
    // A result block in page-locked host memory (kicp_host_alloc, the context's own staging) is written by the persistent kernel
    // itself; anything else is filled by a copy after the kernel.
    kicp_reg_result *result_host = nullptr;
    cudaPointerAttributes at;
    if (persistent && result && cudaPointerGetAttributes(&at, result) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer)
        result_host = static_cast<kicp_reg_result *>(at.devicePointer);
    else if (persistent && result)
        cudaGetLastError();  // (ordinary memory: not an error, just not ours to write)

    KernelArgs ka{};
    ka.st = s.d_state;
    ka.scan = scan;
    ka.map = m->view();
    ka.partials = s.d_partials;
    ka.px.nranks = 1;
    ka.up = UploadArgs{nullptr, 0u, 1};
    ka.init.last = Pose{last[0], last[1], last[2], last[3], last[4], last[5], last[6]};
    ka.init.odom = Pose{odom[0], odom[1], odom[2], odom[3], odom[4], odom[5], odom[6]};
    ka.init.tau = tau, ka.init.conv = p->convergence_criterion, ka.init.fixed_reg = p->fixed_regularization;
    ka.init.adaptive = p->use_adaptive_odometry_regularization ? 1 : 0;
    ka.init.max_iter = max_iter;
    int exp2 = 0;
    ka.pow2_voxel = std::frexp(m->voxel_size, &exp2) == 0.5 ? 1 : 0;
    ka.collect_stats = c->collect_stats;
    ka.timeout_ns = (unsigned long long)c->spin_timeout_ms * 1000000ull;
    ka.result_host = result_host;
    if (host_src && scan.n > 0 && !overlap)
        KICP_CUDA(cudaMemcpyAsync(const_cast<unsigned char *>(scan.base), host_src, (size_t)scan.n * scan.stride, cudaMemcpyHostToDevice,
                                  c->stream));
    if (nn_cache) {
        if (scan.n > s.nn_cap) {
            KICP_CUDA(cudaStreamSynchronize(c->stream));
            cudaFree(s.d_nn);
            s.d_nn = nullptr, s.nn_cap = 0;
            const int64_t cap = scan.n + scan.n / 4 + 1024;
            KICP_CUDA(cudaMalloc(&s.d_nn, (size_t)5 * ((cap + 63) & ~63ll) * sizeof(unsigned int)));
            s.nn_cap = cap;
        }
        const int64_t stride = (s.nn_cap + 63) & ~63ll;
        ka.nn_g = s.d_nn, ka.nn_g2 = s.d_nn + stride, ka.nn_l = reinterpret_cast<float *>(s.d_nn + 2 * stride);
        ka.todo = s.d_nn + 3 * stride, ka.todo2 = s.d_nn + 4 * stride;
    }
    ProfReg *pr = nullptr;
    if (s.profiling && (int64_t)s.prof.size() < kProfCap) {
        pr = &s.prof.emplace_back();
        pr->persistent = persistent;
        pr->d_iters = s.d_prof_iters + (s.prof.size() - 1);
        ka.init.iters_out = pr->d_iters;
    }
    KICP_TRY(between_events(c, pr ? &pr->prep : nullptr, [&]() -> int {
        if (c->collect_stats) KICP_CUDA(cudaMemsetAsync((char *)s.d_state + kr_offset_stats(), 0, kr_stats_bytes(), c->stream));
        if (!persistent) {
            KICP_CUDA(kr_launch_init(s.d_state, ka.init, c->stream));
            c->launches++;
        }
        return KICP_OK;
    }));
    if (overlap) {
        const uint32_t seq = ++s.upload_seq ? s.upload_seq : ++s.upload_seq;  // never 0
        for (int k = 0; k < KICP_UPLOAD_CHUNKS; ++k) s.h_chunk_tags[k] = seq;
        ka.up = UploadArgs{s.d_chunk_flags, seq, ((scan.n + 31) / 32 + KICP_UPLOAD_CHUNKS - 1) / KICP_UPLOAD_CHUNKS};
    }
    if (persistent && p2p) {
        for (int r = 0; r < c->nranks; ++r) ka.px.peer[r] = c->p2p_peer[r];
        ka.px.nranks = c->nranks, ka.px.rank = c->rank;
        ka.px.parity = (int)(c->p2p_seq & 1ull);
        ka.px.tag_base = (uint32_t)((c->p2p_seq * KICP_MAX_ITERATIONS + 1ull) & 0xFFFFFFFFull);
        if (ka.px.tag_base > 0xFFFFFF00u) ka.px.tag_base = 1u, c->p2p_seq = 0;  // wrap (tags stay non-zero)
        c->p2p_seq++;
    }
    const bool dbg = getenv("KICP_DEBUG_SYNC") != nullptr;
    const int passes = persistent ? 1 : max_iter;
    for (int j = 0; j < passes; ++j) {
        KICP_TRY(between_events(c, pr ? &pr->it.emplace_back() : nullptr, [&]() -> int {
            KICP_CUDA(kr_launch_register(persistent, grid, ka, c->stream));
            c->launches++;
            return KICP_OK;
        }));
        if (persistent) {
            // The frame's chunks go out AFTER the launch: the kernel is already resident and takes every chunk as its flag rises, and
            // the host-side cost of the copies (for pageable memory the driver stages each of them on this thread) no longer delays
            // the launch, which matters most to a caller with pageable buffers.
            // (A copy that fails here leaves the kernel to its wait timeout; the call drains both streams and reports the error.)
            if (overlap) KICP_TRY(issue_chunks(c, host_src, ka));
        } else {
            if (sharded) KICP_TRY(kicp_comm_allreduce8(c, (double *)((char *)s.d_state + kr_offset_acc())));
            KICP_CUDA(kr_launch_solve(s.d_state, c->stream));
            c->launches++;
        }
        if (dbg) {
            cudaError_t e = cudaStreamSynchronize(c->stream);
            fprintf(stderr, "[kicp] %s %d of %d (grid %d, n %d): %s\n", persistent ? "persistent launch" : "pass", j, passes, grid, scan.n,
                    cudaGetErrorString(e));
        }
    }
    if (result && !result_host)
        KICP_CUDA(cudaMemcpyAsync(result, (const char *)s.d_state + kr_offset_result(), sizeof(kicp_reg_result), cudaMemcpyDeviceToHost,
                                  c->stream));
    return KICP_OK;
}

const kicp_reg_result *kicp_device_result(kicp_ctx *c) {
    return c && c->reg->d_state ? reinterpret_cast<const kicp_reg_result *>((const char *)c->reg->d_state + kr_offset_result()) : nullptr;
}

// debugging aids (not part of the public header): per-pass device timings and work counters of the last registration
extern "C" int kicp_debug_last_timing(kicp_ctx *c, double *out /* [KICP_MAX_ITERATIONS][6] */) {
    if (!c || !c->reg->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->reg->d_state + kr_offset_dbg(), sizeof(double) * KICP_MAX_ITERATIONS * 6,
                         cudaMemcpyDeviceToHost));
    return KICP_OK;
}
extern "C" int kicp_debug_last_stats(kicp_ctx *c, uint64_t out[4] /* probes, candidate points, 128-byte lines, 0 */) {
    if (!c || !c->reg->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->reg->d_state + kr_offset_stats(), sizeof(uint64_t) * 4, cudaMemcpyDeviceToHost));
    return KICP_OK;
}
extern "C" int kicp_debug_l2_read_bandwidth(kicp_ctx *c, uint64_t bytes, int32_t reps, double *gbps) {
    if (!c || !gbps || bytes < 4096 || bytes > (64ull << 20) || reps < 1) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(c->device));
    uint4 *buf = nullptr;
    unsigned *sink = nullptr;
    KICP_CUDA(cudaMalloc(&buf, bytes));
    KICP_CUDA(cudaMalloc(&sink, sizeof(unsigned)));
    KICP_CUDA(cudaMemsetAsync(buf, 1, bytes, c->stream));
    cudaEvent_t e0, e1;
    KICP_CUDA(cudaEventCreate(&e0));
    KICP_CUDA(cudaEventCreate(&e1));
    double best = 0.0;
    for (int k = 0; k < 4; ++k) {  // the first launch warms L2
        KICP_CUDA(cudaEventRecord(e0, c->stream));
        KICP_CUDA(kr_launch_l2_read(buf, (size_t)bytes, reps, sink, c->sm_count * 8, c->stream));
        KICP_CUDA(cudaEventRecord(e1, c->stream));
        KICP_CUDA(cudaStreamSynchronize(c->stream));
        float ms = 0.f;
        KICP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        if (k > 0) best = std::max(best, (double)bytes * reps / (ms * 1e-3) / 1e9);
    }
    cudaEventDestroy(e0), cudaEventDestroy(e1);
    cudaFree(buf), cudaFree(sink);
    *gbps = best;
    return KICP_OK;
}
extern "C" int kicp_debug_last_prof(kicp_ctx *c, uint64_t out[24] /* -DKR_PROFILE builds: cycles per phase, counts */) {
    if (!c || !c->reg->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->reg->d_state + kr_offset_stats() + sizeof(uint64_t) * 4, sizeof(uint64_t) * 24, cudaMemcpyDeviceToHost));
    return KICP_OK;
}

// -DKR_PROFILE builds: the timeline of the last registration launch, 4 uint64 per record (0 records otherwise)
extern "C" int kicp_debug_window_log(kicp_ctx *c, uint64_t *out, int64_t cap_entries, int64_t *n) {
    if (!c || !out || !n || cap_entries < 0) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    size_t got = 0;
    KICP_CUDA(kr_window_log(reinterpret_cast<unsigned long long *>(out), (size_t)cap_entries, &got));
    *n = (int64_t)got;
    return KICP_OK;
}

extern "C" int kicp_ctx_profile_begin(kicp_ctx *c) {
    if (!c) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(c->device));
    if (!c->reg->d_prof_iters) KICP_CUDA(cudaMalloc(&c->reg->d_prof_iters, (size_t)kProfCap * sizeof(int32_t)));
    c->reg->prof.clear();
    c->reg->prof.reserve(4096);
    c->reg->profiling = true;
    return KICP_OK;
}

extern "C" int kicp_ctx_profile_end(kicp_ctx *c, kicp_profile *out) {
    if (!c || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(c->device));
    c->reg->profiling = false;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    kicp_profile p{};
    std::vector<ProfReg> prof;
    prof.swap(c->reg->prof);
    std::vector<int32_t> iters(prof.size());
    if (!iters.empty())
        KICP_CUDA(cudaMemcpy(iters.data(), c->reg->d_prof_iters, iters.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < prof.size(); ++r) {
        const ProfReg &pr = prof[r];
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, pr.prep.begin, pr.prep.end) == cudaSuccess) p.prep_ms += ms;
        p.assoc_iterations += iters[r];
        for (size_t k = 0; k < pr.it.size(); ++k) {
            ms = 0.f;
            cudaEventElapsedTime(&ms, pr.it[k].begin, pr.it[k].end);
            if (pr.persistent || (int)k < iters[r]) {
                p.assoc_ms += ms, p.assoc_launches++;
            } else {
                p.idle_ms += ms, p.idle_launches++;
            }
            cudaEventDestroy(pr.it[k].begin), cudaEventDestroy(pr.it[k].end);
        }
        cudaEventDestroy(pr.prep.begin), cudaEventDestroy(pr.prep.end);
        p.registrations++;
    }
    cudaGetLastError();
    *out = p;
    return KICP_OK;
}

extern "C" int kicp_register_scan_async(kicp_map *map, kicp_scan *scan, const double last[7], const double odom[7], double tau,
                                        const kicp_reg_params *params, kicp_reg_result *result) {
    if (!scan) return KICP_ERR_INVALID;
    KICP_TRY(check_registration(map, scan->ctx, scan->n, scan->data(), last, odom, params, false));
    return enqueue_registration(map, scan_view(scan), 0, last, odom, tau, params, result, false);
}
extern "C" int kicp_register_scan_sharded_async(kicp_map *map, kicp_scan *scan, const double last[7], const double odom[7],
                                                double tau, const kicp_reg_params *params, kicp_reg_result *result) {
    if (!scan) return KICP_ERR_INVALID;
    KICP_TRY(check_registration(map, scan->ctx, scan->n, scan->data(), last, odom, params, true));
    return enqueue_registration(map, scan_view(scan), 0, last, odom, tau, params, result, true);
}

int kicp_enqueue_registration_device(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double last[7],
                                     const double odom[7], double tau, const kicp_reg_params *p, int64_t n_hint) {
    KICP_TRY(check_registration(m, m ? m->ctx : nullptr, n_max, d_xyz, last, odom, p, false));
    const ScanView v{reinterpret_cast<const unsigned char *>(d_xyz), (int)n_max, d_n, 24, 0, 8, 16, 0};  // packed float64 x, y, z
    return enqueue_registration(m, v, n_hint, last, odom, tau, p, m->ctx->h_result, false);
}

// Host-pointer entry points: validate, lay the frame out in the context's upload scan, register (the enqueue uploads the frame,
// chunked and overlapped with the first pass where it can), read the result back.
static int register_host(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t ox, int32_t oy,
                         int32_t oz, const double last[7], const double odom[7], double tau, const kicp_reg_params *params,
                         double out_pose[7], kicp_reg_result *result, bool sharded) {
    if (!out_pose) return KICP_ERR_INVALID;
    KICP_TRY(check_registration(map, map ? map->ctx : nullptr, n, data, last, odom, params, sharded));
    kicp_ctx *c = map->ctx;
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(reg_reserve(c));
    kicp_scan *s = c->reg->upload_scan;
    KICP_TRY(kicp_scan_set_layout(s, dtype, point_step, ox, oy, oz));
    KICP_TRY(kicp_scan_reserve_bytes(s, n * (int64_t)s->stride));
    s->n = n, s->d_n = nullptr;
    int st = enqueue_registration(map, scan_view(s), 0, last, odom, tau, params, c->h_result, sharded, data);
    cudaError_t e1 = cudaStreamSynchronize(c->stream), e2 = cudaStreamSynchronize(c->copy_stream);  // drain on every path
    if (st != KICP_OK) return st;
    if (e1 != cudaSuccess) return kicp_cuda_fail(e1, "cudaStreamSynchronize(stream)", __FILE__, __LINE__);
    if (e2 != cudaSuccess) return kicp_cuda_fail(e2, "cudaStreamSynchronize(copy_stream)", __FILE__, __LINE__);
    for (int k = 0; k < 7; ++k) out_pose[k] = c->h_result->pose[k];
    if (result) *result = *c->h_result;
    if (c->h_result->status == KICP_ERR_CUDA || c->h_result->status == KICP_ERR_NCCL)
        kicp_set_error("a device-side wait of the registration kernel timed out (upload flag or a peer of the fused exchange)");
    return c->h_result->status;
}

extern "C" int kicp_register(kicp_map *map, const double *frame_xyz, int64_t n, const double last[7], const double odom[7],
                             double tau, const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result) {
    return register_host(map, frame_xyz, n, KICP_DTYPE_F64, 0, 0, 0, 0, last, odom, tau, params, out_pose, result, false);
}
extern "C" int kicp_register_points(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                    int32_t offset_y, int32_t offset_z, const double last[7], const double odom[7], double tau,
                                    const kicp_reg_params *params, double out_pose[7], kicp_reg_result *result) {
    return register_host(map, data, n, dtype, point_step, offset_x, offset_y, offset_z, last, odom, tau, params, out_pose, result, false);
}
extern "C" int kicp_register_sharded(kicp_map *map, const double *frame_xyz, int64_t n_local, const double last[7],
                                     const double odom[7], double tau, const kicp_reg_params *params, double out_pose[7],
                                     kicp_reg_result *result) {
    return register_host(map, frame_xyz, n_local, KICP_DTYPE_F64, 0, 0, 0, 0, last, odom, tau, params, out_pose, result, true);
}
extern "C" int kicp_register_points_sharded(kicp_map *map, const void *data, int64_t n_local, int32_t dtype, int32_t point_step,
                                            int32_t offset_x, int32_t offset_y, int32_t offset_z, const double last[7],
                                            const double odom[7], double tau, const kicp_reg_params *params, double out_pose[7],
                                            kicp_reg_result *result) {
    return register_host(map, data, n_local, dtype, point_step, offset_x, offset_y, offset_z, last, odom, tau, params, out_pose, result,
                         true);
}
