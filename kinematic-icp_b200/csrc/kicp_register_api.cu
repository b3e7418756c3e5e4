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
    } else {
        kicp_set_error(std::string("kicp_ctx_set_option: unknown option ") + name);
        return KICP_ERR_INVALID;
    }
    return KICP_OK;
}

static int reg_reserve(kicp_ctx *c) {
    if (c->d_state) return KICP_OK;
    KICP_CUDA(cudaMalloc((void **)&c->d_state, kr_state_bytes()));
    KICP_CUDA(cudaMemset(c->d_state, 0, kr_state_bytes()));
    int per_sm_p = 0, per_sm_m = 0;
    KICP_CUDA(kr_prepare(&per_sm_p, &per_sm_m));
    c->persistent_ctas_per_sm = std::max(per_sm_p, 1);
    c->pruned_ctas_per_sm = std::max(per_sm_m, 1);
    const int max_grid = c->sm_count * std::max(c->persistent_ctas_per_sm, c->pruned_ctas_per_sm);
    KICP_CUDA(cudaMalloc(&c->d_partials, (size_t)2 * max_grid * 8 * sizeof(double)));
    int coop = 0;
    KICP_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device));
    if (!coop) c->persistent = 0;
    return KICP_OK;
}

static int check_params(const kicp_reg_params *p) {
    if (!p) return KICP_ERR_INVALID;
    if (p->max_num_iterations > KICP_MAX_ITERATIONS) {
        kicp_set_error("max_num_iterations exceeds KICP_MAX_ITERATIONS");
        return KICP_ERR_INVALID;
    }
    return KICP_OK;
}

// Host side of the chunked upload: the frame's bytes go out in KICP_UPLOAD_CHUNKS pieces on the copy stream, each followed
// by a 4-byte flag copy; the persistent kernel's first pass waits per chunk on the flag, so the association starts while
// later chunks are still on the bus.
struct HostUpload {
    const unsigned char *src;
    unsigned char *dst;
    int64_t n, wpc;   // points, windows per chunk
    int64_t stride;   // bytes per point
};
static int issue_chunks(kicp_ctx *c, const HostUpload &hu) {
    // The kernel always sees KICP_UPLOAD_CHUNKS segments; the host groups them into copies of at least ~384 KB (a small frame is
    // ONE copy and one flag copy: every DMA operation costs microseconds, which a 24 KB scan cannot win back by overlapping).
    const int64_t bytes = hu.n * hu.stride;
    const int copies = (int)std::max<int64_t>(1, std::min<int64_t>(KICP_UPLOAD_CHUNKS, bytes / (384 << 10)));
    for (int j = 0; j < copies; ++j) {
        const int k0 = j * KICP_UPLOAD_CHUNKS / copies, k1 = (j + 1) * KICP_UPLOAD_CHUNKS / copies;  // segments [k0, k1)
        const int64_t lo = std::min<int64_t>(hu.n, k0 * hu.wpc * 32), hi = std::min<int64_t>(hu.n, k1 * hu.wpc * 32);
        if (hi > lo)
            KICP_CUDA(cudaMemcpyAsync(hu.dst + lo * hu.stride, hu.src + lo * hu.stride, (size_t)((hi - lo) * hu.stride),
                                      cudaMemcpyHostToDevice, c->copy_stream));
        KICP_CUDA(cudaMemcpyAsync(c->d_chunk_flags + k0, c->h_chunk_tags + k0, (size_t)(k1 - k0) * sizeof(uint32_t), cudaMemcpyHostToDevice,
                                  c->copy_stream));
    }
    return KICP_OK;
}

static ScanView scan_view(const kicp_scan *s) {
    ScanView v;
    v.base = (const unsigned char *)s->d_data, v.n = (int)s->n, v.d_n = s->d_n;
    v.stride = s->stride, v.ox = s->ox, v.oy = s->oy, v.oz = s->oz, v.f32 = s->dtype == KICP_DTYPE_F32 ? 1 : 0;
    return v;
}

// Enqueue one full registration on the context stream.  `sharded`: this rank holds a contiguous index range of the frame;
// the 8 sums of every iteration are exchanged (fused peer-memory exchange when kicp_comm_p2p_init was called, else NCCL).
// Everything that can fail on arguments is checked before any device work is issued.
static int enqueue_registration(kicp_map *m, const kicp_scan *scan, const double last[7], const double odom[7], double tau,
                                const kicp_reg_params *p, kicp_reg_result *result, bool sharded, const HostUpload *host_upload = nullptr) {
    if (!m || !scan || !last || !odom) return KICP_ERR_INVALID;
    KICP_TRY(check_params(p));
    kicp_ctx *c = m->ctx;
    if (scan->ctx != c) return KICP_ERR_INVALID;
    if (scan->n > 0x7FFFFFE0ll) return KICP_ERR_CAPACITY;
    if (sharded && !c->nccl_comm && !c->p2p_ready) {
        kicp_set_error("kicp_register_sharded: neither kicp_comm_p2p_init nor kicp_comm_init has been called on this context");
        return KICP_ERR_INVALID;
    }
    KICP_CUDA(cudaSetDevice(c->device));
    KICP_TRY(reg_reserve(c));
    KernelArgs ka{};
    ka.st = c->d_state;
    ka.scan = scan_view(scan);
    ka.map = m->view();
    ka.partials = c->d_partials;
    ka.px.nranks = 1;
    ka.up = UploadArgs{nullptr, 0u, 1};
    ka.init.last = Pose{last[0], last[1], last[2], last[3], last[4], last[5], last[6]};
    ka.init.odom = Pose{odom[0], odom[1], odom[2], odom[3], odom[4], odom[5], odom[6]};
    ka.init.tau = tau, ka.init.conv = p->convergence_criterion, ka.init.fixed_reg = p->fixed_regularization;
    ka.init.adaptive = p->use_adaptive_odometry_regularization ? 1 : 0;
    // an empty map returns the prediction (Registration.cpp:157): no association, no solve
    ka.init.max_iter = m->num_blocks == 0 ? 0 : p->max_num_iterations;
    ka.init.iters_out = nullptr;
    {
        int e = 0;
        ka.pow2_voxel = std::frexp(m->voxel_size, &e) == 0.5 ? 1 : 0;
    }
    ka.collect_stats = c->collect_stats;
    ka.nn_g = nullptr, ka.nn_g2 = nullptr, ka.nn_l = nullptr, ka.nn_seed = nullptr, ka.todo = nullptr;
    // (1 = automatic: a small scan is one tiny window per warp and gains nothing from the extra phase and its barrier)
    // a frame whose exact count is still on the device is planned (grid, certificates) for the count its producer expects
    const int64_t n_plan = (scan->d_n && c->reg_n_hint > 0) ? std::min<int64_t>(c->reg_n_hint, scan->n) : scan->n;
    c->reg_n_hint = 0;
    if ((c->nn_cache == 2 || (c->nn_cache == 1 && n_plan >= 49152)) && scan->n > 0) {
        if (scan->n > c->nn_cap) {
            KICP_CUDA(cudaStreamSynchronize(c->stream));
            cudaFree(c->d_nn_g), cudaFree(c->d_nn_g2), cudaFree(c->d_nn_l), cudaFree(c->d_nn_seed), cudaFree(c->d_todo);
            c->d_nn_g = nullptr, c->d_nn_g2 = nullptr, c->d_nn_l = nullptr, c->d_nn_seed = nullptr, c->d_todo = nullptr, c->nn_cap = 0;
            const int64_t cap = scan->n + scan->n / 4 + 1024;
            KICP_CUDA(cudaMalloc(&c->d_nn_g, (size_t)cap * sizeof(unsigned int)));
            KICP_CUDA(cudaMalloc(&c->d_nn_g2, (size_t)cap * sizeof(unsigned int)));
            KICP_CUDA(cudaMalloc(&c->d_nn_l, (size_t)cap * sizeof(float)));
            KICP_CUDA(cudaMalloc(&c->d_nn_seed, (size_t)cap * sizeof(float)));
            KICP_CUDA(cudaMalloc(&c->d_todo, (size_t)cap * sizeof(unsigned int)));
            c->nn_cap = cap;
        }
        ka.nn_g = c->d_nn_g, ka.nn_g2 = c->d_nn_g2, ka.nn_l = c->d_nn_l, ka.nn_seed = c->d_nn_seed, ka.todo = c->d_todo;
    }
    ka.timeout_ns = (unsigned long long)c->spin_timeout_ms * 1000000ull;
    // A result block in page-locked host memory (kicp_host_alloc, the context's own staging) is written by the persistent kernel
    // itself; anything else is filled by a copy after the kernel.
    ka.result_host = nullptr;
    if (result && c->persistent && (!sharded || c->p2p_ready) && m->num_blocks != 0 && p->max_num_iterations > 0) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, result) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer)
            ka.result_host = static_cast<kicp_reg_result *>(at.devicePointer);
        else
            cudaGetLastError();  // (ordinary memory: not an error, just not ours to write)
    }
    const int n = (int)scan->n;
    const bool p2p = sharded && c->p2p_ready;
    const bool persistent = c->persistent && (!sharded || p2p);

    kicp_ctx::ProfReg *pr = nullptr;
    if (c->profiling && (int64_t)c->prof.size() < c->prof_cap) {
        c->prof.emplace_back();
        pr = &c->prof.back();
        pr->d_iters = c->d_prof_iters + (c->prof.size() - 1);
        ka.init.iters_out = pr->d_iters;
        KICP_CUDA(cudaEventCreate(&pr->prep0));
        KICP_CUDA(cudaEventCreate(&pr->prep1));
        KICP_CUDA(cudaEventRecord(pr->prep0, c->stream));
    }
    if (c->collect_stats)
        KICP_CUDA(cudaMemsetAsync((char *)c->d_state + kr_offset_stats(), 0, kr_stats_bytes(), c->stream));

    const bool dbg = getenv("KICP_DEBUG_SYNC") != nullptr;
    if (ka.init.max_iter <= 0 || !persistent) {
        KICP_CUDA(kr_launch_init(c->d_state, ka.init, c->stream));
        c->launches++;
    }
    if (pr) KICP_CUDA(cudaEventRecord(pr->prep1, c->stream));
    if (ka.init.max_iter > 0) {
        // every CTA is resident and pulls 32-point windows from a device-side counter; a small scan is spread one window per
        // CTA over the whole machine (a window is a chain of dependent memory round trips: latency, not throughput)
        // (the persistent kernel sizes its windows so that a phase that fits one round spreads evenly over the grid: a small scan
        // runs as many tiny windows on the whole machine)
        const int num_windows = persistent ? (int)((n_plan + 7) / 8) : (n + 31) / 32;
        int per_sm = persistent ? c->persistent_ctas_per_sm : c->pruned_ctas_per_sm;
        if (c->ctas_per_sm_cap > 0) per_sm = std::min(per_sm, c->ctas_per_sm_cap);
        const int grid = std::max(1, std::min(num_windows, c->sm_count * per_sm));
        if (persistent) {
            if (host_upload && c->overlap_upload) {
                const uint32_t seq = ++c->upload_seq ? c->upload_seq : ++c->upload_seq;  // never 0
                for (int k = 0; k < KICP_UPLOAD_CHUNKS; ++k) c->h_chunk_tags[k] = seq;
                ka.up = UploadArgs{c->d_chunk_flags, seq, (int)host_upload->wpc};  // (the copies are issued right after the launch)
            }
            if (p2p) {
                for (int r = 0; r < c->nranks; ++r) ka.px.peer[r] = c->p2p_peer[r];
                ka.px.nranks = c->nranks, ka.px.rank = c->rank;
                ka.px.parity = (int)(c->p2p_seq & 1ull);
                ka.px.tag_base = (uint32_t)((c->p2p_seq * KICP_MAX_ITERATIONS + 1ull) & 0xFFFFFFFFull);
                if (ka.px.tag_base > 0xFFFFFF00u) ka.px.tag_base = 1u, c->p2p_seq = 0;  // wrap (tags stay non-zero)
                c->p2p_seq++;
            }
            cudaEvent_t e0 = nullptr, e1 = nullptr;
            if (pr) {
                KICP_CUDA(cudaEventCreate(&e0));
                KICP_CUDA(cudaEventCreate(&e1));
                pr->it.push_back(e0), pr->it.push_back(e1);
                pr->persistent = true;
                KICP_CUDA(cudaEventRecord(e0, c->stream));
            }
            KICP_CUDA(kr_launch_register(true, grid, ka, c->stream));
            c->launches++;
            if (pr) KICP_CUDA(cudaEventRecord(e1, c->stream));
            // The frame's chunks go out AFTER the launch: the kernel is already resident and takes every chunk as its flag rises, and the
            // host-side cost of the copies (for pageable memory the driver stages each of them on this thread) no longer delays the
            // launch, which matters most to a caller with pageable buffers.
            // (A copy that fails here leaves the kernel to its wait timeout; the call drains both streams and reports the error.)
            if (ka.up.flags != nullptr) KICP_TRY(issue_chunks(c, *host_upload));
            if (dbg) {
                cudaError_t e = cudaStreamSynchronize(c->stream);
                fprintf(stderr, "[kicp] persistent launch (grid %d, n %d): %s\n", grid, n, cudaGetErrorString(e));
            }
        } else {
            for (int j = 0; j < ka.init.max_iter; ++j) {
                cudaEvent_t e0 = nullptr, e1 = nullptr;
                if (pr) {
                    KICP_CUDA(cudaEventCreate(&e0));
                    KICP_CUDA(cudaEventCreate(&e1));
                    pr->it.push_back(e0), pr->it.push_back(e1);
                    KICP_CUDA(cudaEventRecord(e0, c->stream));
                }
                KICP_CUDA(kr_launch_register(false, grid, ka, c->stream));
                c->launches++;
                if (pr) KICP_CUDA(cudaEventRecord(e1, c->stream));
                if (sharded) KICP_TRY(kicp_comm_allreduce8(c, (double *)((char *)c->d_state + kr_offset_acc())));
                KICP_CUDA(kr_launch_solve(c->d_state, c->stream));
                c->launches++;
                if (dbg) {
                    cudaError_t e = cudaStreamSynchronize(c->stream);
                    fprintf(stderr, "[kicp] pass %d (grid %d, n %d): %s\n", j, grid, n, cudaGetErrorString(e));
                }
            }
        }
    }
    if (result && !ka.result_host)
        KICP_CUDA(cudaMemcpyAsync(result, (const char *)c->d_state + kr_offset_result(), sizeof(kicp_reg_result), cudaMemcpyDeviceToHost,
                                  c->stream));
    return KICP_OK;
}

const kicp_reg_result *kicp_device_result(kicp_ctx *c) {
    return c && c->d_state ? reinterpret_cast<const kicp_reg_result *>((const char *)c->d_state + kr_offset_result()) : nullptr;
}

// debugging aids (not part of the public header): per-pass device timings and work counters of the last registration
extern "C" int kicp_debug_last_timing(kicp_ctx *c, double *out /* [KICP_MAX_ITERATIONS][6] */) {
    if (!c || !c->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->d_state + kr_offset_dbg(), sizeof(double) * KICP_MAX_ITERATIONS * 6,
                         cudaMemcpyDeviceToHost));
    return KICP_OK;
}
extern "C" int kicp_debug_last_stats(kicp_ctx *c, uint64_t out[4] /* probes, candidate points, 128-byte lines, 0 */) {
    if (!c || !c->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->d_state + kr_offset_stats(), sizeof(uint64_t) * 4, cudaMemcpyDeviceToHost));
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
    if (!c || !c->d_state || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    KICP_CUDA(cudaMemcpy(out, (const char *)c->d_state + kr_offset_stats() + sizeof(uint64_t) * 4, sizeof(uint64_t) * 24, cudaMemcpyDeviceToHost));
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
    if (!c->d_prof_iters) {
        c->prof_cap = 1 << 16;
        KICP_CUDA(cudaMalloc(&c->d_prof_iters, (size_t)c->prof_cap * sizeof(int32_t)));
    }
    c->prof.clear();
    c->prof.reserve(4096);
    c->profiling = true;
    return KICP_OK;
}

extern "C" int kicp_ctx_profile_end(kicp_ctx *c, kicp_profile *out) {
    if (!c || !out) return KICP_ERR_INVALID;
    KICP_CUDA(cudaSetDevice(c->device));
    c->profiling = false;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    kicp_profile p{};
    std::vector<int32_t> iters(c->prof.size());
    if (!iters.empty())
        KICP_CUDA(cudaMemcpy(iters.data(), c->d_prof_iters, iters.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < c->prof.size(); ++r) {
        kicp_ctx::ProfReg &pr = c->prof[r];
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, pr.prep0, pr.prep1) == cudaSuccess) p.prep_ms += ms;
        p.assoc_iterations += iters[r];
        for (size_t k = 0; k + 1 < pr.it.size(); k += 2) {
            ms = 0.f;
            cudaEventElapsedTime(&ms, pr.it[k], pr.it[k + 1]);
            if (pr.persistent || (int)(k / 2) < iters[r]) {
                p.assoc_ms += ms, p.assoc_launches++;
            } else {
                p.idle_ms += ms, p.idle_launches++;
            }
            cudaEventDestroy(pr.it[k]), cudaEventDestroy(pr.it[k + 1]);
        }
        cudaEventDestroy(pr.prep0), cudaEventDestroy(pr.prep1);
        p.registrations++;
    }
    cudaGetLastError();
    c->prof.clear();
    *out = p;
    return KICP_OK;
}

extern "C" int kicp_register_scan_async(kicp_map *map, kicp_scan *scan, const double last[7], const double odom[7], double tau,
                                        const kicp_reg_params *params, kicp_reg_result *result) {
    return enqueue_registration(map, scan, last, odom, tau, params, result, false);
}
extern "C" int kicp_register_scan_sharded_async(kicp_map *map, kicp_scan *scan, const double last[7], const double odom[7],
                                                double tau, const kicp_reg_params *params, kicp_reg_result *result) {
    return enqueue_registration(map, scan, last, odom, tau, params, result, true);
}

int kicp_enqueue_registration_device(kicp_map *m, const double *d_xyz, int64_t n_max, const int *d_n, const double last[7],
                                     const double odom[7], double tau, const kicp_reg_params *p) {
    if (!m || n_max < 0 || (n_max > 0 && !d_xyz)) return KICP_ERR_INVALID;
    kicp_scan view;  // non-owning alias of the caller's device buffer (packed xyz doubles)
    view.ctx = m->ctx, view.d_data = const_cast<double *>(d_xyz), view.cap_bytes = n_max * 24, view.n = n_max, view.d_n = d_n;
    const int st = enqueue_registration(m, &view, last, odom, tau, p, m->ctx->h_result, false);
    view.d_data = nullptr;  // not ours
    return st;
}

// Host-pointer entry points: validate, upload (chunked, overlapped with the first pass), register, read the result back.
static int register_host(kicp_map *map, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t ox, int32_t oy,
                         int32_t oz, const double last[7], const double odom[7], double tau, const kicp_reg_params *params,
                         double out_pose[7], kicp_reg_result *result, bool sharded) {
    if (!map || n < 0 || (n > 0 && !data) || !out_pose || !last || !odom) return KICP_ERR_INVALID;
    KICP_TRY(check_params(params));
    kicp_ctx *c = map->ctx;
    if (sharded && !c->nccl_comm && !c->p2p_ready) {
        kicp_set_error("kicp_register_sharded: neither kicp_comm_p2p_init nor kicp_comm_init has been called on this context");
        return KICP_ERR_INVALID;
    }
    KICP_CUDA(cudaSetDevice(c->device));
    if (!c->upload_scan) KICP_TRY(kicp_scan_create(c, 0, &c->upload_scan));
    kicp_scan *s = c->upload_scan;
    KICP_TRY(kicp_scan_set_layout(s, dtype, point_step, ox, oy, oz));
    KICP_TRY(kicp_scan_reserve_bytes(s, n * (int64_t)s->stride));
    s->n = n, s->d_n = nullptr;
    const bool overlap = n > 0 && c->overlap_upload && c->persistent && (!sharded || c->p2p_ready) && map->num_blocks != 0 &&
                         params->max_num_iterations > 0;
    HostUpload hu{(const unsigned char *)data, (unsigned char *)s->d_data, n, 1, s->stride};
    if (n > 0) {
        const int64_t windows = (n + 31) / 32;
        hu.wpc = (windows + KICP_UPLOAD_CHUNKS - 1) / KICP_UPLOAD_CHUNKS;
        if (!overlap) {
            KICP_CUDA(cudaMemcpyAsync(s->d_data, data, (size_t)(n * s->stride), cudaMemcpyHostToDevice, c->stream));
        }
    }
    int st = enqueue_registration(map, s, last, odom, tau, params, c->h_result, sharded, overlap ? &hu : nullptr);
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
