// The planar alignment of a cloud against the voxel map (kicp_map_align_planar*): Gauss-Newton in (x, y, yaw) from up to 64 starting
// poses at once, every iteration on the device, one host synchronisation per call.  A translation unit of its own, compiled with
// -fmad=false like kicp_map.cu (so the transform and the neighbour search are the map's, bit for bit), so that the map's kernels stay
// as they are.
#include <algorithm>
#include <cmath>
#include <vector>

#include "kicp_align_kernels.cuh"  // k_align_eval, k_align_step, k_align_finish; the arithmetic of kicp_align.h

// Device buffers of kicp_map_align_planar*, grown on demand and kept: the widened or uploaded points, the per-slot partials, the
// alignments' states and the records.  A repeated call of the same size allocates nothing.
struct AlignScratch {
    double *pts = nullptr, *part = nullptr;
    AlignState *state = nullptr;
    kicp_planar_alignment *rec = nullptr;
    size_t pts_cap = 0, part_cap = 0;
    int eval_grid = 0;  // k_align_eval's resident grid (occupancy x SMs)
};

void kicp_align_scratch_free(kicp_map *m) {
    AlignScratch *S = m->align;
    if (!S) return;
    cudaFree(S->pts), cudaFree(S->part), cudaFree(S->state), cudaFree(S->rec);
    delete S;
    m->align = nullptr;
}

// `p` holds at least `need` doubles (growth by 1.25x; the stream is drained before a buffer it may use is freed)
static int al_grow(kicp_ctx *c, double *&p, size_t &cap, size_t need) {
    if (need <= cap) return KICP_OK;
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    cudaFree(p);
    p = nullptr, cap = 0;
    const size_t n = std::max<size_t>(need + need / 4, 64);
    KICP_CUDA(cudaMalloc(&p, n * sizeof(double)));
    cap = n;
    return KICP_OK;
}

// the checks shared by both entry points, before any device work (the map last, so that every argument check is reachable without
// one); creates the scratch
static int al_prepare(kicp_map *m, const char *fn, const double *initial, int32_t n_initial, const kicp_planar_align_params *p,
                      kicp_planar_alignment *out) {
    if (!initial) return kicp_invalid(fn, "initial: null pointer");
    if (!p) return kicp_invalid(fn, "params: null pointer");
    if (!out) return kicp_invalid(fn, "out: null pointer");
    if (n_initial < 1 || n_initial > kAlignMaxInitial) return kicp_invalid(fn, "n_initial: not in 1..64");
    for (int64_t k = 0; k < 7 * (int64_t)n_initial; ++k)
        if (!std::isfinite(initial[k])) return kicp_invalid(fn, "initial: not finite");
    if (!std::isfinite(p->tau)) return kicp_invalid(fn, "params->tau: not finite");
    if (!(p->tau > 0.0)) return kicp_invalid(fn, "params->tau: not > 0");
    if (!std::isfinite(p->convergence)) return kicp_invalid(fn, "params->convergence: not finite");
    if (p->convergence < 0.0) return kicp_invalid(fn, "params->convergence: negative");
    if (p->max_iterations < 1 || p->max_iterations > KICP_MAX_ITERATIONS) return kicp_invalid(fn, "params->max_iterations: not in 1..64");
    if (!m) return kicp_invalid(fn, "null map");
    KICP_CUDA(cudaSetDevice(m->ctx->device));
    if (!m->align) {  // the scratch is attached only once its grid is known, so a failed occupancy query is reported every call
        int per_sm = 0;
        KICP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_align_eval, kAlignThreads, 0));
        if (per_sm < 1) return kicp_invalid(fn, "k_align_eval cannot be resident on this device");
        AlignScratch *S = new AlignScratch();
        S->eval_grid = per_sm * m->ctx->sm_count;
        if (cudaMalloc(&S->state, kAlignMaxInitial * sizeof(AlignState)) != cudaSuccess ||
            cudaMalloc(&S->rec, kAlignMaxInitial * sizeof(kicp_planar_alignment)) != cudaSuccess) {
            cudaFree(S->state), cudaFree(S->rec);
            delete S;
            return kicp_cuda_fail(cudaErrorMemoryAllocation, "cudaMalloc (alignment state)", __FILE__, __LINE__);
        }
        m->align = S;
    }
    return KICP_OK;
}

// The launch sequence over device points d_pts (packed doubles); validated arguments.  max_iterations x (k_align_eval, k_align_step),
// the report pass of k_align_eval at the returned poses, k_align_finish, one copy back and one synchronisation.
static int al_run(kicp_map *m, const double *d_pts, int64_t n, const double *initial, int32_t n_initial, const kicp_planar_align_params *p,
                  kicp_planar_alignment *out) {
    kicp_ctx *c = m->ctx;
    AlignScratch &S = *m->align;
    const int C = align_slots(n);
    KICP_TRY(al_grow(c, S.part, S.part_cap, (size_t)n_initial * C * kAlignStride));
    std::vector<AlignState> init((size_t)n_initial);
    for (int32_t a = 0; a < n_initial; ++a) {
        AlignState &s = init[a];
        for (int k = 0; k < 7; ++k) s.pose[k] = initial[7 * (int64_t)a + k];
        s.status = KICP_ALIGN_MAX_ITERATIONS, s.iterations = 0, s.last_step = 0.0, s.done = 0, s.pad = 0;
    }
    KICP_CUDA(cudaMemcpyAsync(S.state, init.data(), init.size() * sizeof(AlignState), cudaMemcpyHostToDevice, c->stream));
    const MapView v = m->view();
    const unsigned grid = (unsigned)std::min<int64_t>((int64_t)n_initial * C, S.eval_grid);
    const unsigned step_grid = (unsigned)((n_initial + 7) / 8);  // 256-thread CTAs, one warp per alignment
    for (int32_t it = 0; it < p->max_iterations; ++it) {
        k_align_eval<<<grid, kAlignThreads, 0, c->stream>>>(v, d_pts, n, p->tau, S.state, n_initial, 0, S.part);
        KICP_CHECK_LAUNCH(c);
        k_align_step<<<step_grid, 256, 0, c->stream>>>(S.part, n, n_initial, p->convergence, S.state);
        KICP_CHECK_LAUNCH(c);
    }
    k_align_eval<<<grid, kAlignThreads, 0, c->stream>>>(v, d_pts, n, p->tau, S.state, n_initial, 1, S.part);
    KICP_CHECK_LAUNCH(c);
    k_align_finish<<<step_grid, 256, 0, c->stream>>>(S.part, n, n_initial, S.state, S.rec);
    KICP_CHECK_LAUNCH(c);
    KICP_CUDA(cudaMemcpyAsync(out, S.rec, (size_t)n_initial * sizeof(kicp_planar_alignment), cudaMemcpyDeviceToHost, c->stream));
    KICP_CUDA(cudaStreamSynchronize(c->stream));
    return KICP_OK;
}

extern "C" int kicp_map_align_planar(kicp_map *m, const double *xyz, int64_t n, const double *initial, int32_t n_initial,
                                     const kicp_planar_align_params *params, kicp_planar_alignment *out) {
    static const char fn[] = "kicp_map_align_planar";
    if (n < 0) return kicp_invalid(fn, "n < 0");
    if (n >= kAlignMaxPoints) return kicp_invalid(fn, "n: 2^40 points or more");
    if (n > 0 && !xyz) return kicp_invalid(fn, "xyz: null pointer");
    KICP_TRY(al_prepare(m, fn, initial, n_initial, params, out));
    kicp_ctx *c = m->ctx;
    AlignScratch &S = *m->align;
    KICP_TRY(al_grow(c, S.pts, S.pts_cap, (size_t)std::max<int64_t>(n, 1) * 3));
    if (n) KICP_CUDA(cudaMemcpyAsync(S.pts, xyz, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    return al_run(m, S.pts, n, initial, n_initial, params, out);
}

extern "C" int kicp_map_align_planar_device(kicp_map *m, const void *data, int64_t n, int32_t dtype, int32_t point_step, int32_t offset_x,
                                            int32_t offset_y, int32_t offset_z, const double *initial, int32_t n_initial,
                                            const kicp_planar_align_params *params, kicp_planar_alignment *out) {
    static const char fn[] = "kicp_map_align_planar_device";
    const kicp_frame_input in{data, n, dtype, point_step, offset_x, offset_y, offset_z, nullptr, 0};
    KICP_TRY(kicp_check_cloud_args(&in, fn));  // also n < 2^30, well inside kAlignMaxPoints
    KICP_TRY(al_prepare(m, fn, initial, n_initial, params, out));
    bool packed = false;
    KICP_TRY(kicp_check_device_cloud(m->ctx, &in, fn, &packed));
    kicp_ctx *c = m->ctx;
    AlignScratch &S = *m->align;
    const double *q = static_cast<const double *>(data);
    if (!packed && n > 0) {  // widened once into the alignment's own buffer (the map's input buffer is left alone)
        KICP_TRY(al_grow(c, S.pts, S.pts_cap, (size_t)n * 3));
        KICP_TRY(kicp_enqueue_widen(c, &in, S.pts));
        q = S.pts;
    }
    return al_run(m, q, n, initial, n_initial, params, out);
}
