// kinematic_icp::KinematicRegistration::ComputeRobotMotion on the device
// (reference: cpp/kinematic_icp/registration/Registration.cpp:48-190 + kiss_icp::VoxelHashMap::GetClosestNeighbor).
//
// One registration = ONE cooperative launch of k_register<true>.  Every IRLS iteration ("pass") fuses, for every scan point,
//   q = T p                                          Registration.cpp:74
//   27-voxel probe + nearest neighbour               GetClosestNeighbor (KISS-ICP v1.2.0)
//   gate d < tau                                     Registration.cpp:75
//   r = T p - n,  J = [R e_x | R (-p_y, p_x, 0)]     Registration.cpp:86-93
//   sum of J^T J, J^T r, N, |r|^2                    Registration.cpp:95-118, 48-60
// and ends in a grid barrier after which EVERY CTA sums the per-CTA partials in the same fixed order and solves the 2x2
// system, applies the unicycle motion model and decides convergence redundantly (Registration.cpp:119-125, 159-167,
// 181-184): identical inputs give identical poses, so there is no serial section and no broadcast.  The correspondence
// list of the reference is never materialised: association and linearisation use the same T.
//
// THE SEARCH (pooled, warp-cooperative).  A warp owns a window of up to 32 scan points ("owners").  The work of the window is
// turned into flat streams that all 32 lanes consume together, so no lane waits for the slowest owner:
//   tasks      (owner, neighbour shift k): one hash probe each (home slot + the next, loaded together).  Three stages — the
//              own voxels, the 6 faces, the 12 edges + 8 corners — each pruned with the best distance the previous one left;
//              a stage's tasks form one owner-major stream in the reference's visiting order, processed 32 at a time;
//   lines      a found voxel's points are one contiguous run of 32-byte records, 4 per 128-byte line.  The lines of a stage
//              are described in a per-warp buffer and evaluated in full rounds: a quad (4 lanes) takes one line, each lane
//              loads ONE point (a 128-bit and a 64-bit load: a warp instruction touches 8 lines), KR_G rounds in flight;
//   reduction  the quad's minimum (two shuffles) goes to shared memory; every lane, as an owner, then scans the minima of
//              its own lines in visiting order with the reference's rule (strict <, compared as norms: first minimum wins) and
//              finally re-evaluates the winning line (pinned arithmetic) to name the point.  No atomics.
// Exact pruning: with q in voxel v the cube of v + s is at least lb^2 = sum of the squared face gaps along the shifted axes
// away, so a voxel with lb^2 > bound (1 + 1e-6) + 1e-10 cannot hold the answer (the margin covers the rounding of the face
// coordinates by 9 orders of magnitude); bound = min(best so far, tau^2) — a neighbour at tau or beyond is rejected by the
// gate anyway.  Everything that could tie or win is still evaluated, so the chosen neighbour is the reference's.
//
// CERTIFICATES (passes after the first, option "nn_cache").  Each search leaves, per point, its neighbour g1, the runner-up g2 and
// a lower bound l on the distance to every OTHER candidate of the 27-voxel neighbourhood (evaluated points and skipped cubes alike).
// The next pass first checks every point (phase A): if it moved by delta, all other candidates are still at least l - delta away
// (a step into a neighbouring voxel brings one layer of voxels in: those lie beyond the far face of the new own voxel), so
// min(|q' - g1|, |q' - g2|) < l - delta proves the nearer of the two is still THE strict nearest neighbour and the search is skipped.
// The remaining points are compacted and searched (phase B) with |q' - g| as an exact pruning bound: the usual ones — few voxels
// inside that bound — in ONE merged stage, the stragglers staged, in small windows of their own, so that no ordinary window walks
// through three stages for the sake of one lane.  Phase A sorts the merged ones into cost classes by task count; phase B deals the
// class-ordered list to its windows, so every window gets the same share of each class and no window outlasts the others by much.
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>

#include "kicp_register.cuh"
#include "kicp_solve.cuh"

using namespace kicp_dev;

#ifndef KR_WARPS
#define KR_WARPS 8                    // warps per CTA (3 x 8 warps per SM; 64 K registers and 228 KB of shared memory per SM)
#endif
#define KR_THREADS (KR_WARPS * 32)
#ifndef KR_MINB
#define KR_MINB 3                     // resident CTAs per SM the kernel is compiled for (80 registers: 24 warps hide more latency)
#endif
#ifndef KR_LCAP
#define KR_LCAP 192                   // lines the per-warp buffer holds (a batch of 32 tasks adds at most 160 at 20 points per voxel)
#endif
#ifndef KR_G
#define KR_G 3                        // line-rounds (of 8 lines = 32 points) in flight together
#endif
#ifndef KR_MERGE_MAX
#define KR_MERGE_MAX 19               // neighbour voxels a seeded point may bring into its single merged stage (20 tasks x 32 owners = KR_TCAP)
#endif
#ifndef KR_SLOWWIN
#define KR_SLOWWIN 8                  // points per window of the staged stragglers of a later pass
#endif
// Cost classes of the points a later pass searches again: 0 = staged stragglers; 1, 2, 3 = one merged stage of >= KR_CLS_HEAVY,
// >= KR_CLS_MID, fewer tasks (own voxel + the neighbour voxels inside the bound).
#define KR_CLASSES 4
#ifndef KR_CLS_HEAVY
#define KR_CLS_HEAVY 8
#endif
#ifndef KR_CLS_MID
#define KR_CLS_MID 4
#endif
#define KR_DBLMAX_BITS 0x7FEFFFFFFFFFFFFFull
// Development aid (-DKR_PROFILE): per-phase cycle accounting of the window loop (lane 0 of every warp, clock64 deltas).
#ifdef KR_PROFILE
#define KR_PROF_DECL long long prof_t[24] = {0}; long long prof_last = clock64(); int prof_o = 0;
#define KR_PROF(i) { const long long t__ = clock64(); prof_t[prof_o + (i)] += t__ - prof_last; prof_last = t__; }
#define KR_PROF_COUNT(i) { prof_t[prof_o + (i)] += 1; }
#define KR_PROF_PASS(it) { prof_o = (it) ? 12 : 0; }
#define KR_PROF_FLUSH if (lane == 0) { for (int k__ = 0; k__ < 24; ++k__) atomicAdd(&st->prof[k__], (unsigned long long)prof_t[k__]); }
// ... and a timeline: one record per window / per warp and certificate phase {start ns, end ns, kind|pass|SM|warp, a|b}
#define KR_WLOG_CAP 65536
__device__ unsigned long long g_wlog[KR_WLOG_CAP][4];
__device__ unsigned int g_wlog_n;
__device__ __forceinline__ unsigned smid() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }
#define KR_WLOG(kind, t0, t1, a_, b_) if (lane == 0) { const unsigned i__ = atomicAdd(&g_wlog_n, 1u); if (i__ < KR_WLOG_CAP) { \
    g_wlog[i__][0] = (t0), g_wlog[i__][1] = (t1); \
    g_wlog[i__][2] = ((unsigned long long)(kind) << 56) | ((unsigned long long)it << 48) | ((unsigned long long)smid() << 32) | gwarp; \
    g_wlog[i__][3] = ((unsigned long long)(unsigned)(a_) << 32) | (unsigned)(b_); } }
#define KR_WLOG_DO(x) x
#else
#define KR_WLOG(kind, t0, t1, a_, b_)
#define KR_WLOG_DO(x)
#define KR_PROF_DECL
#define KR_PROF(i)
#define KR_PROF_COUNT(i)
#define KR_PROF_PASS(it)
#define KR_PROF_FLUSH
#endif

struct RegState {
    PoseState pose;                 // multi-launch path only
    unsigned int win_ctr;           // window tickets handed out so far (monotonic inside a registration)
    unsigned int arrive;            // grid-barrier arrivals so far (monotonic inside a registration)
    unsigned int exit_ctr;          // CTAs that have left the kernel; the last one zeroes the three counters
    unsigned int ticket;            // multi-launch path: last-CTA detection
    unsigned int a_arrive;          // warps that finished the certificate phase of a pass (monotonic inside a registration)
    union {  // per cost class and pass: points whose neighbour has to be searched again (arrival counters of the class lists)
        unsigned int cls_n[KR_CLASSES][KICP_MAX_ITERATIONS];
        // (the same counters by class name; the CPU test harness in tests/emu checks todo_n and slow_n)
        struct { unsigned int slow_n[KICP_MAX_ITERATIONS], heavy_n[KICP_MAX_ITERATIONS], mid_n[KICP_MAX_ITERATIONS], todo_n[KICP_MAX_ITERATIONS]; };
    };
    int abort;                      // a device-side wait gave up (status code); every CTA leaves after the current pass
    int *iters_out;                 // optional: where to publish the iteration count (profiling)
    double acc[8];                  // multi-launch path: JTJ00 JTJ01 JTJ11 JTr0 JTr1 N sum|r|^2 (unused)
    unsigned long long stats[4];    // optional work counters: probes, candidate points evaluated, lines, windows
    unsigned long long prof[24];    // -DKR_PROFILE builds only: SM cycles per phase of the window loop, summed over warps
    double dbg[KICP_MAX_ITERATIONS][6];  // per pass, ns (CTA 0): certificate phase, its barrier, search phase, barrier wait, partial sum (+ exchange), solve
    kicp_reg_result result;
};

#ifndef KR_EMU  // (tests/emu compiles this file for the host against a SIMT emulator and supplies these few PTX helpers itself)
__device__ __forceinline__ unsigned long long gtime_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned int ld_acquire_gpu_u32(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
#endif
// one stored map point {x, y, z, pad}, a 32-byte record in one 32-byte sector: x, y with one 128-bit load, z with a 64-bit one
// (sm_90 has no 256-bit load; the pad is never read)
struct __align__(32) Point4 {
    double x, y, z, w;
};
#ifndef KR_EMU
__device__ __forceinline__ Point4 ld_point(const double *p) {
    Point4 r;
    asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
    asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(r.z) : "l"(p + 2));
    r.w = 0.0;
    return r;
}
#endif

// Multi-launch path and the "nothing to do" case (empty map / max_iter <= 0): state in global memory.
__global__ void k_reg_init(RegState *st, RegArgs a) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    pose_init(&st->pose, a);
    result_init(&st->result, &st->pose);
    st->ticket = 0, st->win_ctr = 0, st->arrive = 0, st->exit_ctr = 0, st->abort = 0, st->a_arrive = 0;
    for (int c = 0; c < KR_CLASSES; ++c)
        for (int k = 0; k < KICP_MAX_ITERATIONS; ++k) st->cls_n[c][k] = 0;
    st->iters_out = a.iters_out;
    if (a.iters_out) *a.iters_out = 0;
    for (int k = 0; k < 8; ++k) st->acc[k] = 0.0;
}

// Multi-launch path: the solve between the NCCL allreduce and the next association launch.
__global__ void k_solve(RegState *st) {
    if (threadIdx.x == 0 && blockIdx.x == 0 && !st->pose.done) {
        double s[8];
        for (int k = 0; k < 8; ++k) s[k] = st->acc[k];
        solve_and_update(&st->pose, s, &st->result, st->iters_out);
        for (int k = 0; k < 8; ++k) st->acc[k] = 0.0;
    }
}

// ------------------------------------------------------------------------------------------- per-warp shared state
#define KR_TCAP 640  // tasks of one stage: 32 owners x (6 faces | 20 edges + corners)
struct __align__(8) LineDesc {   // one 128-byte line of a found voxel's run, as the task lane that probed it describes it
    unsigned gline;              // global index of the line's first point
    unsigned short owner;        // the scan point (lane of the window) this line is a candidate set for
    unsigned short nvalid;       // points of the line that exist (1..4)
};
struct __align__(16) WarpSm {
    double2 qxy[32];                 // owner's query point (map frame)
    double qz[32];
    double lmin[KR_LCAP];            // minimum squared distance over each line of the current chunk, in visiting order
    LineDesc ldesc[KR_LCAP];         // the lines of the current chunk
    int vx[32], vy[32], vz[32];      // owner's voxel
    double acc[7][32];               // per-lane running sums of the pass (kept here, not in registers)
    double px[32], py[32];           // owner's scan point (for the Jacobian)
    unsigned short task[KR_TCAP];    // task stream of the current stage: owner << 5 | shift index
};

// The reference compares NORMS with a strict < (first minimum wins).  d2 and best are the reference's own squares (dist2 at the
// reference's query, query_rn); sqrt is monotone, so the squares decide — except when two squares within an ulp or two round to the
// same norm: then the earlier point stays.  So the association of the first pass is the reference's, point for point, given the
// same prior (later passes start from a pose whose last bits depend on the summation order).  Kept out of line: needed about never.
__device__ __noinline__ bool same_norm(double a, double b) { return sqrt(a) == sqrt(b); }
__device__ __forceinline__ bool closer(double d2, double best) {  // "norm(d2) < norm(best)" as the reference evaluates it
    if (!(d2 < best)) return false;
    if (d2 >= best * (1.0 - 4e-16)) return !same_norm(d2, best);
    return true;
}

// |c - q|^2 as the reference's (c - q).norm() squares it: (dx dx + dy dy) + dz dz, every operation rounded on its own (an FMA
// would give other squares, and two points the reference sees at the same distance could then differ here).  The owner
// re-evaluates the winning line with it: both evaluations agree bit for bit.
__device__ __forceinline__ double dist2(double cx, double cy, double cz, double qx, double qy, double qz) {
    const double dx = cx - qx, dy = cy - qy, dz = cz - qz;
    return add_rn(add_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// q = T p as the reference evaluates it: Sophus' quaternion rotation, then the translation (Registration.cpp:74), without FMA
// contraction — the query of the search is the reference's to the last bit (the rotation matrix R would differ in the last bits)
__device__ __forceinline__ void query_rn(const double q[4], const double t[3], double px, double py, double pz, double &ox, double &oy,
                                         double &oz) {
    quat_rotate_rn(q[0], q[1], q[2], q[3], px, py, pz, ox, oy, oz);
    ox = add_rn(ox, t[0]), oy = add_rn(oy, t[1]), oz = add_rn(oz, t[2]);
}

__device__ __forceinline__ void load_scan_point(const ScanView &sv, int i, double &x, double &y, double &z) {
    const unsigned char *p = sv.base + (size_t)i * (size_t)sv.stride;
    if (sv.f32) {
        x = (double)__ldg(reinterpret_cast<const float *>(p + sv.ox));
        y = (double)__ldg(reinterpret_cast<const float *>(p + sv.oy));
        z = (double)__ldg(reinterpret_cast<const float *>(p + sv.oz));
    } else {
        x = __ldg(reinterpret_cast<const double *>(p + sv.ox));
        y = __ldg(reinterpret_cast<const double *>(p + sv.oy));
        z = __ldg(reinterpret_cast<const double *>(p + sv.oz));
    }
}

// The shifts of one search stage that survive the exact bound (bit k <-> voxel_shifts[k]).  Stage 0: the own voxel;
// stage 1: the 6 faces; stage 2: the 12 edges and 8 corners, pruned with the best the faces left behind.
__device__ __forceinline__ unsigned stage_mask(int stage, bool valid, double bound, double qx, double qy, double qz, int vx, int vy,
                                               int vz, double vs, double &minpruned) {
    if (!valid) return 0u;
    if (stage == 0) return 1u;
    double t;
    t = (double)(vx + 1) * vs - qx; const double gxp = t * t;
    t = qx - (double)vx * vs;       const double gxm = t * t;
    t = (double)(vy + 1) * vs - qy; const double gyp = t * t;
    t = qy - (double)vy * vs;       const double gym = t * t;
    t = (double)(vz + 1) * vs - qz; const double gzp = t * t;
    t = qz - (double)vz * vs;       const double gzm = t * t;
    if (stage == 1) {  // the six faces are decided here for good: remember how close a skipped one can be
        unsigned mask = 0u;
        if (gxp <= bound) mask |= 1u << 1; else minpruned = fmin(minpruned, gxp);
        if (gxm <= bound) mask |= 1u << 2; else minpruned = fmin(minpruned, gxm);
        if (gyp <= bound) mask |= 1u << 3; else minpruned = fmin(minpruned, gyp);
        if (gym <= bound) mask |= 1u << 4; else minpruned = fmin(minpruned, gym);
        if (gzp <= bound) mask |= 1u << 5; else minpruned = fmin(minpruned, gzp);
        if (gzm <= bound) mask |= 1u << 6; else minpruned = fmin(minpruned, gzm);
        return mask;
    }
    unsigned mask = 0u;
#pragma unroll
    for (int kk = 7; kk < 27; ++kk) {  // edges and corners: the summed gap decides
        const double lb2 = (shift_x(kk) > 0 ? gxp : (shift_x(kk) < 0 ? gxm : 0.0)) + (shift_y(kk) > 0 ? gyp : (shift_y(kk) < 0 ? gym : 0.0)) +
                           (shift_z(kk) > 0 ? gzp : (shift_z(kk) < 0 ? gzm : 0.0));
        if (lb2 <= bound) mask |= 1u << kk; else minpruned = fmin(minpruned, lb2);
    }
    return mask;
}

// A point that enters a later pass with `sd`, the distance to its previous neighbour at the new position, has an exact pruning bound
// from the start: the neighbour voxels that survive it.  Evaluated identically by the certificate sweep (which sorts the point into
// a cost class by their number) and by the search itself.
__device__ __forceinline__ unsigned seeded_near_mask(double sd, double tau, double qx, double qy, double qz, int vx, int vy, int vz, double vs,
                                                     double &minpruned) {
    const double seed2 = sd * sd * (1.0 + 1e-6);
    const double bound = fmin(tau * tau, seed2) * (1.0 + 1e-6) + 1e-10;
    return stage_mask(1, true, bound, qx, qy, qz, vx, vy, vz, vs, minpruned) | stage_mask(2, true, bound, qx, qy, qz, vx, vy, vz, vs, minpruned);
}

// Entry `pos` of cost class c's list.  The four classes share two arrays of n entries, one class growing from each end, so the
// lists come out class-ordered without knowing the class sizes in advance.
__device__ __forceinline__ unsigned *class_entry(const KernelArgs &a, int n, int c, unsigned pos) {
    unsigned *const base = (c == 0 || c == 3) ? a.todo : a.todo2;
    return base + ((c & 1) ? pos : (unsigned)n - 1u - pos);
}

// gate, residual, Jacobian and the seven sums of one correspondence (Registration.cpp:75, 86-93, 110-118).  rr is the caller's
// dist2 of the pair: the reference's own square, so the gate sqrt(rr) < tau is its (neighbor - query).norm() < tau bit for bit (a
// square recomputed here would be contracted, and a point at tau could fall on the other side); Σ|r|^2 sums the same squares.
__device__ __forceinline__ void accumulate(WarpSm &sm, int lane, const PoseState &ps, double nx, double ny, double nz, double qx, double qy,
                                           double qz, double px, double py, double rr) {
    const double rx = qx - nx, ry = qy - ny, rz = qz - nz;  // r = T p - n
    if (sqrt(rr) < ps.tau) {  // distance < max_correspondance_distance   (Registration.cpp:75)
        // J = [R e_x | R (-p_y, p_x, 0)]      (Registration.cpp:89-91)
        const double c0x = ps.R[0], c0y = ps.R[3], c0z = ps.R[6];
        const double c1x = ps.R[1] * px - ps.R[0] * py, c1y = ps.R[4] * px - ps.R[3] * py, c1z = ps.R[7] * px - ps.R[6] * py;
        sm.acc[0][lane] += c0x * c0x + c0y * c0y + c0z * c0z;
        sm.acc[1][lane] += c0x * c1x + c0y * c1y + c0z * c1z;
        sm.acc[2][lane] += c1x * c1x + c1y * c1y + c1z * c1z;
        sm.acc[3][lane] += c0x * rx + c0y * ry + c0z * rz;
        sm.acc[4][lane] += c1x * rx + c1y * ry + c1z * rz;
        sm.acc[5][lane] += 1.0;
        sm.acc[6][lane] += rr;
    }
}

__device__ __forceinline__ int voxel_of(double x, double vs, double inv_vs, int pow2) {
    // PointToVoxel: floor(x / voxel_size); for a power-of-two voxel size the product with the (exact) reciprocal is the same
    // double as the quotient, so the cheaper form is used; both convert like voxel_coord, or the keys the map stores and the keys
    // probed here would disagree for non-finite and huge coordinates
    return pow2 ? voxel_floor(x * inv_vs) : voxel_coord(x, vs);
}

// ---------------------------------------------------------------------------------------------------------------
// k_register.  PERSISTENT = true: cooperative launch, every CTA resident, all IRLS iterations inside the launch
// (single GPU, and the sharded path with the exchange over NVLink peer memory fused into the barrier).
// PERSISTENT = false: one pass per launch; the last CTA leaves the local sums in st->acc for the NCCL allreduce.
// ---------------------------------------------------------------------------------------------------------------
template <bool PERSISTENT>
__global__ void __launch_bounds__(KR_THREADS, KR_MINB) k_register(const KernelArgs a) {
#ifndef KR_EMU
    extern __shared__ __align__(16) unsigned char s_dyn[];  // KR_WARPS x WarpSm (more than the 48 KB static limit)
#else
    __shared__ __align__(16) unsigned char s_dyn[KR_WARPS * sizeof(WarpSm)];
#endif
    __shared__ PoseState s_ps;
    __shared__ double s_part[KR_WARPS][8];
    __shared__ double s_sum[8];
    __shared__ int s_flag[2];
    __shared__ volatile int s_ncls[2];  // a later pass's search: points of the heavy and the middle class
    // thread 0's %globaltimer stamps of the pass (start, end of the certificate phase, end of its barrier): in shared memory, so
    // that no register of the window loop is spent on them
    __shared__ unsigned long long s_t[3];

    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int quad = lane >> 2, sub = lane & 3;
    const unsigned FULL = 0xFFFFFFFFu;
    WarpSm &sm = reinterpret_cast<WarpSm *>(s_dyn)[wid];
    RegState *const st = a.st;
    const int n = a.scan.d_n ? min(__ldg(a.scan.d_n), a.scan.n) : a.scan.n;
    const int num_windows = (n + 31) >> 5;
    const unsigned total_warps = gridDim.x * KR_WARPS;
    const unsigned gwarp = blockIdx.x * KR_WARPS + (threadIdx.x >> 5);  // this warp's index in the grid

    if (threadIdx.x == 0) {
        if (PERSISTENT) {
            pose_init(&s_ps, a.init);
            if (blockIdx.x == 0) {
                result_init(&st->result, &s_ps);
                if (a.init.iters_out) *a.init.iters_out = 0;
            }
        } else {
            s_ps = st->pose;
        }
    }
    __syncthreads();
    if (!PERSISTENT && s_ps.done) return;

    unsigned tbase = 0;  // first ticket of the current phase (identical in every warp of the grid)
    KR_PROF_DECL

    for (unsigned it = 0; !s_ps.done; ++it) {
#pragma unroll
        for (int k = 0; k < 7; ++k) sm.acc[k][lane] = 0.0;
        if (threadIdx.x == 0) s_t[0] = s_t[1] = s_t[2] = gtime_ns();
        KR_WLOG_DO(const unsigned long long wl_it0 = gtime_ns();)
        KR_PROF_PASS(it)
        const double inv_vs = 1.0 / a.map.voxel_size;
        // tasks per batch: a batch's lines must fit the line buffer even if every voxel is full
        const int tpb = max(1, min(32, KR_LCAP / ((a.map.cap + 3) >> 2)));
        const bool cache = PERSISTENT && a.nn_g != nullptr;
        // Window tickets come from one monotonic counter; every phase owns a contiguous range of it (each warp draws exactly one
        // ticket beyond the range of a phase, so a phase of W windows consumes W + total_warps tickets).
        unsigned tk = 0;  // lane 0: the ticket drawn ahead of time (the atomic's round trip is off the critical path)
        int nsearch = num_windows;  // windows of the search phase of this pass

        if (cache && it > 0u) {
            // ------------------------------------------------------------------------------------------------------------
            // Phase A: CERTIFICATES.  Between two IRLS passes the pose moves by millimetres to centimetres.  The last search
            // left, per point, its neighbour g and a lower bound l on the distance to every other candidate of the 27-voxel
            // neighbourhood (evaluated points and the cubes of pruned voxels alike).  If the query stays in its voxel (same
            // candidate set) and moved by delta, every other candidate is still at least l - delta away; so when
            // |q' - g| < l - delta, g is still THE strict nearest neighbour and the search is skipped (and when nothing was within
            // reach and l - delta > tau, nothing can be accepted now).  Everything else goes to the list of the search phase,
            // with |q' - g| as an exact pruning bound when g still lies in the new neighbourhood.
            // ------------------------------------------------------------------------------------------------------------
            // the certificate of a point costs the same everywhere: the windows are dealt out statically (no ticket traffic)
            for (int w = (int)gwarp; w < num_windows; w += (int)total_warps) {
                const int i = w * 32 + lane;
                const bool valid = i < n;
                double px = 0, py = 0, pz = 0;
                if (valid) load_scan_point(a.scan, i, px, py, pz);
                const unsigned g1 = valid ? __ldcg(&a.nn_g[i]) : 0xFFFFFFFFu;
                const unsigned g2 = valid ? __ldcg(&a.nn_g2[i]) : 0xFFFFFFFFu;
                const double l = valid ? (double)__ldcg(&a.nn_l[i]) : 0.0;
                const bool haveg = g1 != 0xFFFFFFFFu, have2 = g2 != 0xFFFFFFFFu;
                const Point4 c1 = ld_point(a.map.pts + (size_t)(haveg ? g1 : 0u) * KICP_PSTRIDE);
                const Point4 c2 = ld_point(a.map.pts + (size_t)(have2 ? g2 : 0u) * KICP_PSTRIDE);
                // the query of this pass and the previous one, both as the search evaluates them (query_rn): the search of this
                // pass starts from the very q the certificate was judged at, and o is bit for bit the query the previous search used
                double qx, qy, qz, ox, oy, oz;
                query_rn(s_ps.q, s_ps.t, px, py, pz, qx, qy, qz);
                query_rn(s_ps.qp, s_ps.tp, px, py, pz, ox, oy, oz);
                const double vs = a.map.voxel_size;
                const int vx = voxel_of(qx, vs, inv_vs, a.pow2_voxel), vy = voxel_of(qy, vs, inv_vs, a.pow2_voxel),
                          vz = voxel_of(qz, vs, inv_vs, a.pow2_voxel);
                const int ovx = voxel_of(ox, vs, inv_vs, a.pow2_voxel), ovy = voxel_of(oy, vs, inv_vs, a.pow2_voxel),
                          ovz = voxel_of(oz, vs, inv_vs, a.pow2_voxel);
                const double mx = qx - ox, my = qy - oy, mz = qz - oz;
                const double delta = sqrt(mx * mx + my * my + mz * mz) * (1.0 + 1e-9) + 1e-12;
                const double s1 = dist2(c1.x, c1.y, c1.z, qx, qy, qz);
                const double s2 = have2 ? dist2(c2.x, c2.y, c2.z, qx, qy, qz) : DBL_MAX;
                const double d1 = sqrt(s1), d2 = have2 ? sqrt(s2) : DBL_MAX;
                // the two remembered candidates may have swapped; a near-tie between them is left to the search (only it applies the
                // reference's visiting-order rule)
                const bool second_wins = d2 < d1;
                const double dn = second_wins ? d2 : d1;
                const bool clear = !have2 || fabs(d1 - d2) > 1e-9 * (d1 + d2) + 1e-12;
                const Point4 c = second_wins ? c2 : c1;
                // A step into a NEIGHBOURING voxel shifts the 27-voxel neighbourhood by one layer per changed axis: the layer that
                // drops out only removes candidates, the layer that comes in lies beyond the far face of the new own voxel along
                // that axis — `slab` away at least.  Both remembered candidates must still be inside the new neighbourhood.
                double slab = DBL_MAX;
                bool reach = true;
                if (vx != ovx || vy != ovy || vz != ovz) {
                    reach = abs(vx - ovx) <= 1 && abs(vy - ovy) <= 1 && abs(vz - ovz) <= 1;
                    if (vx > ovx) slab = fmin(slab, (double)(vx + 1) * vs - qx); else if (vx < ovx) slab = fmin(slab, qx - (double)vx * vs);
                    if (vy > ovy) slab = fmin(slab, (double)(vy + 1) * vs - qy); else if (vy < ovy) slab = fmin(slab, qy - (double)vy * vs);
                    if (vz > ovz) slab = fmin(slab, (double)(vz + 1) * vs - qz); else if (vz < ovz) slab = fmin(slab, qz - (double)vz * vs);
                    if (haveg)
                        reach = reach && abs(voxel_of(c1.x, vs, inv_vs, a.pow2_voxel) - vx) <= 1 && abs(voxel_of(c1.y, vs, inv_vs, a.pow2_voxel) - vy) <= 1 &&
                                abs(voxel_of(c1.z, vs, inv_vs, a.pow2_voxel) - vz) <= 1;
                    if (have2)
                        reach = reach && abs(voxel_of(c2.x, vs, inv_vs, a.pow2_voxel) - vx) <= 1 && abs(voxel_of(c2.y, vs, inv_vs, a.pow2_voxel) - vy) <= 1 &&
                                abs(voxel_of(c2.z, vs, inv_vs, a.pow2_voxel) - vz) <= 1;
                }
                // every other candidate of the (new) neighbourhood is at least this far from the new position
                const double room = fmin(l - delta, slab * (1.0 - 1e-9) - 1e-12);
                const bool cert = valid && reach && (haveg ? (clear && dn * (1.0 + 1e-9) + 1e-12 < room) : (room > s_ps.tau * (1.0 + 1e-9)));
                if (cert) {
                    a.nn_l[i] = __double2float_rz(room * (1.0 - 1e-7));
                    if (second_wins) a.nn_g[i] = g2, a.nn_g2[i] = g1;
                    if (haveg) accumulate(sm, lane, s_ps, c.x, c.y, c.z, qx, qy, qz, px, py, second_wins ? s2 : s1);
                }
                // Everything else is searched again.  The old neighbour bounds that search if it is one of the new 27 voxels' points; with
                // few neighbour voxels inside the bound the search is ONE merged stage, else it is staged.  The point goes to the list
                // of its cost class: staged, or by the tasks of its merged stage (its own voxel and the neighbours inside the bound).
                const bool again = valid && !cert;
                int cls = -1;
                if (again) {
                    float seed = 3.0e38f;
                    if (haveg && abs(voxel_of(c.x, vs, inv_vs, a.pow2_voxel) - vx) <= 1 && abs(voxel_of(c.y, vs, inv_vs, a.pow2_voxel) - vy) <= 1 &&
                        abs(voxel_of(c.z, vs, inv_vs, a.pow2_voxel) - vz) <= 1)
                        seed = __double2float_ru(dn * (1.0 + 1e-7));
                    a.nn_l[i] = seed;  // (the search reads it from here and then writes the new certificate)
                    cls = 0;
                    if (seed < 1.0e38f) {
                        double mp = DBL_MAX;
                        const int near = __popc(seeded_near_mask((double)seed, s_ps.tau, qx, qy, qz, vx, vy, vz, vs, mp));
                        if (near <= KR_MERGE_MAX) cls = near + 1 >= KR_CLS_HEAVY ? 1 : near + 1 >= KR_CLS_MID ? 2 : 3;
                    }
                }
                // one arrival counter per class (lane k < KR_CLASSES bumps class k's): the lanes of a class take consecutive entries of its list
                unsigned need = 0u, cnt = 0u;
#pragma unroll
                for (int k = 0; k < KR_CLASSES; ++k) {
                    const unsigned m = __ballot_sync(FULL, cls == k);
                    if (cls == k) need = m;
                    if (lane == k) cnt = m;
                }
                unsigned pos = 0;
                if (cnt) pos = atomicAdd(&st->cls_n[lane][it], (unsigned)__popc(cnt));
                pos = __shfl_sync(FULL, pos, max(cls, 0)) + (unsigned)__popc(need & ((1u << lane) - 1u));
                if (cls >= 0) *class_entry(a, n, cls, pos) = (unsigned)i;
            }
            KR_WLOG(1, wl_it0, gtime_ns(), 0, 0)
            // every CTA of the grid has to be through phase A before the list is complete
            __syncthreads();
            if (threadIdx.x == 0) {
                s_t[1] = gtime_ns();
                __threadfence();
                atomicAdd(&st->a_arrive, 1u);
                const unsigned target = it * gridDim.x;
                const unsigned long long deadline = gtime_ns() + a.timeout_ns;
                while (ld_acquire_gpu_u32(&st->a_arrive) < target) {
                    __nanosleep(20);
                    if (gtime_ns() > deadline) {
                        atomicExch(&st->abort, KICP_ERR_CUDA);
                        break;
                    }
                }
                s_t[2] = gtime_ns();
                s_ncls[0] = (int)__ldcg(&st->cls_n[1][it]), s_ncls[1] = (int)__ldcg(&st->cls_n[2][it]);
            }
            __syncthreads();
        }
        const bool indirect = cache && it > 0u;
        // points of the search phase: in pass 0 the whole frame; afterwards the uncertified ones — those that get by with ONE merged
        // stage (the usual case) in three cost classes, heaviest first, and the few that need the staged search
        const int nfast = indirect ? (int)(__ldcg(&st->cls_n[1][it]) + __ldcg(&st->cls_n[2][it]) + __ldcg(&st->cls_n[3][it])) : n;
        const int nslow = indirect ? (int)__ldcg(&st->cls_n[0][it]) : 0;
        // Window size of the phase.  A window is a chain of dependent steps whose length depends little on how many points it holds,
        // so full windows are the efficient unit; but when the whole phase fits ONE round of the grid, the points are spread evenly
        // over all warps (a small scan, the remainder of a later pass), and a phase of k rounds sizes its windows so that every warp
        // gets k of them (no last round that only part of the grid takes part in).  The staged stragglers of a later pass go into
        // small windows of their own (KR_SLOWWIN points, handed out first, and counted in the rounds): one of them inside an ordinary
        // window would make all its 32 lanes walk through the three stages.
        const int P = (int)total_warps;
        const int nslowwin = (nslow + KR_SLOWWIN - 1) / KR_SLOWWIN;
        const int Pf = max(P - nslowwin, P / 2);  // warps left for the ordinary windows of a single-round phase
        int wsz = 32;
        if (PERSISTENT && nfast > 0) {
            if (nfast <= 32 * Pf) {
                wsz = max(1, (nfast + Pf - 1) / Pf);
            } else {
                const int rounds = (nfast + 32 * (P + nslowwin) - 1) / (32 * P);  // (a staged window takes a warp's turn)
                wsz = min(32, (nfast + rounds * Pf - 1) / (rounds * Pf));
            }
        }
        // pass 0: the frame in KICP_UPLOAD_CHUNKS segments of `segpts` points (the host uploads it in exactly these pieces)
        const int segpts = max(32, ((((n + 31) >> 5) + KICP_UPLOAD_CHUNKS - 1) / KICP_UPLOAD_CHUNKS) * 32);
        const int segwin = (segpts + wsz - 1) / wsz;  // windows per (full) segment
        int nfastwin;
        if (indirect) {
            nfastwin = (nfast + wsz - 1) / wsz;
        } else {
            const int nseg = min(KICP_UPLOAD_CHUNKS, (n + segpts - 1) / segpts), lastn = n - (nseg - 1) * segpts;
            nfastwin = n > 0 ? (nseg - 1) * segwin + (lastn + wsz - 1) / wsz : 0;
        }
        nsearch = nslowwin + nfastwin;

        // ------------------------------------------------------------------------------------------------------------------
        // Phase B: THE SEARCH (all points in pass 0; the uncertified ones, compacted, afterwards)
        // ------------------------------------------------------------------------------------------------------------------
        // the first window of every warp is its own index (no burst of atomics on one word when a phase starts); the remaining
        // windows [total_warps, nsearch) are handed out dynamically, because windows differ in cost
        int w = min((int)gwarp, nsearch);
        const unsigned dyn = (unsigned)max(nsearch - (int)total_warps, 0);  // windows behind tickets
        KR_PROF(11)
        while (w < nsearch) {
            if (lane == 0) tk = atomicAdd(&st->win_ctr, 1u);
            KR_PROF_COUNT(8)
            KR_WLOG_DO(const unsigned long long wl_t0 = gtime_ns(); unsigned wl_tasks = 0; unsigned wl_lines = 0;)
            // ---------------------------------------------------------------- owners: q = T p and its voxel
            // The points of a phase are DEALT to its windows like cards (owner `lane` of window w = entry lane * windows + w): points
            // that are expensive to search (little or no map around them) sit next to each other in the scan and in the list, and a
            // window made of them alone would outlast the phase.  In a later pass the list is ordered by cost class, so every window
            // gets the same share of each class: the windows of the phase cost about the same.  Pass 0 deals inside each of the
            // KICP_UPLOAD_CHUNKS segments the frame is uploaded in, so that a window still needs only its own chunk.
            int slot, limit, seg_of_w = 0, wlanes = wsz, cls = 0;
            if (indirect) {
                if (w < nslowwin) {  // a small window of staged stragglers
                    slot = lane * nslowwin + w, limit = nslow, wlanes = KR_SLOWWIN;
                } else {             // the one-stage classes, heaviest first
                    slot = lane * nfastwin + (w - nslowwin), limit = nfast, cls = 1;
                }
            } else {
                const int sgi = min(w / segwin, KICP_UPLOAD_CHUNKS - 1), lw = w - sgi * segwin;
                const int sbase = sgi * segpts, sn = min(segpts, n - sbase);  // this segment's points
                const int sw = (sn + wsz - 1) / wsz;                          // ... and windows
                slot = sbase + lane * sw + lw, limit = lw < sw ? sbase + sn : 0;
                seg_of_w = sgi;
            }
            const bool valid = lane < wlanes && slot < limit;
            int pi = valid ? slot : 0;  // the owner's scan point
            if (indirect) {
                int pos = slot;  // ... the entry `pos` of its class's list
                if (cls == 1 && pos >= s_ncls[0]) pos -= s_ncls[0], cls = 2;
                if (cls == 2 && pos >= s_ncls[1]) pos -= s_ncls[1], cls = 3;
                pi = valid ? (int)__ldcg(class_entry(a, n, cls, (unsigned)pos)) : 0;
            }
            if (PERSISTENT && a.up.flags != nullptr && it == 0u) {
                // first pass over a frame that is still being uploaded: wait until this window's chunk has landed
                const uint32_t *f = a.up.flags + seg_of_w;
                const unsigned long long deadline = gtime_ns() + a.timeout_ns;
                bool pend = true;
                while (__any_sync(FULL, pend)) {  // warp-uniform: every lane polls the same word (one transaction)
                    if (pend) {
                        if (ld_acquire_sys_u32(f) == a.up.seq) {
                            pend = false;
                        } else if (gtime_ns() > deadline) {  // the copy never arrived
                            if (lane == 0) atomicExch(&st->abort, KICP_ERR_CUDA);
                            pend = false;
                        }
                    }
                }
            }
            double seed_d = 3.0e38;  // distance to the previous neighbour — an exact pruning bound —, if it applies (< 1e38)
            {
                double px = 0, py = 0, pz = 0;
                if (valid) load_scan_point(a.scan, pi, px, py, pz);
                if (indirect && valid) {
                    const double sd = (double)__ldcg(&a.nn_l[pi]);  // (the seed, left there by the certificate sweep)
                    if (sd < 1.0e38) seed_d = sd;
                }
                double qx, qy, qz;
                query_rn(s_ps.q, s_ps.t, px, py, pz, qx, qy, qz);
                sm.qxy[lane] = make_double2(qx, qy), sm.qz[lane] = qz;
                sm.vx[lane] = voxel_of(qx, a.map.voxel_size, inv_vs, a.pow2_voxel);
                sm.vy[lane] = voxel_of(qy, a.map.voxel_size, inv_vs, a.pow2_voxel);
                sm.vz[lane] = voxel_of(qz, a.map.voxel_size, inv_vs, a.pow2_voxel);
                sm.px[lane] = px, sm.py[lane] = py;
            }
            // the owner's running minimum lives in its lane's registers: d^2, the line that holds it, how many points that line has;
            // the runner-up line and `lo` feed the certificate of the next pass.  `lo` is the smallest line minimum that is neither
            // `best` nor `second` (whatever either of them gives up goes into it) and the cubes of the voxels that were skipped: the
            // certificate only needs the minimum of all of these, so one register holds it
            double best = DBL_MAX, second = DBL_MAX, lo = DBL_MAX;
            unsigned bline = 0xFFFFFFFFu, bvalid = 0u;   // the line holding `best` ...
            unsigned sline = 0xFFFFFFFFu, svalid = 0u;   // ... and the one holding `second`
            __syncwarp();
            KR_PROF(0)

            // A point that comes with the distance to its previous neighbour (search phase of a later pass) already has a tight
            // pruning bound: its few surviving neighbour voxels join the own voxel in ONE stage instead of three.
            unsigned donem = 0u;    // shifts of this owner that have been scheduled already
            bool merged = false;
            for (int stage = 0; stage < 3; ++stage) {
                // ------------------------------------------------------------ task stream of the stage (owner-major, KISS order)
                if (stage == 1 && !__any_sync(FULL, valid && !merged)) break;  // every owner of the window took the short way
                int total, tfirst, tcount;  // tasks of the stage; this owner's range [tfirst, tfirst + tcount) of the stream
                {
                    const double2 qq = sm.qxy[lane];
                    // exact pruning bound: the best squared distance found so far, and never more than the gate — a neighbour at
                    // tau or beyond is rejected anyway (Registration.cpp:75), so voxels that can only hold such points are skipped
                    const double tau2 = s_ps.tau * s_ps.tau;
                    const double seed2 = seed_d < 1.0e38 ? seed_d * seed_d * (1.0 + 1e-6) : DBL_MAX;
                    const double bsq = fmin(fmin(tau2, best), seed2);
                    const double bound = bsq * (1.0 + 1e-6) + 1e-10;
                    unsigned mask = stage_mask(stage, valid, bound, qq.x, qq.y, sm.qz[lane], sm.vx[lane], sm.vy[lane], sm.vz[lane],
                                               a.map.voxel_size, lo);
                    if (stage == 0 && valid && seed_d < 1.0e38) {
                        double mp = lo;
                        const unsigned near = seeded_near_mask(seed_d, s_ps.tau, qq.x, qq.y, sm.qz[lane], sm.vx[lane], sm.vy[lane], sm.vz[lane],
                                                               a.map.voxel_size, mp);
                        if (__popc(near) <= KR_MERGE_MAX) mask |= near, lo = mp, merged = true;  // (a loose bound keeps the staged way)
                    }
                    mask &= ~donem;
                    donem |= mask;
                    const int no = __popc(mask);
                    int tin = no;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const int y = __shfl_up_sync(FULL, tin, d);
                        if (lane >= d) tin += y;
                    }
                    total = __shfl_sync(FULL, tin, 31);
                    int pos = tin - no;
                    tfirst = pos, tcount = no;
                    const int maxno = __reduce_max_sync(FULL, no);
                    for (int i = 0; i < maxno; ++i) {  // warp-uniform trip count, the store predicated per lane
                        if (mask) {
                            const int k = __ffs(mask) - 1;
                            mask &= mask - 1;
                            sm.task[pos++] = (unsigned short)((lane << 5) | k);
                        }
                    }
                    __syncwarp();
                }
                KR_PROF(1)
                // The lines of the stage's found runs are collected in a buffer of KR_LCAP lines (stage-global numbering, visiting
                // order) and evaluated whenever it would overflow and at the end of the stage — full rounds of 8 lines x KR_G.
                KR_WLOG_DO(wl_tasks += (unsigned)total;)
                int fill = 0, lbase = 0;           // lines in the buffer; stage-global index of its first line
                int olb = 0, ole = 0;              // this lane's, as an owner: its lines so far are [olb, ole) (stage-global)
                bool ohas = false;
                for (int base = 0;; base += tpb) {
                    const bool more = base < total;
                    // -------------------------------------------------------- this lane's task and its hash probe
                    const bool act = more && lane < tpb && base + lane < total;
                    const unsigned okpack = act ? (unsigned)sm.task[base + lane] : 0u;
                    uint32_t meta = KICP_SLOT_EMPTY;
                    bool kmin = false;  // a key coordinate is INT_MIN
                    if (more) {
                        KR_PROF_COUNT(9)
                        const int o = (int)(okpack >> 5), k = (int)(okpack & 31u);
                        const int kx = sm.vx[o] + shift_x(k), ky = sm.vy[o] + shift_y(k), kz = sm.vz[o] + shift_z(k);
                        uint32_t h = voxel_hash(kx, ky, kz) & a.map.mask;
                        // the home slot and the next one travel together: with a load factor <= 0.25 a longer chain is rare
                        const int4 s0 = __ldg(&a.map.slots[h]);
                        const int4 s1 = __ldg(&a.map.slots[(h + 1) & a.map.mask]);
                        bool pend = false;
                        if (act && (uint32_t)s0.w != KICP_SLOT_EMPTY) {
                            if (s0.x == kx && s0.y == ky && s0.z == kz) {
                                meta = (uint32_t)s0.w;
                            } else if ((uint32_t)s1.w != KICP_SLOT_EMPTY) {
                                if (s1.x == kx && s1.y == ky && s1.z == kz) {
                                    meta = (uint32_t)s1.w;
                                } else {
                                    pend = true, h = (h + 2) & a.map.mask;
                                }
                            }
                        }
                        while (__any_sync(FULL, pend)) {  // warp-uniform loop
                            if (pend) {
                                const int4 sl = __ldg(&a.map.slots[h]);
                                if ((uint32_t)sl.w == KICP_SLOT_EMPTY) {
                                    pend = false;
                                } else if (sl.x == kx && sl.y == ky && sl.z == kz) {
                                    meta = (uint32_t)sl.w, pend = false;
                                } else {
                                    h = (h + 1) & a.map.mask;
                                }
                            }
                        }
                        kmin = min(min(kx, ky), kz) == INT_MIN;
                    }
                    KR_PROF(2)
                    // -------------------------------------------------------- number the 128-byte lines of the batch
                    // The voxel's min_element starts from its first point and replaces it only by a point at a smaller distance: a first
                    // point with a NaN coordinate (NaN distance to every query) is never replaced, and the comparison across voxels never
                    // takes it — the reference finds nothing in that voxel.  A NaN coordinate has the key INT_MIN: only such are looked at.
                    if (kmin && meta != KICP_SLOT_EMPTY) {
                        const double *p0 = a.map.pts + (size_t)(meta >> 8) * (size_t)a.map.cap * KICP_PSTRIDE;
                        if (isnan(__ldg(p0)) || isnan(__ldg(p0 + 1)) || isnan(__ldg(p0 + 2))) meta = KICP_SLOT_EMPTY;
                    }
                    const int cnt = meta == KICP_SLOT_EMPTY ? 0 : (int)(meta & 0xFFu);
                    const int nl = (cnt + 3) >> 2;
                    int incl = nl;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const int y = __shfl_up_sync(FULL, incl, d);
                        if (lane >= d) incl += y;
                    }
                    const int ltot = __shfl_sync(FULL, incl, 31);
                    if (a.collect_stats) {  // option "stats": the batch's warp sums, one atomic per counter (no register held for them)
                        int csum = cnt;
#pragma unroll
                        for (int d = 16; d > 0; d >>= 1) csum += __shfl_xor_sync(FULL, csum, d);
                        const unsigned nprobe = (unsigned)__popc(__ballot_sync(FULL, act));
                        if (lane == 0)
                            atomicAdd(&st->stats[0], (unsigned long long)nprobe), atomicAdd(&st->stats[1], (unsigned long long)csum),
                                atomicAdd(&st->stats[2], (unsigned long long)ltot);
                    }

                    if ((!more || fill + ltot > KR_LCAP) && fill > 0) {
                        // ---------------------------------------------------- evaluate the buffered lines
                        KR_PROF(3)
                        for (int r0 = 0; r0 < fill; r0 += 8 * KR_G) {
                            // a quad takes a line, a lane ONE point of it; KR_G independent point loads per lane in flight
                            unsigned own[KR_G], gix[KR_G];
                            unsigned hasm = 0;
#pragma unroll
                            for (int g = 0; g < KR_G; ++g) {
                                const int line = r0 + g * 8 + quad;
                                LineDesc ld;
                                ld.gline = 0u, ld.owner = 0, ld.nvalid = 0;
                                if (line < fill) ld = sm.ldesc[line];
                                const bool has = sub < (int)ld.nvalid;
                                own[g] = ld.owner;
                                gix[g] = ld.gline + (has ? (unsigned)sub : 0u);
                                hasm |= has ? (1u << g) : 0u;
                            }
                            Point4 c[KR_G];
#pragma unroll
                            for (int g = 0; g < KR_G; ++g) c[g] = ld_point(a.map.pts + (size_t)gix[g] * KICP_PSTRIDE);
                            KR_PROF_COUNT(10)
                            KR_PROF(4)
#pragma unroll
                            for (int g = 0; g < KR_G; ++g) {
                                const double2 qq = sm.qxy[own[g]];
                                double d2 = (hasm >> g) & 1u ? dist2(c[g].x, c[g].y, c[g].z, qq.x, qq.y, sm.qz[own[g]]) : DBL_MAX;
                                // the line's minimum (a NaN distance never wins, as in the reference's comparisons)
                                d2 = fmin(d2, __shfl_xor_sync(FULL, d2, 1));
                                d2 = fmin(d2, __shfl_xor_sync(FULL, d2, 2));
                                if (sub == 0 && r0 + g * 8 + quad < fill) sm.lmin[r0 + g * 8 + quad] = d2;
                            }
                        }
                        __syncwarp();
                        // every lane, as an owner: first strict minimum over its lines in the buffer, in visiting order
                        {
                            const int lb = ohas ? max(olb - lbase, 0) : 0, le = ohas ? min(ole - lbase, fill) : 0;
                            const int maxlen = __reduce_max_sync(FULL, max(le - lb, 0));
                            for (int u = 0; u < maxlen; ++u) {  // warp-uniform trip count
                                if (lb + u < le) {
                                    const double dl = sm.lmin[lb + u];
                                    if (closer(dl, best)) {
                                        const LineDesc ld = sm.ldesc[lb + u];
                                        lo = fmin(lo, second);
                                        second = best, sline = bline, svalid = bvalid;
                                        best = dl, bline = ld.gline, bvalid = ld.nvalid;
                                    } else if (dl < second) {
                                        const LineDesc ld = sm.ldesc[lb + u];
                                        lo = fmin(lo, second);
                                        second = dl, sline = ld.gline, svalid = ld.nvalid;
                                    } else {
                                        lo = fmin(lo, dl);
                                    }
                                }
                            }
                        }
                        __syncwarp();
                        KR_WLOG_DO(wl_lines += (unsigned)fill;)
                        lbase += fill, fill = 0;
                        KR_PROF(5)
                    }
                    if (!more) break;
                    // -------------------------------------------------------- describe the batch's lines in the buffer
                    {
                        const int gl = lbase + fill + (incl - nl);  // stage-global index of this task's first line
                        // the lines of an owner are contiguous (tasks are owner-major): this lane's, as an owner, are those of the
                        // task lanes [t0, t1) of the batch
                        const int t0 = max(tfirst - base, 0), t1 = min(tfirst + tcount - base, tpb);
                        const int b0 = __shfl_sync(FULL, gl, t0 & 31), e1 = __shfl_sync(FULL, gl + nl, (t1 - 1) & 31);
                        if (t1 > t0) {
                            if (!ohas) olb = b0, ohas = true;
                            ole = e1;
                        }
                        const int maxnl = __reduce_max_sync(FULL, nl);
                        for (int li = 0; li < maxnl; ++li) {  // warp-uniform trip count
                            if (li < nl) {
                                LineDesc ld;
                                ld.gline = (meta >> 8) * (unsigned)a.map.cap + (unsigned)(li * 4);
                                ld.owner = (unsigned short)(okpack >> 5);
                                ld.nvalid = (unsigned short)min(cnt - li * 4, 4);
                                sm.ldesc[gl - lbase + li] = ld;
                            }
                        }
                        fill += ltot;
                    }
                    __syncwarp();
                    KR_PROF(3)
                }
                __syncwarp();
            }
            KR_PROF(1)
            // ---------------------------------------------------------------- gate, residual, Jacobian, sums
            {
                // the winning line is re-evaluated by its owner (same pinned arithmetic): the first of its points at the minimum is
                // the neighbour the reference returns
                const bool have = valid && bline != 0xFFFFFFFFu;
                const unsigned g0 = have ? bline : 0u;
                Point4 cc[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) cc[j] = ld_point(a.map.pts + (size_t)(g0 + (j < (int)bvalid ? j : 0)) * KICP_PSTRIDE);
                const double2 q0 = sm.qxy[lane];
                const double q0z = sm.qz[lane];
                double dj[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) dj[j] = dist2(cc[j].x, cc[j].y, cc[j].z, q0.x, q0.y, q0z);
                int jw = 0;  // (a NaN distance is the line's minimum never: a point before the minimum at NaN gives way to it)
#pragma unroll
                for (int j = 1; j < 4; ++j)
                    if (j < (int)bvalid && (closer(dj[j], dj[jw]) || dj[jw] != dj[jw])) jw = j;
                Point4 c = cc[0];
                double dw = dj[0];
#pragma unroll
                for (int j = 1; j < 4; ++j)
                    if (jw == j) c = cc[j], dw = dj[j];
                if (have) accumulate(sm, lane, s_ps, c.x, c.y, c.z, q0.x, q0.y, q0z, sm.px[lane], sm.py[lane], dw);
                if (cache && valid) {
                    // What the next pass may rely on: the neighbour g1, the runner-up g2 among the points of the two best lines, and
                    // l = how far every OTHER candidate is at least (third point of those lines, every other line, skipped cubes).
                    const bool have2 = have && sline != 0xFFFFFFFFu;
                    Point4 ce[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) ce[j] = ld_point(a.map.pts + (size_t)((have2 ? sline : 0u) + (j < (int)svalid ? j : 0)) * KICP_PSTRIDE);
                    double ru = DBL_MAX, ru2 = DBL_MAX;  // smallest and second smallest squared distance among the non-winners
                    unsigned g2 = 0xFFFFFFFFu;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (have && j < (int)bvalid && j != jw) {
                            if (dj[j] < ru) ru2 = ru, ru = dj[j], g2 = g0 + (unsigned)j;
                            else ru2 = fmin(ru2, dj[j]);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const double de = dist2(ce[j].x, ce[j].y, ce[j].z, q0.x, q0.y, q0z);
                        if (have2 && j < (int)svalid) {
                            if (de < ru) ru2 = ru, ru = de, g2 = sline + (unsigned)j;
                            else ru2 = fmin(ru2, de);
                        }
                    }
                    const double lo2 = fmin(ru2, lo);
                    a.nn_g[pi] = have ? g0 + (unsigned)jw : 0xFFFFFFFFu;
                    a.nn_g2[pi] = g2;
                    a.nn_l[pi] = lo2 >= 1.0e60 ? 1.0e30f : __double2float_rz(sqrt(lo2) * (1.0 - 1e-7));
                }
            }
            __syncwarp();
            KR_PROF(6)
            KR_WLOG_DO(const unsigned wl_pts = (unsigned)__popc(__ballot_sync(FULL, valid));)
            KR_WLOG(0, wl_t0, gtime_ns(), (wl_tasks << 8) | wl_pts, wl_lines)
            w = (int)(total_warps + min(__shfl_sync(FULL, tk, 0) - tbase, dyn));  // >= nsearch once the tickets are used up
            KR_PROF(7)
        }
        // every processed window drew exactly one ticket (its warp's request for the next one), so the phase consumed `nsearch`
        tbase += (unsigned)nsearch;
        KR_PROF(11)

        const unsigned long long t_win = gtime_ns();
        // ---------------------------------------------------------------- warp -> CTA partial (plain stores, fixed order)
        double v[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) v[k] = sm.acc[k][lane];
#pragma unroll
        for (int k = 0; k < 7; ++k) {
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) v[k] += __shfl_xor_sync(FULL, v[k], d);
        }
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 7; ++k) s_part[wid][k] = v[k];
            s_part[wid][7] = 0.0;
        }
        __syncthreads();
        double *const part = a.partials + (size_t)(PERSISTENT ? (it & 1u) : 0u) * gridDim.x * 8;
        if (threadIdx.x < 8) {
            double s = 0.0;
            for (int k = 0; k < KR_WARPS; ++k) s += s_part[k][threadIdx.x];
            __stcg(&part[(size_t)blockIdx.x * 8 + threadIdx.x], s);
            __threadfence();
        }
        __syncthreads();

        if (!PERSISTENT) {
            // one pass per launch: the last CTA sums the partials into st->acc (the NCCL allreduce and k_solve follow)
            if (threadIdx.x == 0) {
                const unsigned ticket = atomicAdd(&st->ticket, 1u);
                s_flag[0] = (ticket == gridDim.x - 1);
            }
            __syncthreads();
            if (s_flag[0]) {
                __threadfence();
                if (threadIdx.x < 8) {
                    double s = 0.0;
                    for (unsigned bb = 0; bb < gridDim.x; ++bb) s += __ldcg(&part[(size_t)bb * 8 + threadIdx.x]);
                    st->acc[threadIdx.x] = s;
                }
                if (threadIdx.x == 0) st->ticket = 0, st->win_ctr = 0;
            }
            return;
        }

        // ---------------------------------------------------------------- grid barrier: arrive, then everyone reduces
        const bool multi = a.px.nranks > 1;
        unsigned long long t_arr = 0, t_red = 0;
        if (threadIdx.x == 0) {
            atomicAdd(&st->arrive, 1u);
            if (!multi || blockIdx.x == 0) {
                const unsigned target = (it + 1u) * gridDim.x;
                const unsigned long long deadline = t_win + a.timeout_ns;  // per-thread register: no uniform read inside the spin
                while (ld_acquire_gpu_u32(&st->arrive) < target) {
                    __nanosleep(40);  // the spinning thread shares its scheduler with warps that are still working
                    if (gtime_ns() > deadline) {  // a CTA of this grid never arrived: give up instead of hanging
                        atomicExch(&st->abort, KICP_ERR_CUDA);
                        break;
                    }
                }
            }
            t_arr = gtime_ns();
        }
        __syncthreads();
        if (!multi || blockIdx.x == 0) {
            // column k = thread & 7, rows strided by 32: fixed summation tree, identical in every CTA
            const int col = threadIdx.x & 7, row0 = threadIdx.x >> 3;
            double s = 0.0;
            const unsigned nrow = (gridDim.x + KR_THREADS / 8 - 1) / (KR_THREADS / 8);  // uniform trip count, tail predicated
            for (unsigned kr = 0; kr < nrow; ++kr) {
                const unsigned bb = kr * (KR_THREADS / 8) + (unsigned)row0;
                if (bb < gridDim.x) s += __ldcg(&part[(size_t)bb * 8 + col]);
            }
            s += __shfl_xor_sync(FULL, s, 8);
            s += __shfl_xor_sync(FULL, s, 16);
            if (lane < 8) s_part[wid][lane] = s;
            __syncthreads();
            if (threadIdx.x < 8) {
                double tsum = 0.0;
                for (int k = 0; k < KR_WARPS; ++k) tsum += s_part[k][threadIdx.x];
                s_sum[threadIdx.x] = tsum;
            }
            __syncthreads();
        }
        if (multi) {
            // Exchange fused into the barrier (NCCL-LL style): CTA 0 writes its 8 local sums as sixteen 8-byte words
            // {32 data bits, 32-bit tag} into EVERY rank's mailbox over NVLink — an aligned 8-byte store arrives whole, so no
            // fence and no separate flag are needed; every CTA of every rank polls its OWN GPU's mailbox until all ranks'
            // words carry the tag and adds them IN RANK ORDER (same values, same order -> the same pose on every rank).
            const uint32_t tag = a.px.tag_base + it;
            if (wid == 0) {
                if (blockIdx.x == 0) {
                    const double val = s_sum[(lane & 15) >> 1];
                    const unsigned long long bits = (unsigned long long)__double_as_longlong(val);
                    const uint32_t half = (lane & 1) ? (uint32_t)(bits >> 32) : (uint32_t)bits;
                    const unsigned long long word = ((unsigned long long)tag << 32) | half;
                    // lanes 16..31 repeat the stores of lanes 0..15 (same address, same value): no divergent section
#pragma unroll 1
                    for (int r = 0; r < a.px.nranks; ++r) {
                        st_relaxed_sys_u64(&a.px.peer[r]->ll[a.px.parity][it][a.px.rank][lane & 15], word);
                        __syncwarp();
                    }
                }
                __syncwarp();
                double tot = 0.0;
                bool timed_out = false;
                const unsigned long long deadline = gtime_ns() + a.timeout_ns;
                for (int r = 0; r < a.px.nranks; ++r) {
                    unsigned long long wv = 0;
                    const unsigned long long *src = &a.px.peer[a.px.rank]->ll[a.px.parity][it][r][lane & 15];
                    bool pend = true;
                    while (__any_sync(FULL, pend)) {  // warp-uniform loop
                        if (pend) {
                            wv = ld_relaxed_sys_u64(src);
                            if ((uint32_t)(wv >> 32) == tag) {
                                pend = false;
                            } else if (gtime_ns() > deadline) {  // a peer is missing
                                timed_out = true, pend = false;
                            }
                        }
                    }
                    const uint32_t lo = __shfl_sync(FULL, (uint32_t)wv, (lane & 7) * 2);
                    const uint32_t hi = __shfl_sync(FULL, (uint32_t)wv, (lane & 7) * 2 + 1);
                    tot += __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
                }
                timed_out = __any_sync(FULL, timed_out);
                if (lane < 8) s_sum[lane] = tot;
                if (lane == 0) s_flag[1] = timed_out ? 1 : 0;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            t_red = gtime_ns();
            // a wait that gave up (upload flag on this GPU, a peer's words): keep the last pose, report, leave
            int ab = (int)ld_acquire_gpu_u32((const unsigned int *)&st->abort);
            if (!ab && multi && s_flag[1]) ab = KICP_ERR_NCCL;
            if (ab) {
                s_ps.status = ab, s_ps.done = 1;
                if (blockIdx.x == 0) st->result.status = ab;
            } else {
                double s[8];
                for (int k = 0; k < 8; ++k) s[k] = s_sum[k];
                solve_and_update(&s_ps, s, blockIdx.x == 0 ? &st->result : nullptr, blockIdx.x == 0 ? a.init.iters_out : nullptr);
            }
            if (blockIdx.x == 0 && it < KICP_MAX_ITERATIONS) {
                st->dbg[it][0] = (double)(s_t[1] - s_t[0]), st->dbg[it][1] = (double)(s_t[2] - s_t[1]), st->dbg[it][2] = (double)(t_win - s_t[2]);
                st->dbg[it][3] = (double)(t_arr - t_win), st->dbg[it][4] = (double)(t_red - t_arr), st->dbg[it][5] = (double)(gtime_ns() - t_red);
            }
        }
        __syncthreads();
    }

    if (PERSISTENT) {
        KR_PROF_FLUSH
        __syncthreads();
        // the result block goes straight to the caller's page-locked host memory (no copy-engine operation after the kernel)
        if (blockIdx.x == 0 && a.result_host != nullptr) {
            const double *src = reinterpret_cast<const double *>(&st->result);
            double *dst = reinterpret_cast<double *>(a.result_host);
            for (unsigned i = threadIdx.x; i < sizeof(kicp_reg_result) / sizeof(double); i += KR_THREADS) dst[i] = __ldcg(src + i);
            __threadfence_system();
        }
        // the last CTA to leave zeroes the counters for the next registration on this stream
        if (threadIdx.x == 0) {
            __threadfence();
            const unsigned left = atomicAdd(&st->exit_ctr, 1u);
            if (left == gridDim.x - 1) {
                st->win_ctr = 0, st->arrive = 0, st->abort = 0, st->a_arrive = 0;
                for (int c = 0; c < KR_CLASSES; ++c)
                    for (int k = 0; k < KICP_MAX_ITERATIONS; ++k) st->cls_n[c][k] = 0;
                __threadfence();
                st->exit_ctr = 0;
            }
        }
    }
}


// ---------------------------------------------------------------------------------------- entry points for the API file
#ifndef KR_EMU
// Read bandwidth of an L2-resident buffer on this GPU: the physical ceiling of a path whose working set lives in L2 (bench.py
// reports the registration kernel's touched bytes against it).  `bytes` (<= 64 MiB) are read `reps` times by one launch of a
// grid-stride kernel with 128-bit loads; returns GB/s of the best of 3 launches.
__global__ void k_l2_read(const uint4 *__restrict__ p, size_t n, int reps, unsigned *sink) {
    unsigned acc = 0;
    for (int r = 0; r < reps; ++r)
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
            const uint4 v = __ldcg(p + i);
            acc += v.x ^ v.y ^ v.z ^ v.w;
        }
    if (acc == 0x12345678u) *sink = acc;  // keeps the loads alive
}
size_t kr_state_bytes() { return sizeof(RegState); }
size_t kr_offset_result() { return offsetof(RegState, result); }
size_t kr_offset_acc() { return offsetof(RegState, acc); }
size_t kr_offset_dbg() { return offsetof(RegState, dbg); }
size_t kr_offset_stats() { return offsetof(RegState, stats); }
size_t kr_stats_bytes() { return sizeof(((RegState *)0)->stats) + sizeof(((RegState *)0)->prof); }
size_t kr_smem_bytes() { return (size_t)KR_WARPS * sizeof(WarpSm); }

cudaError_t kr_prepare(int *persistent_ctas_per_sm, int *multilaunch_ctas_per_sm) {
    cudaError_t e = cudaFuncSetAttribute(k_register<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kr_smem_bytes());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_register<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kr_smem_bytes());
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(persistent_ctas_per_sm, k_register<true>, KR_THREADS, kr_smem_bytes());
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(multilaunch_ctas_per_sm, k_register<false>, KR_THREADS, kr_smem_bytes());
    return e;
}
cudaError_t kr_launch_init(RegState *st, const RegArgs &a, cudaStream_t stream) {
    k_reg_init<<<1, 32, 0, stream>>>(st, a);
    return cudaGetLastError();
}
cudaError_t kr_launch_solve(RegState *st, cudaStream_t stream) {
    k_solve<<<1, 32, 0, stream>>>(st);
    return cudaGetLastError();
}
cudaError_t kr_window_log(unsigned long long *out, size_t cap_entries, size_t *n) {  // -DKR_PROFILE builds: the last launch's timeline
    *n = 0;
#ifdef KR_PROFILE
    unsigned cnt = 0;
    cudaError_t e = cudaMemcpyFromSymbol(&cnt, g_wlog_n, sizeof(cnt));
    if (e != cudaSuccess) return e;
    *n = std::min<size_t>(std::min<size_t>(cnt, KR_WLOG_CAP), cap_entries);
    return cudaMemcpyFromSymbol(out, g_wlog, *n * 4 * sizeof(unsigned long long));
#else
    (void)out, (void)cap_entries;
    return cudaSuccess;
#endif
}
cudaError_t kr_launch_register(bool persistent, int grid, KernelArgs &ka, cudaStream_t stream) {
#ifdef KR_PROFILE
    {
        void *p = nullptr;
        cudaGetSymbolAddress(&p, g_wlog_n);
        cudaMemsetAsync(p, 0, sizeof(unsigned), stream);
    }
#endif
    if (persistent) {  // cooperative: every CTA resident (the grid barrier inside the kernel relies on it)
        void *args[] = {&ka};
        return cudaLaunchCooperativeKernel((const void *)k_register<true>, dim3(grid), dim3(KR_THREADS), args, kr_smem_bytes(), stream);
    }
    k_register<false><<<grid, KR_THREADS, kr_smem_bytes(), stream>>>(ka);
    return cudaGetLastError();
}
cudaError_t kr_launch_l2_read(const void *buf, size_t bytes, int reps, unsigned *sink, int grid, cudaStream_t stream) {
    k_l2_read<<<grid, 256, 0, stream>>>((const uint4 *)buf, bytes / 16, reps, sink);
    return cudaGetLastError();
}
#endif  // KR_EMU
