// Shared between the registration kernels (kicp_register.cu) and their host-side API (kicp_register_api.cu): the kernel
// argument block and the few entry points through which the API file launches the kernels and finds the fields of the
// device-side state it copies back.  RegState itself stays private to kicp_register.cu.
#pragma once
#include "kicp_device.cuh"

using kicp_dev::Pose;

struct RegArgs {
    Pose last, odom;
    double tau, conv, fixed_reg;
    int adaptive, max_iter;
    int *iters_out;
};

// The frame as it lies in HBM: float64 or float32 x,y,z fields at a byte stride (std::vector<Eigen::Vector3d> is
// {f64, 24, 0, 8, 16}; a PointCloud2 message is f32 at point_step with its field offsets, RosUtils.cpp:30-39).
struct ScanView {
    const unsigned char *base;
    int n;            // number of points (an upper bound when d_n is given)
    const int *d_n;   // optional device-resident count produced by an earlier stage on the same stream
    int stride, ox, oy, oz;
    int f32;
};

// Chunked upload overlapped with the first pass: chunk c (windows [c*windows_per_chunk, ...)) may be read once
// flags[c] == seq — the flag is copied by the same copy stream right after the chunk's data.
struct UploadArgs {
    const uint32_t *flags;  // nullptr: the scan is already resident
    uint32_t seq;
    int windows_per_chunk;  // in 32-point windows
};

struct P2PArgs {
    P2PMailbox *peer[KICP_MAX_RANKS];
    int nranks, rank, parity;
    uint32_t tag_base;  // + pass index = the tag of this registration's words
};

struct KernelArgs {
    RegState *st;
    ScanView scan;
    MapView map;
    double *partials;  // [2][grid][8]
    P2PArgs px;
    UploadArgs up;
    RegArgs init;
    int pow2_voxel;
    int collect_stats;
    // nearest-neighbour cache carried from pass to pass (persistent kernel, option "nn_cache"), one entry per scan point
    unsigned int *nn_g;            // the neighbour found by the last search (global point index, 0xFFFFFFFF = none)
    unsigned int *nn_g2;           // the runner-up of that search (0xFFFFFFFF = none): between passes the two may swap
    float *nn_l;                   // certified lower bound on the distance to every candidate OTHER than those two; for a point that is
                                   // searched again, from the certificate sweep to its search: the distance to the old neighbour from
                                   // the new position (the pruning bound of that search)
    unsigned int *todo;            // points of the current pass that need the search: two cost classes, one from each end ...
    union {
        unsigned int *todo2;       // ... and the other two (same size)
        float *nn_seed;            // (the name the CPU test harness in tests/emu gives this buffer)
    };
    kicp_reg_result *result_host;   // optional: device-visible alias of the caller's page-locked result block (written by CTA 0 at the end)
    unsigned long long timeout_ns;  // device-side waits (upload flags, peers) give up after this long
};


struct RegState;  // device-side state of one registration (kicp_register.cu)

// layout of RegState as far as the host needs it
size_t kr_state_bytes();
size_t kr_offset_result();  // kicp_reg_result
size_t kr_offset_acc();     // double[8]: the sums the NCCL path all-reduces
size_t kr_offset_dbg();     // double[KICP_MAX_ITERATIONS][6]
size_t kr_offset_stats();   // uint64[4] followed by the uint64[24] of -DKR_PROFILE builds
size_t kr_stats_bytes();
size_t kr_smem_bytes();     // dynamic shared memory of k_register
// launches (all on `stream`); every function returns the CUDA error of the launch / query
cudaError_t kr_prepare(int *persistent_ctas_per_sm, int *multilaunch_ctas_per_sm);  // opt-in shared memory + occupancy
cudaError_t kr_launch_init(RegState *st, const RegArgs &a, cudaStream_t stream);
cudaError_t kr_launch_solve(RegState *st, cudaStream_t stream);
cudaError_t kr_window_log(unsigned long long *out, size_t cap_entries, size_t *n);
cudaError_t kr_launch_register(bool persistent, int grid, KernelArgs &ka, cudaStream_t stream);
cudaError_t kr_launch_l2_read(const void *buf, size_t bytes, int reps, unsigned *sink, int grid, cudaStream_t stream);
