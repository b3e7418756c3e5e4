// Device-side helpers shared by the map and registration kernels.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kicp_internal.h"

// KISS-ICP v1.2.0 VoxelHashMap.cpp `voxel_shifts`: centre, 6 faces, 12 edges, 8 corners.  The visiting order
// matters only for exact distance ties (strict <, first minimum wins) — we keep it so ties resolve identically.
// Packed 2 bits per entry per axis (value + 1) so a lane can decode its shift without a divergent table read.
namespace kicp_dev {
constexpr int kShifts[27][3] = {
    {0, 0, 0},   {1, 0, 0},   {-1, 0, 0},  {0, 1, 0},   {0, -1, 0},  {0, 0, 1},   {0, 0, -1},  {1, 1, 0},   {1, -1, 0},
    {-1, 1, 0},  {-1, -1, 0}, {1, 0, 1},   {1, 0, -1},  {-1, 0, 1},  {-1, 0, -1}, {0, 1, 1},   {0, 1, -1},  {0, -1, 1},
    {0, -1, -1}, {1, 1, 1},   {1, 1, -1},  {1, -1, 1},  {1, -1, -1}, {-1, 1, 1},  {-1, 1, -1}, {-1, -1, 1}, {-1, -1, -1}};
constexpr unsigned long long pack_axis(int a) {
    unsigned long long r = 0;
    for (int k = 0; k < 27; ++k) r |= (unsigned long long)(kShifts[k][a] + 1) << (2 * k);
    return r;
}
constexpr unsigned long long kShiftX = pack_axis(0), kShiftY = pack_axis(1), kShiftZ = pack_axis(2);

// 27-bit masks of the shifts whose x / y / z component is 0, +1, -1 (bit k <-> voxel_shifts[k])
constexpr uint32_t axis_mask(int a, int val) {
    uint32_t r = 0;
    for (int k = 0; k < 27; ++k)
        if (kShifts[k][a] == val) r |= 1u << k;
    return r;
}
constexpr uint32_t kX0 = axis_mask(0, 0), kXP = axis_mask(0, 1), kXM = axis_mask(0, -1);
constexpr uint32_t kY0 = axis_mask(1, 0), kYP = axis_mask(1, 1), kYM = axis_mask(1, -1);
constexpr uint32_t kZ0 = axis_mask(2, 0), kZP = axis_mask(2, 1), kZM = axis_mask(2, -1);

__device__ __forceinline__ int shift_x(int k) { return (int)((kShiftX >> (2 * k)) & 3ull) - 1; }
__device__ __forceinline__ int shift_y(int k) { return (int)((kShiftY >> (2 * k)) & 3ull) - 1; }
__device__ __forceinline__ int shift_z(int k) { return (int)((kShiftZ >> (2 * k)) & 3ull) - 1; }

// Voxel hash: the reference's 3-prime XOR (KISS VoxelUtils.hpp) followed by a murmur3 finaliser so that linear
// probing sees well-mixed low bits.  The hash only decides WHERE a voxel lives, never which neighbour wins.
__host__ __device__ __forceinline__ uint32_t voxel_hash(int x, int y, int z) {
    uint32_t h = ((uint32_t)x * 73856093u) ^ ((uint32_t)y * 19349669u) ^ ((uint32_t)z * 83492791u);
    h ^= h >> 16;
    h *= 0x85ebca6bu;
    h ^= h >> 13;
    h *= 0xc2b2ae35u;
    h ^= h >> 16;
    return h;
}

// PointToVoxel (KISS VoxelUtils.hpp): static_cast<int>(floor(x / voxel_size)).  A true FP64 division, not a
// multiplication by the reciprocal, so voxel boundaries fall exactly where the reference puts them.
__device__ __forceinline__ int voxel_coord(double x, double vs) { return (int)floor(x / vs); }

// DIVERGENCE SAFETY.  nvcc keeps loop-invariant kernel parameters (table mask, base pointers) in UNIFORM registers,
// which are shared by the 32 lanes of a warp.  Inside a per-lane loop (a hash-probe chain, a voxel scan) that is only
// sound while the sibling lanes wait at the reconvergence point; observed under cuda-gdb (DESIGN.md): siblings
// ran past a BSYNC.RECONVERGENT, re-used the uniform register, and the lanes still probing read mask == 0 and spun on
// slot 0 forever.  Two rules keep every kernel in this library safe (scripts/check_ur_loops.py verifies rule 1 on the
// SASS):
//   1. the map view used inside per-lane loops is read back from a PER-LANE copy in shared memory (MapRegs): a value
//      loaded from a lane-dependent address cannot be proven warp-uniform, so ptxas keeps it in per-thread registers
//      (a copy at a uniform address is not enough — ptxas moves it back into a uniform register with R2UR);
//   2. every divergent phase ends with a hard __syncwarp().
struct MapRegs {
    const int4 *slots;
    const double *pts;
    uint32_t mask;
    int cap;
};

// All threads of the CTA call this once at kernel start (it contains a __syncthreads()); shared_copies[32].
__device__ __forceinline__ MapRegs map_regs(const MapView &m, MapView *shared_copies) {
    if (threadIdx.x < 32) shared_copies[threadIdx.x] = m;
    __syncthreads();
    const volatile MapView *v = shared_copies + (threadIdx.x & 31);
    MapRegs r;
    r.slots = v->slots, r.pts = v->pts, r.mask = v->mask, r.cap = v->cap;
    return r;
}

// Same trick for a single scalar or pointer (the table mask of the map-maintenance kernels, ...): shared_words[32].
template <class T>
__device__ __forceinline__ T lane_private(T v, T *shared_words) {
    if (threadIdx.x < 32) shared_words[threadIdx.x] = v;
    __syncthreads();
    return ((const volatile T *)shared_words)[threadIdx.x & 31];
}

// Read-only probe (no concurrent writers): returns the slot's meta word, or KICP_SLOT_EMPTY when absent.
__device__ __forceinline__ uint32_t map_probe(const MapRegs &m, int kx, int ky, int kz) {
    uint32_t h = voxel_hash(kx, ky, kz) & m.mask;
    while (true) {
        const int4 s = __ldg(&m.slots[h]);
        if ((uint32_t)s.w == KICP_SLOT_EMPTY) return KICP_SLOT_EMPTY;
        if (s.x == kx && s.y == ky && s.z == kz) return (uint32_t)s.w;
        h = (h + 1) & m.mask;
    }
}

struct Pose {  // Sophus::SE3d: unit quaternion (x,y,z,w) + translation
    double qx, qy, qz, qw, tx, ty, tz;
};

// Sophus SO3Base::operator*(Point): uv = 2 (q.vec x p); p + w uv + q.vec x uv
__device__ __forceinline__ void quat_rotate(double qx, double qy, double qz, double qw, double px, double py, double pz,
                                            double &ox, double &oy, double &oz) {
    double ux = qy * pz - qz * py, uy = qz * px - qx * pz, uz = qx * py - qy * px;
    ux = ux + ux, uy = uy + uy, uz = uz + uz;
    ox = px + qw * ux + (qy * uz - qz * uy);
    oy = py + qw * uy + (qz * ux - qx * uz);
    oz = pz + qw * uz + (qx * uy - qy * ux);
}
// a + b with one rounding of the exact sum, never contracted with a neighbouring product: an FMA with a unit factor is exactly
// that (and, unlike __dadd_rn, it is among the intrinsics the host-side kernel emulator of tests/emu supplies)
__device__ __forceinline__ double add_rn(double a, double b) { return __fma_rn(a, 1.0, b); }

// The same rotation with every operation rounded on its own (__dmul_rn / add_rn): the reference's plain IEEE result bit for bit
// in a file that is compiled with FMA contraction (kicp_register.cu).
__device__ __forceinline__ void quat_rotate_rn(double qx, double qy, double qz, double qw, double px, double py, double pz,
                                               double &ox, double &oy, double &oz) {
    double ux = add_rn(__dmul_rn(qy, pz), -__dmul_rn(qz, py));
    double uy = add_rn(__dmul_rn(qz, px), -__dmul_rn(qx, pz));
    double uz = add_rn(__dmul_rn(qx, py), -__dmul_rn(qy, px));
    ux = add_rn(ux, ux), uy = add_rn(uy, uy), uz = add_rn(uz, uz);
    ox = add_rn(add_rn(px, __dmul_rn(qw, ux)), add_rn(__dmul_rn(qy, uz), -__dmul_rn(qz, uy)));
    oy = add_rn(add_rn(py, __dmul_rn(qw, uy)), add_rn(__dmul_rn(qz, ux), -__dmul_rn(qx, uz)));
    oz = add_rn(add_rn(pz, __dmul_rn(qw, uz)), add_rn(__dmul_rn(qx, uy), -__dmul_rn(qy, ux)));
}
__device__ __forceinline__ void pose_apply(const Pose &T, double px, double py, double pz, double &ox, double &oy, double &oz) {
    quat_rotate(T.qx, T.qy, T.qz, T.qw, px, py, pz, ox, oy, oz);
    ox += T.tx, oy += T.ty, oz += T.tz;
}

}  // namespace kicp_dev
