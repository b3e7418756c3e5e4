// The registration emulator (kr_emu.cpp) as tests/emu/variants.py builds it: plain (-ffp-contract=off) and with FMA contraction
// (-O2 -mfma -ffp-contract=fast, as nvcc compiles kicp_register.cu), plus the entry points that check a build.
//
// __dmul_rn is one rounded product on the device.  cuda_emu.hpp's plain `a * b` could be fused into the add_rn that follows once
// the compiler contracts, so here the product goes through an empty asm that makes it opaque: the pinned helpers of the kernel
// (dist2, query_rn) stay unfused in both builds, and only its unpinned expressions are contracted.
#define EMU_CHAOS 1  // (as kr_emu.cpp sets it, which includes this header only after us)
#define __dmul_rn kr_emu_plain_dmul_rn
#include "cuda_emu.hpp"
#undef __dmul_rn
inline double __dmul_rn(double a, double b) {
    double r = a * b;
#if defined(__x86_64__)
    __asm__ volatile("" : "+x"(r));
#else
    __asm__ volatile("" : "+m"(r));
#endif
    return r;
}

#include "kr_emu.cpp"

// kr_emu_probe_fma: a * b + c written plainly, as the kernel writes its unpinned expressions — fused in a build that contracts, two
// roundings in one that does not.  kr_emu_dist2 / kr_emu_query: the kernel's pinned square and query (dist2, query_rn), which must
// come out as the reference's in every build.
extern "C" double kr_emu_probe_fma(double a, double b, double c) { return a * b + c; }
extern "C" double kr_emu_dist2(const double c[3], const double q[3]) { return dist2(c[0], c[1], c[2], q[0], q[1], q[2]); }
extern "C" void kr_emu_query(const double pose[7], const double p[3], double out[3]) {
    query_rn(pose, pose + 4, p[0], p[1], p[2], out[0], out[1], out[2]);
}
