// Host-side emulation of the planar alignment (kinematic-icp_b200/csrc/kicp_align_kernels.cuh): k_align_eval at any grid, k_align_step
// and k_align_finish, driven by kicp_align.cu's launch sequence restated here on host memory, on a map built by the launch sequences
// of tests/emu/km_emu.cpp.  Also records every iteration's state (the per-iteration trajectory the library does not return) and
// exports the arithmetic of kicp_align.h alone for tests/test_align_planar_cpu.py.  Test infrastructure
// (tests/test_align_planar_emu_cpu.py); never part of the product library.
#include "km_emu.cpp"

#include "../../kinematic-icp_b200/csrc/kicp_align_kernels.cuh"

extern "C" {
// kicp_align.h: T [+] dx, the LDL^T solve (1 when it succeeds), the step norm, and one step of a state from summed partials
void kal_update(const double *T, const double *dx, double *out) { align_update(T, dx, out); }
int kal_solve(const double *A, const double *b, double *dx) { return align_solve(A, b, dx) ? 1 : 0; }
double kal_step_norm(const double *dx) { return align_step_norm(dx); }
int32_t kal_align_slots(int64_t n) { return align_slots(n); }
int32_t kal_state_size() { return (int32_t)sizeof(AlignState); }

// The whole call under the emulator with k_align_eval on `grid` CTAs.  traj[a][it][7] (max_iterations entries per alignment): the
// pose after each k_align_step (the pose before it when the alignment had already stopped), status[a][it] likewise.  Returns 0, or
// -1 for a bad grid.
int kal_emu_align(void *h, const double *src, int64_t n, const double *initial, int32_t n_initial, const kicp_planar_align_params *p,
                  int32_t grid, kicp_planar_alignment *out, double *traj, int32_t *traj_status) {
    EmuMap &m = *static_cast<EmuMap *>(h);
    if (grid <= 0 || n_initial < 1 || n_initial > kAlignMaxInitial) return -1;
    const MapView v = m.view();
    const int C = align_slots(n);
    std::vector<double> part((size_t)n_initial * C * kAlignStride, NAN);
    std::vector<AlignState> state((size_t)n_initial);
    for (int32_t a = 0; a < n_initial; ++a) {
        AlignState &s = state[a];
        for (int k = 0; k < 7; ++k) s.pose[k] = initial[7 * a + k];
        s.status = KICP_ALIGN_MAX_ITERATIONS, s.iterations = 0, s.last_step = 0.0, s.done = 0, s.pad = 0;
    }
    double *pp = part.data();
    AlignState *st = state.data();
    const double tau = p->tau, conv = p->convergence;
    const int step_grid = (n_initial + 7) / 8;
    for (int32_t it = 0; it < p->max_iterations; ++it) {
        emu::launch_waves(grid, kAlignThreads, [=]() { k_align_eval(v, src, n, tau, st, n_initial, 0, pp); });
        emu::launch_waves(step_grid, 256, [=]() { k_align_step(pp, n, n_initial, conv, st); });
        for (int32_t a = 0; a < n_initial; ++a) {
            for (int k = 0; k < 7; ++k) traj[((size_t)a * p->max_iterations + it) * 7 + k] = state[a].pose[k];
            traj_status[(size_t)a * p->max_iterations + it] = state[a].status;
        }
    }
    emu::launch_waves(grid, kAlignThreads, [=]() { k_align_eval(v, src, n, tau, st, n_initial, 1, pp); });
    emu::launch_waves(step_grid, 256, [=]() { k_align_finish(pp, n, n_initial, st, out); });
    return 0;
}
}
