"""The registration kernel's LOGIC, checked without a GPU: kinematic-icp_b200/csrc/kicp_register.cu is compiled unchanged by g++
against a small SIMT emulator (tests/emu/cuda_emu.hpp: one fiber per CUDA thread, warp collectives and __syncthreads() as
rendezvous points, one OS thread per CTA, real atomics between CTAs and between "ranks") and run as a multi-CTA grid on a map laid
out exactly as the device holds it.  Covered: the persistent kernel with and without neighbour certificates, the one-launch-per-
pass path (k_reg_init / k_register<false> / k_solve), several registrations in a row on the same state, float32 ingest, the edge
cases of the GPU suite, the reference's golden poses — and the SHARDED path: two emulated ranks exchanging their sums through the
peer mailboxes, whose poses must be bit-identical to each other (on the GPU box that path needs two GPUs to run at all).

The results must equal the CPU oracle's: pose within the north-star tolerance, the same number of iterations, the same integer
correspondence count in every pass (any neighbour or gate flip would show there).

This is test infrastructure: nothing here is linked into the product, and the GPU parity tests remain the proof for the device
build — the emulator cannot see the GPU memory model, launch limits or register-level hazards."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL_T, TOL_R = 1e-6, 1e-7


from emu import harness as H
import scenes as S


@pytest.fixture(scope="module")
def emu():
    return H.kr_lib()


def run_emu(lib, om, scan, last, odom, tau, **kw):
    return H.register(om, scan, last, odom, tau, **kw)


def check(lib, ko, om, scan, last, odom, tau, **kw):
    res, stats = run_emu(lib, om, scan, last, odom, tau, **kw)
    okw = {k: kw[k] for k in ("max_iter", "conv", "adaptive", "fixed_reg") if k in kw}
    po, st = om.register(np.asarray(scan, dtype=np.float64), last, odom, tau, **okw)
    for r in res:
        dt, ang = ko.pose_delta(r.pose_np(), po)
        assert dt <= TOL_T and ang <= TOL_R, (dt, ang)
        assert r.iterations == st.iterations
        assert np.array_equal(r.sums_np()[:, 5], st.sums_np()[:, 5])
        assert np.allclose(r.sums_np()[:, :5], st.sums_np()[:, :5], rtol=1e-9, atol=1e-9)
        assert r.beta == pytest.approx(st.beta, rel=1e-10)
    for r in res[1:]:  # every rank of a sharded registration holds the very same result
        assert np.array_equal(r.pose_np(), res[0].pose_np()) and np.array_equal(r.sums_np(), res[0].sums_np())
    return res[0], stats


@pytest.mark.parametrize("cfg,grid,persistent,nn_cache", [(1, 1, 1, 1), (1, 3, 1, 0), (1, 2, 0, 0), (2, 4, 1, 1), (2, 3, 1, 0), (2, 3, 0, 0)])
def test_kernel_matches_oracle(emu, oracle, workload, cfg, grid, persistent, nn_cache):
    ko = oracle
    w = workload(cfg)
    r, stats = check(emu, ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=grid, persistent=persistent, nn_cache=nn_cache)
    assert stats[0] >= w.N and stats[1] > 0 and stats[2] > 0
    # float32 ingest: the workload's coordinates are float32-representable, so the same pose (the sums may differ in their last bits:
    # with certificates the order of the repeat list depends on atomic arrival)
    r32, _ = check(emu, ko, w.map, w.scan.astype(np.float32), w.last_pose, w.rel_odom, w.tau, grid=grid, persistent=persistent, nn_cache=nn_cache)
    dt, ang = ko.pose_delta(r32.pose_np(), r.pose_np())
    assert dt <= 1e-12 and ang <= 1e-12


@pytest.mark.parametrize("cfg,grid,nranks,nn_cache", [(1, 2, 2, 1), (2, 2, 2, 1), (2, 2, 3, 0), (2, 1, 8, 1), (1, 1, 4, 0)])
def test_sharded_ranks_agree_bit_for_bit(emu, oracle, workload, cfg, grid, nranks, nn_cache):
    """kicp_register_sharded's fused exchange: every rank writes its 8 sums into every rank's mailbox as tagged 8-byte words, every
    CTA adds them in rank order — identical inputs, identical order, identical pose on all ranks; three registrations in a row
    exercise the mailbox parity and the growing tags."""
    ko = oracle
    w = workload(cfg)
    check(emu, ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=grid, nranks=nranks, nn_cache=nn_cache, registrations=3)


@pytest.mark.parametrize("cfg,n,grid", [(1, None, 2), (2, None, 3), (1, 100, 2)])
def test_frame_uploaded_while_the_kernel_runs(emu, oracle, workload, cfg, n, grid):
    """The host-pointer entry points launch the persistent kernel first and issue the frame's chunks right after; the first pass
    takes every chunk as its flag rises.  Here the kernel starts on a buffer full of NaN and an uploader thread fills it in segment by
    segment, raising each flag after its bytes: any window that read its segment before the flag would poison the sums."""
    ko = oracle
    w = workload(cfg)
    scan = w.scan if n is None else w.scan[:n]
    check(emu, ko, w.map, scan, w.last_pose, w.rel_odom, w.tau, grid=grid, late_upload=1, registrations=2)
    check(emu, ko, w.map, scan.astype(np.float32), w.last_pose, w.rel_odom, w.tau, grid=grid, late_upload=1)


@pytest.mark.parametrize("seed", [1])
def test_interleaving_stress(oracle, workload, seed):
    """The same checks in a fresh process with KICP_EMU_CHAOS = seed: every atomic, fence and L2 load / store of the kernel
    additionally gives the fiber's turn away with probability 1/4, so lanes, warps and ranks interleave in many more orders than the
    round robin produces — certificates, the sharded exchange and the upload flags included."""
    import subprocess
    import sys
    env = dict(os.environ, KICP_EMU_CHAOS=str(seed))
    sel = "(sharded and 1-2-2-1) or (sharded and 2-2-2-1) or (uploaded and 1-) or (matches_oracle and 1-)"  # (other seeds, other cases: by hand)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-k", sel, "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.parametrize("count", [0, 1, 700, 1992])
def test_point_count_read_from_device_memory(emu, oracle, workload, count):
    """kicp_register_frame registers a frame whose survivor count only exists on the device: the grid is planned for an upper bound,
    the kernel reads the count itself.  The points beyond the count (here far away, they would all be rejected — or poison N) are not
    part of the frame."""
    from kinematic_icp_b200 import _capi
    ko = oracle
    w = workload(1)
    count = min(count, w.N)
    buf = np.concatenate([w.scan[:count], np.full((w.N - count, 3), np.nan)])
    res, _ = run_emu(emu, w.map, buf, w.last_pose, w.rel_odom, w.tau, grid=3, device_count=count)
    if count == 0:
        assert np.all(np.isnan(res[0].pose_np())) and res[0].status == _capi.KICP_WARN_NO_CORRESPONDENCES
        return
    po, st = w.map.register(w.scan[:count], w.last_pose, w.rel_odom, w.tau)
    dt, ang = ko.pose_delta(res[0].pose_np(), po)
    assert dt <= TOL_T and ang <= TOL_R and res[0].iterations == st.iterations
    assert np.array_equal(res[0].sums_np()[:, 5], st.sums_np()[:, 5])


def test_kernel_edge_cases(emu, oracle, workload):
    from kinematic_icp_b200 import _capi
    ko = oracle
    w = workload(1)
    for n in (1, 31, 32, 33, 1000):  # ragged sizes around the 32-point window
        check(emu, ko, w.map, w.scan[:n], w.last_pose, w.rel_odom, w.tau, grid=2)
        check(emu, ko, w.map, w.scan[:n], w.last_pose, w.rel_odom, w.tau, grid=2, nranks=2)
    # no correspondences: NaN pose as in the reference, plus a status; the empty frame
    res, _ = run_emu(emu, w.map, w.scan + 500.0, w.last_pose, w.rel_odom, w.tau, grid=2)
    assert np.all(np.isnan(res[0].pose_np())) and res[0].status == _capi.KICP_WARN_NO_CORRESPONDENCES
    res, _ = run_emu(emu, w.map, np.zeros((0, 3)), w.last_pose, w.rel_odom, w.tau, grid=1)
    assert np.all(np.isnan(res[0].pose_np()))
    # strict gate and max_iter = 1, fixed regularisation, many iterations, several registrations on the same state
    check(emu, ko, w.map, w.scan, w.last_pose, w.rel_odom, 0.3, grid=2, max_iter=1)
    check(emu, ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=2, adaptive=False, fixed_reg=2.0)
    check(emu, ko, w.map, w.scan, w.last_pose, w.rel_odom, w.tau, grid=3, conv=1e-6, max_iter=40, registrations=2)
    # points not representable in float32, a general 3-D pose
    rng = np.random.default_rng(2)
    scan = w.scan + rng.normal(size=w.scan.shape) * 1e-3
    last = ko.se3_compose(w.last_pose, ko.se3_exp([0, 0, 0, 0.01, -0.02, 0.0]))
    check(emu, ko, w.map, scan, last, w.rel_odom, w.tau, grid=2)


@pytest.mark.parametrize("name", ["reg_cfg1", "reg_cfg2_small"])
def test_kernel_vs_reference_golden(emu, oracle, name):
    """Final pose against the pose the reference's own Registration.cpp produced (tests/golden)."""
    ko = oracle
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    om = ko.OracleMap(float(z["voxel_size"]), float(z["max_range"]), int(z["max_points_per_voxel"]))
    om.add_points(z["map_points"])
    for case in z["cases"]:
        r, _ = check(emu, ko, om, z["scan"], z["last_pose"], z["rel_odom"], case[4], grid=3, max_iter=int(case[0]), conv=case[1],
                     adaptive=bool(case[2]), fixed_reg=case[3])
        dt, ang = ko.pose_delta(r.pose_np(), case[5:])
        assert dt <= TOL_T and ang <= TOL_R, (dt, ang)


# ------------------------------------------------------------------------------------------ ties, map shapes, randomised scenes
TIE_IDS = ["permuted-vs1", "permuted-vs0.5", "permuted-rotated", "stage-vs1", "stage-vs0.5", "near-vs1", "near-vs0.5", "near-rotated"]
SHAPE_IDS = ["vs0.3-cap1", "vs0.75-cap24", "vs0.6-cap25", "vs0.75-cap29-far", "vs0.3-cap255", "vs0.75-cap20-utm"]
LAUNCHES = [(1, 1, 0), (2, 1, 1), (3, 0, 0)]  # (grid, persistent, certificates)


@pytest.fixture(scope="module")
def tie_scenes(oracle):
    return S.tie_scenes(oracle)


@pytest.fixture(scope="module")
def shape_scenes(oracle):
    return S.shape_scenes(oracle)


@pytest.mark.parametrize("k", range(len(TIE_IDS)), ids=TIE_IDS)
def test_neighbour_ties_match_reference(emu, oracle, tie_scenes, k):
    """Exact ties and ulp-level near-ties of the first pass: the kernel must take the reference's point at every query (exact N,
    sums to 1e-9, the pose).  Each permuted-tie scene holds pairs at which squaring with an FMA picks the other point."""
    sc = tie_scenes[k]
    if TIE_IDS[k].startswith("permuted"):
        assert sc.traps >= 5, sc.traps
    for grid, persistent, cache in LAUNCHES:
        check(emu, oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, grid=grid, persistent=persistent, nn_cache=cache, **sc.kw)


def test_map_kernel_nearest_on_ties(oracle, tie_scenes):
    """The map kernels' batched GetClosestNeighbor (built without FMA contraction) on the same ties: point and distance bit for bit."""
    for sc in tie_scenes:
        em = H.EmuMap(sc.voxel_size, S.FAR, sc.cap)
        try:
            em.load_voxels(*sc.voxels)
            q = sc.queries(oracle)
            pe, de = em.nearest(q)
            po, do = sc.om.nearest(q)
            assert np.array_equal(de, do) and np.array_equal(pe, po), sc.name
        finally:
            em.close()


@pytest.mark.parametrize("k", range(len(SHAPE_IDS)), ids=SHAPE_IDS)
def test_map_shapes_match_oracle(emu, oracle, shape_scenes, k):
    """Voxel sizes that are not powers of two (the division branch of voxel_of), voxels filled to caps of 1 to 255 (fewer than 32
    tasks per batch, a full line buffer), queries exactly on voxel faces and at negative coordinates, maps far from the origin."""
    sc = shape_scenes[k]
    assert np.frexp(sc.voxel_size)[0] != 0.5 and np.all(sc.voxels[1] == sc.cap)
    for grid, persistent, cache in LAUNCHES:
        check(emu, oracle, sc.om, sc.scan, sc.last, sc.odom, sc.tau, grid=grid, persistent=persistent, nn_cache=cache, **sc.kw)


def test_fuzz_scenes_vs_reference(emu, oracle):
    """The 40 randomised scenes of the oracle's pin (voxel 0.5 / 1 / 2, caps 1 / 5 / 20, gates from 5 cm to 3 m, 0 to 25
    iterations, empty scans) through the kernel, against the poses the reference's own sources returned: same NaN pattern, pose
    within the north-star tolerance.  Launch shapes and certificates alternate from scene to scene."""
    ref = np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))["poses"]
    ran = 0
    for case, (om, _, _, _, scan, last, odom, tau, kw) in enumerate(S.fuzz_cases(oracle)):
        res, _ = run_emu(emu, om, scan, last, odom, tau, grid=1 + case % 3, nn_cache=case % 2, **kw)
        pose, pr = res[0].pose_np(), ref[case]
        assert np.array_equal(np.isnan(pose), np.isnan(pr)), (case, kw)
        if not np.isnan(pr).any():
            dt, ang = oracle.pose_delta(pose, pr)
            assert dt <= TOL_T and ang <= TOL_R, (case, kw, dt, ang)
        ran += 1
    assert case == 39 and ran == 40
