"""The frame path's map-update policy on the GPU (kicp_ctx_set_map_update, kicp_frame_map_update): NEVER on a prior map leaves it
bit-identical and registers as the frame path does against that map; GATED rejects a frame given a grossly wrong odometry, in both
synchronisation orders and through RegisterFrame and the staged call, with every outcome the rule applied to the frame's report;
GATED with thresholds that pass everything is ALWAYS plus the report's and the gate's launches; the first frame on an empty map, a
NaN-pose frame and a policy switch; kicp_replay's --save-map / --load-map round trip; and the C++ facade against the C calls."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

import map_update_rule as R
import scenes as S
from test_gpu_parity import sorted_voxels
from test_map_update_cpu import numpy_read

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KW = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
MAP_LAUNCHES = 6  # k_add_find_or_create, k_add_commit, k_mark_far, k_exclusive_sum, k_compact_blocks, k_table_rebuild
REPORT_LAUNCHES = 2  # k_corr_eval, k_corr_finish


def _seq():
    from oracle import sequences as S2
    return S2.unpack_sequence(np.load(os.path.join(GOLDEN, "pipeline_seq.npz")), True)


def _same_map(a, b):
    return all(np.array_equal(x, y) for x, y in zip(sorted_voxels(*a), sorted_voxels(*b)))


def _bytes(v):
    return tuple(a.tobytes() for a in v)


class _Drive:
    """the golden drive frame by frame on one context and map, the threshold as the facade keeps it"""

    def __init__(self, kb, ko, seq, staged=False, frame_sync=0, correspondences=0):
        self.kb, self.ko, self.seq, self.staged = kb, ko, seq, staged
        self.ctx = kb.Context(0)
        self.ctx.set_option("frame_sync", frame_sync)
        self.ctx.set_option("correspondences", correspondences)
        self.gm = kb.VoxelHashMap(self.ctx, 1.0, 100.0, 20)
        self.reset()

    def reset(self):
        self.threshold = self.ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
        self.last = np.array(self.seq["start"], dtype=np.float64)

    def frame(self, k, bad=False):
        """frame k (a scan of another place with `bad`): (pose, launches)"""
        kb, ko, seq = self.kb, self.ko, self.seq
        l2b = seq["lidar_to_base"]
        odom = seq["odoms"][k]
        motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
        tau = self.threshold.compute()
        frame, stamps = seq["frames"][k], seq["stamps"][k]
        if bad:
            frame = _elsewhere(frame)
        if self.staged:
            sf = kb.StageFrame(self.ctx, frame, timestamps=stamps)
            l0 = self.ctx.launch_count
            pose = kb.RegisterStagedFrame(self.gm, sf, motion, l2b, self.last, odom, tau, **KW)[0]
        else:
            l0 = self.ctx.launch_count
            pose = kb.RegisterFrame(self.gm, frame, stamps, motion, l2b, self.last, odom, tau, **KW)[0]
        launches = self.ctx.launch_count - l0
        self.threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(self.last, odom)), pose))
        self.last = pose
        return pose, launches

    def close(self):
        self.gm.close()
        self.ctx.close()


def test_never_on_a_prior_map(oracle):
    """the map built by the golden drive, then the drive again against it under NEVER: after every frame export_voxels is the prior's
    bytes, every outcome SKIPPED, every pose the one a context registers with the same map re-loaded before each frame, and every
    frame launches the map's six kernels fewer; the live publication finds nothing to write"""
    import kinematic_icp_b200 as kb
    seq = _seq()
    n = len(seq["frames"])
    a, b = _Drive(kb, oracle, seq), _Drive(kb, oracle, seq)
    try:
        for k in range(n):
            a.frame(k)
        prior = a.gm.export_voxels()
        b.gm.load_voxels(*prior)
        b.ctx.set_map_update(R.NEVER)
        a.reset()
        mine = b.gm.export_voxels()  # the prior as loaded: its bytes are what must survive
        b.gm.PointcloudF32Live()
        for k in range(n):
            a.gm.load_voxels(*prior)
            pa, la = a.frame(k)
            pb, lb = b.frame(k)
            assert kb.frame_map_update(b.ctx) == R.SKIPPED and kb.frame_map_update(a.ctx) == R.APPLIED
            assert S.same_bits(pa, pb), k
            assert lb == la - MAP_LAUNCHES, (k, la, lb)
            assert _bytes(b.gm.export_voxels()) == _bytes(mine), k
        _, stats = b.gm.PointcloudF32Live()
        assert stats["written"] == 0 and stats["added"] == 0 and stats["removed"] == 0
    finally:
        a.close()
        b.close()


BAD_FRAME = 6


def _elsewhere(frame):
    """the frame as a scan of another place: turned by 1.2 rad about z and moved 30 m"""
    c, s = np.cos(1.2), np.sin(1.2)
    return np.c_[c * frame[:, 0] - s * frame[:, 1] + 30.0, s * frame[:, 0] + c * frame[:, 1] - 20.0, frame[:, 2]]


@pytest.mark.parametrize("frame_sync", [0, 1])
@pytest.mark.parametrize("staged", [False, True])
def test_gated_rejects_a_bad_frame(oracle, frame_sync, staged):
    """GATED on min_fitness between the worst good frame's and the bad one's: the scan of another place is REJECTED, every other APPLIED,
    each outcome the rule applied to kicp_frame_correspondences; the map equals that of ALWAYS with the bad frame's Update skipped
    (NEVER for that frame alone), and the poses are the same bits"""
    import kinematic_icp_b200 as kb
    seq = _seq()
    n = len(seq["frames"])
    probe = _Drive(kb, oracle, seq, correspondences=1)  # the fitness of every frame, the bad one's Update skipped
    try:
        fits = []
        for k in range(n):
            probe.ctx.set_map_update(R.NEVER if k == BAD_FRAME else R.ALWAYS)
            probe.frame(k, k == BAD_FRAME)
            fits.append(kb.frame_correspondences(probe.ctx).fitness)
    finally:
        probe.close()
    good = min(f for k, f in enumerate(fits) if k not in (0, BAD_FRAME))
    assert fits[BAD_FRAME] < good, fits
    min_fit = 0.5 * (good + fits[BAD_FRAME])
    policy = (R.GATED, 0, min_fit, math.inf)
    g = _Drive(kb, oracle, seq, staged=staged, frame_sync=frame_sync)
    t = _Drive(kb, oracle, seq, staged=staged, frame_sync=frame_sync)
    g.ctx.set_map_update(policy[0], min_inliers=policy[1], min_fitness=policy[2], max_inlier_rmse=policy[3])
    try:
        outcomes = []
        for k in range(n):
            empty = g.gm.num_points() == 0
            t.ctx.set_map_update(R.NEVER if k == BAD_FRAME else R.ALWAYS)
            pg, lg = g.frame(k, k == BAD_FRAME)
            pt, lt = t.frame(k, k == BAD_FRAME)
            assert S.same_bits(pg, pt), k
            o = kb.frame_map_update(g.ctx)
            st = kb.frame_correspondences(g.ctx)
            assert st.n_points > 0
            assert o == R.rule_stats(policy, 0, empty, st), (k, o, st)
            outcomes.append(o)
            if frame_sync == 0 and k < BAD_FRAME:  # (from the bad frame on the two maps grow their tables at different frames)
                assert lg == lt + REPORT_LAUNCHES + 1, (k, lg, lt)
            assert _same_map(g.gm.export_voxels(), t.gm.export_voxels()), k
        assert outcomes == [R.REJECTED if k == BAD_FRAME else R.APPLIED for k in range(n)], outcomes
    finally:
        g.close()
        t.close()


@pytest.mark.parametrize("correspondences", [0, 1])
def test_gated_passing_everything_is_always(oracle, correspondences):
    import kinematic_icp_b200 as kb
    seq = _seq()
    a, g = _Drive(kb, oracle, seq, correspondences=correspondences), _Drive(kb, oracle, seq, correspondences=correspondences)
    g.ctx.set_map_update(R.GATED, min_inliers=0, min_fitness=0.0, max_inlier_rmse=math.inf)
    try:
        for k in range(len(seq["frames"])):
            pa, la = a.frame(k)
            pg, lg = g.frame(k)
            assert S.same_bits(pa, pg) and kb.frame_map_update(g.ctx) == kb.frame_map_update(a.ctx) == R.APPLIED
            assert lg - la == (0 if correspondences else REPORT_LAUNCHES) + 1, (k, la, lg)
            assert _same_map(a.gm.export_voxels(), g.gm.export_voxels())
            if correspondences:
                assert kb.frame_correspondences(a.ctx) == kb.frame_correspondences(g.ctx)
    finally:
        a.close()
        g.close()


def test_first_frame_nan_frame_and_policy_switch(oracle):
    import kinematic_icp_b200 as kb
    seq = _seq()
    d = _Drive(kb, oracle, seq)
    try:
        assert kb.frame_map_update(d.ctx) == R.NONE
        d.ctx.set_map_update(R.GATED, min_fitness=1.0, min_inliers=10 ** 9, max_inlier_rmse=1e-300)
        d.frame(0)
        assert kb.frame_map_update(d.ctx) == R.APPLIED and d.gm.num_points() > 0  # the empty-map clause
        d.frame(1)
        assert kb.frame_map_update(d.ctx) == R.REJECTED
        before = _bytes(d.gm.export_voxels())
        # an empty frame: zero correspondences, NaN pose
        for mode, want in ((R.ALWAYS, R.NO_CORRESPONDENCES), (R.GATED, R.NO_CORRESPONDENCES), (R.NEVER, R.SKIPPED)):
            d.ctx.set_map_update(mode)
            pose = kb.RegisterFrame(d.gm, np.zeros((0, 3)), np.zeros(0), seq["odoms"][2], seq["lidar_to_base"], d.last, seq["odoms"][2],
                                    1.0, **KW)[0]
            assert np.isnan(pose).all()
            assert kb.frame_map_update(d.ctx) == want and _bytes(d.gm.export_voxels()) == before
        # a failing set keeps the policy
        with pytest.raises(kb.KicpError):
            d.ctx.set_map_update(R.GATED, min_fitness=2.0)
        n0 = d.gm.num_points()
        d.frame(2)
        assert kb.frame_map_update(d.ctx) == R.SKIPPED and d.gm.num_points() == n0
        d.ctx.set_map_update(R.ALWAYS)
        d.frame(3)
        assert kb.frame_map_update(d.ctx) == R.APPLIED and _bytes(d.gm.export_voxels()) != before
        kb.VoxelDownsample(d.ctx, seq["frames"][0], 0.5)  # another front-end call
        assert kb.frame_map_update(d.ctx) == R.NONE
    finally:
        d.close()


def test_replay_save_and_load_map(oracle, tmp_path):
    """kicp_replay --save-map writes export_voxels of the map the drive built (a Python drive of the same frames); --load-map with
    --map-update never replays the drive against it as the Python NEVER drive does; a voxel size that differs is refused"""
    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    ko = oracle
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    seq = _seq()
    n = len(seq["frames"])
    header = [100.0 + 0.1 * k for k in range(n)]
    kseq, mp = str(tmp_path / "drive.kseq"), str(tmp_path / "drive.kmap")
    S2.write_kseq(seq, kseq, header_stamps=header)
    out = subprocess.run([exe, kseq, str(tmp_path / "a.tum"), "--deskew", "1", "--save-map", mp], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    info = json.loads(out.stdout.strip().splitlines()[-1])
    assert info["map_update"] == "always" and info["map_update_outcomes"]["applied"] == n
    vs, cap, keys, counts, pts = numpy_read(mp)
    assert (vs, cap) == (1.0, 20)
    d = _Drive(kb, ko, seq)
    try:
        for k in range(n):
            d.frame(k)
        # the same voxels and counts, the points to 1e-6: the two drives' thresholds come from two restatements of
        # CorrespondenceThreshold
        a, b = sorted_voxels(keys, counts, pts), sorted_voxels(*d.gm.export_voxels())
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.allclose(a[2], b[2], rtol=0, atol=1e-6)
        d.gm.load_voxels(keys, counts, pts)
        d.ctx.set_map_update(R.NEVER)
        d.reset()
        poses = [d.frame(k)[0] for k in range(n)]
    finally:
        d.close()
    tum = str(tmp_path / "b.tum")
    out = subprocess.run([exe, kseq, tum, "--deskew", "1", "--load-map", mp, "--map-update", "never", "--save-map", str(tmp_path / "c.kmap")],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    info = json.loads(out.stdout.strip().splitlines()[-1])
    assert info["map_update_outcomes"]["skipped"] == n and info["map_points"] == len(pts)
    assert open(str(tmp_path / "c.kmap"), "rb").read() == open(mp, "rb").read()  # the prior map, untouched
    got = np.loadtxt(tum, ndmin=2)
    assert got.shape == (n, 8)
    for row, p in zip(got, poses):
        # TUM: stamp tx ty tz qx qy qz qw, six decimals
        dt, ang = ko.pose_delta(np.r_[row[4:8], row[1:4]], p)
        assert dt <= 2e-6 and ang <= 1e-5, (dt, ang)
    bad = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--voxel-size", "0.5", "--load-map", mp, "--map-update", "never"],
                         capture_output=True, text=True, timeout=300)
    assert bad.returncode != 0 and "differ" in bad.stderr
    bad = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--min-fitness", "0.5"], capture_output=True, text=True, timeout=300)
    assert bad.returncode == 2 and "gated" in bad.stderr


def test_facade_agrees_with_the_c_calls(oracle):
    """KinematicICP::SetMapUpdate sets the process-wide context's policy (kicp_ctx_set_map_update on it), throws on a bad field, and
    LastMapUpdate is kicp_frame_map_update of that context"""
    from kinematic_icp_b200 import _capi
    seq = _seq()
    H = C.CDLL(os.path.join(ROOT, "tests", "hooks", "_build", "libkicp_map_update_hooks.so"))
    F = C.CDLL(os.path.join(ROOT, "tests", "hooks", "_build", "libkicp_facade_hooks.so"))
    H.kmu_set_map_update.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    H.kmu_last_map_update.argtypes = [C.c_void_p]
    H.kmu_default_context.restype = C.c_void_p
    F.kfac_pipeline_create.restype = C.c_void_p
    F.kfac_pipeline_create.argtypes = [C.c_double, C.c_double, C.c_double, C.c_uint, C.c_int, C.c_double, C.c_int, C.c_double, C.c_int,
                                       C.c_int, C.c_double, C.c_int]
    F.kfac_pipeline_register_frame.restype = C.c_int64
    F.kfac_pipeline_register_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                               C.c_void_p]
    F.kfac_pipeline_destroy.argtypes = [C.c_void_p]
    F.kfac_pipeline_num_map_points.restype = C.c_int64
    F.kfac_pipeline_num_map_points.argtypes = [C.c_void_p]
    L = _capi.lib()
    ctx = C.c_void_p(H.kmu_default_context())
    err = C.create_string_buffer(256)
    p = _capi.MapUpdatePolicy(R.GATED, 0, 2.0, math.inf)
    assert H.kmu_set_map_update(C.addressof(p), err, 256) == -1 and b"min_fitness" in err.value
    pipe = F.kfac_pipeline_create(100.0, 0.0, 1.0, 20, 1, 1.0, 10, 1e-3, 1, 1, 0.0, 1)
    try:
        out = np.zeros(7)
        l2b = np.ascontiguousarray(seq["lidar_to_base"], dtype=np.float64)
        counts = []
        for k, mode in enumerate((R.ALWAYS, R.NEVER, R.GATED, R.ALWAYS)):
            p = _capi.MapUpdatePolicy(mode, 0, 0.0, math.inf)
            assert H.kmu_set_map_update(C.addressof(p), err, 256) == 0
            fr = np.ascontiguousarray(seq["frames"][k], dtype=np.float64)
            st = np.ascontiguousarray(seq["stamps"][k], dtype=np.float64)
            od = np.ascontiguousarray(seq["odoms"][k], dtype=np.float64)
            F.kfac_pipeline_register_frame(pipe, fr.ctypes.data, len(fr), st.ctypes.data, len(st), l2b.ctypes.data, od.ctypes.data,
                                           out.ctypes.data)
            o = C.c_int32(-1)
            assert L.kicp_frame_map_update(ctx, C.byref(o)) == 0
            assert H.kmu_last_map_update(C.c_void_p(pipe)) == o.value == (R.SKIPPED if mode == R.NEVER else R.APPLIED), (k, o.value)
            counts.append(F.kfac_pipeline_num_map_points(C.c_void_p(pipe)))
        assert counts[1] == counts[0] and counts[2] != counts[1]
    finally:
        F.kfac_pipeline_destroy(C.c_void_p(pipe))
        p = _capi.MapUpdatePolicy(R.ALWAYS, 0, 0.0, math.inf)
        H.kmu_set_map_update(C.addressof(p), err, 256)
