"""Free-space clearing on the GPU (kicp_map_clear_free_space[_device], kicp_ctx_set_free_space, kicp_frame_free_space): the host and
device variants against the oracle of tests/free_space_oracle.py byte for byte on constructed scenes (a van in front of a wall: cleared
when live, a van voxel holding one endpoint kept, the same van frozen as prior kept and counted) and random ones; the frame path in both
synchronisation orders, staged and unstaged, under ALWAYS, GATED (pass and reject), NEVER and with a frozen prior, each frame equal to
the option-off frame followed by ClearFreeSpace of its down-sampled frame; the launch counts; the live export after clearing; the
multi-sensor rejection and argument validation; and kicp_replay --free-space."""
import os

import numpy as np
import pytest

import free_space_oracle as F
from test_gpu_parity import sorted_voxels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KW = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
I7 = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
POSE = np.array([0.0, 0.0, np.sin(0.05), np.cos(0.05), 0.4, -0.3, 0.1])


def _bytes(v):
    return tuple(np.ascontiguousarray(a).tobytes() for a in v)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(sorted_voxels(*a), sorted_voxels(*b)))


def _q(a):
    return np.round(np.asarray(a) * 1024) / 1024


def _scene(seed, n_rays=3000):
    """a wall at x ~ 12 m, a van of voxels at x in [5, 7), clutter; rays from near the origin to the wall"""
    rng = np.random.default_rng(seed)
    wall = _q(np.c_[np.full(4000, 12.2) + rng.uniform(0, 0.2, 4000), rng.uniform(-6, 6, 4000), rng.uniform(-1, 2, 4000)])
    van = _q(np.c_[rng.uniform(5, 7, 1500), rng.uniform(-1.5, 1.5, 1500), rng.uniform(-0.5, 1.5, 1500)])
    clutter = _q(rng.uniform(-10, 10, (2000, 3)))
    rays = _q(np.c_[np.full(n_rays, 12.3) + rng.uniform(0, 0.05, n_rays), rng.uniform(-5, 5, n_rays), rng.uniform(-0.8, 1.8, n_rays)])
    return wall, van, clutter, rays


def _map(kb, ctx, points, vs=0.5, md=30.0, freeze=False, live=None):
    gm = kb.VoxelHashMap(ctx, vs, md, 20)
    gm.AddPoints(points)
    if freeze:
        gm.freeze()
    if live is not None:
        gm.AddPoints(live)
    return gm


def _check(oracle, gm, pts, pose, origin, margin, mm, device=False, torch_dtype=None):
    before = gm.export_voxels()
    want, wst = F.clear_free_space(oracle, before, gm.num_prior_voxels(), gm.voxel_size_, gm.max_distance_, pts, pose, origin, margin, mm)
    if device:
        import torch
        t = torch.tensor(np.asarray(pts), dtype=torch_dtype, device="cuda")
        st = gm.ClearFreeSpace(t, pose, origin, min_misses=mm, end_margin=margin)
        if torch_dtype == torch.float32:  # the oracle sees the widened float32 values
            want, wst = F.clear_free_space(oracle, before, gm.num_prior_voxels(), gm.voxel_size_, gm.max_distance_,
                                           np.asarray(pts, np.float32).astype(np.float64), pose, origin, margin, mm)
    else:
        st = gm.ClearFreeSpace(pts, pose, origin, min_misses=mm, end_margin=margin)
    assert st._asdict() == wst
    got = gm.export_voxels()
    assert _bytes(got) == _bytes(want)
    assert gm.num_voxels() == len(want[1]) and gm.num_points() == len(want[2])
    return st


def test_van_leaves_the_live_map_and_is_counted_as_prior(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    wall, van, clutter, rays = _scene(1)
    vs = 0.5
    van_keys = {tuple(k) for k in np.floor(van / vs).astype(int).tolist()}
    # live van: cleared; one van voxel that holds a ray's endpoint is kept
    gm = _map(kb, gpu_ctx, np.concatenate([wall, clutter]), live=van)
    try:
        keep_ray = np.array([[6.01, 0.01, 0.51]])
        st = _check(oracle, gm, np.concatenate([rays, keep_ray]), I7, [0.0, 0.0, 0.5], 0.5, 2)
        left = {tuple(k) for k in gm.export_voxels()[0].tolist()} & van_keys
        assert st.cleared_voxels > 0 and st.prior_contradicted == 0
        assert tuple(np.floor(keep_ray[0] / vs).astype(int).tolist()) in left
        # the pose and the sensor origin move the rays: the same scene seen from a moved frame
        _check(oracle, gm, rays, POSE, [0.2, -0.1, 0.4], 0.25, 1)
        # PointcloudF32Live after clearing is still the full export as a multiset
        recs, _ = gm.PointcloudF32Live()
        full = gm.PointcloudF32()
        assert sorted(map(tuple, np.asarray(recs).tolist())) == sorted(map(tuple, full.tolist()))
    finally:
        gm.close()
    # the same van frozen as prior: kept, counted as contradicted
    gm = _map(kb, gpu_ctx, np.concatenate([wall, clutter, van]), freeze=True)
    try:
        st = _check(oracle, gm, rays, I7, [0.0, 0.0, 0.5], 0.5, 2)
        assert st.cleared_voxels == 0 and st.prior_contradicted > 0
    finally:
        gm.close()


@pytest.mark.parametrize("seed", [2, 3, 4])
def test_random_scenes_match_the_oracle_host_and_device(oracle, gpu_ctx, seed):
    import torch

    import kinematic_icp_b200 as kb
    rng = np.random.default_rng(seed)
    world = _q(rng.uniform(-15, 15, (20000, 3)))
    for prior in (False, True):
        gm = _map(kb, gpu_ctx, world[:12000], vs=0.5, md=20.0, freeze=prior, live=world[12000:])
        try:
            pts = _q(rng.uniform(-18, 18, (6000, 3)))
            pose = np.array([0.0, 0.0, np.sin(0.3), np.cos(0.3), 1.0, 2.0, -0.5])
            _check(oracle, gm, pts, pose, [0.1, 0.2, 0.3], 0.3, 1)
            _check(oracle, gm, pts[:3000], POSE, [0.0, 0.0, 0.0], 0.0, 2, device=True, torch_dtype=torch.float64)
            _check(oracle, gm, pts[3000:], I7, [0.5, 0.0, 0.0], 1.0, 1, device=True, torch_dtype=torch.float32)
        finally:
            gm.close()


def test_full_size_cloud_matches_the_oracle(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    rng = np.random.default_rng(9)
    gm = _map(kb, gpu_ctx, _q(rng.uniform(-60, 60, (200000, 3)) * [1, 1, 0.05]), vs=1.0, md=100.0)
    try:
        pts = _q(rng.uniform(-80, 80, (131072, 3)) * [1, 1, 0.05])
        st = _check(oracle, gm, pts, I7, [0.0, 0.0, 1.0], 1.0, 2)
        assert st.rays == len(pts) and st.cleared_voxels > 0
    finally:
        gm.close()


def test_argument_validation(gpu_ctx):
    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import _capi
    gm = kb.VoxelHashMap(gpu_ctx, 1.0, 100.0, 20)
    try:
        gm.AddPoints(np.array([[1.0, 2.0, 3.0]]))
        pts = np.array([[5.0, 0.0, 0.0]])
        for kw, pose, origin in ((dict(min_misses=0, end_margin=0.0), I7, (0, 0, 0)), (dict(min_misses=1, end_margin=-1.0), I7, (0, 0, 0)),
                                 (dict(min_misses=1, end_margin=np.nan), I7, (0, 0, 0)), (dict(min_misses=1, end_margin=np.inf), I7, (0, 0, 0)),
                                 (dict(min_misses=1, end_margin=0.0), [0, 0, 0, 1, np.nan, 0, 0], (0, 0, 0)),
                                 (dict(min_misses=1, end_margin=0.0), I7, (0, np.inf, 0))):
            with pytest.raises(kb.KicpError) as e:
                gm.ClearFreeSpace(pts, pose, origin, **kw)
            assert e.value.status == _capi.KICP_ERR_INVALID
        p = _capi.FreeSpaceParams(0.0, 1)
        o = np.zeros(3)
        st = _capi.FreeSpaceStats()
        L = _capi.lib()
        assert L.kicp_map_clear_free_space(gm.h, None, 1, _capi.dp(I7), _capi.dp(o), p, st) == _capi.KICP_ERR_INVALID
        assert L.kicp_map_clear_free_space(gm.h, _capi.dp(pts), -1, _capi.dp(I7), _capi.dp(o), p, st) == _capi.KICP_ERR_INVALID
        assert L.kicp_map_clear_free_space(gm.h, _capi.dp(pts), 1 << 40, _capi.dp(I7), _capi.dp(o), p, st) == _capi.KICP_ERR_INVALID
        assert L.kicp_map_clear_free_space(None, _capi.dp(pts), 1, _capi.dp(I7), _capi.dp(o), p, st) == _capi.KICP_ERR_INVALID
        assert L.kicp_map_clear_free_space(gm.h, _capi.dp(pts), 1, _capi.dp(I7), _capi.dp(o), p, None) == _capi.KICP_OK  # stats may be NULL
        assert L.kicp_map_clear_free_space_device(gm.h, _capi.dp(pts), 1, 0, 0, 0, 0, 0, _capi.dp(I7), _capi.dp(o), p, st) == \
            _capi.KICP_ERR_INVALID  # host memory
        # the context setting: a failing call keeps the previous one
        ctx = kb.Context(0)
        try:
            ctx.set_free_space(3, 0.5)
            with pytest.raises(kb.KicpError):
                ctx.set_free_space(-1, 0.5)
            with pytest.raises(kb.KicpError):
                ctx.set_free_space(1, -0.5)
            assert kb.frame_free_space(ctx) == kb.FreeSpaceStats(0, 0, 0, 0, 0)
        finally:
            ctx.close()
    finally:
        gm.close()


def _seq():
    from oracle import sequences as S2
    return S2.unpack_sequence(np.load(os.path.join(GOLDEN, "pipeline_seq.npz")), True)


class _Drive:
    """the golden drive on one context and map, the threshold as the facade keeps it"""

    def __init__(self, kb, ko, seq, staged, frame_sync, free=None, policy=None):
        self.kb, self.ko, self.seq, self.staged = kb, ko, seq, staged
        self.ctx = kb.Context(0)
        self.ctx.set_option("frame_sync", frame_sync)
        if policy:
            self.ctx.set_map_update(*policy[0], **policy[1])
        if free:
            self.ctx.set_free_space(*free)
        self.gm = kb.VoxelHashMap(self.ctx, 1.0, 100.0, 20)
        self.threshold = ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
        self.last = np.array(seq["start"], dtype=np.float64)

    def frame(self, k):
        kb, ko, seq = self.kb, self.ko, self.seq
        l2b = seq["lidar_to_base"]
        odom = seq["odoms"][k]
        motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
        tau = self.threshold.compute()
        frame, stamps = seq["frames"][k], seq["stamps"][k]
        if self.staged:
            sf = kb.StageFrame(self.ctx, frame, timestamps=stamps)
            l0 = self.ctx.launch_count
            out = kb.RegisterStagedFrame(self.gm, sf, motion, l2b, self.last, odom, tau, **KW)
        else:
            l0 = self.ctx.launch_count
            out = kb.RegisterFrame(self.gm, frame, stamps, motion, l2b, self.last, odom, tau, **KW)
        launches = self.ctx.launch_count - l0
        pose = out[0]
        self.threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(self.last, odom)), pose))
        self.last = pose
        return out, launches, kb.frame_map_update(self.ctx), kb.frame_free_space(self.ctx)

    def close(self):
        self.gm.close()
        self.ctx.close()


POLICIES = {
    "always": None,
    "gated": ((2,), dict(min_inliers=0, min_fitness=0.5)),
    "gated_reject": ((2,), dict(min_inliers=0, min_fitness=1.0)),
    "never": ((1,), {}),
}


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("staged,frame_sync", [(False, 0), (True, 0), (False, 1), (True, 1)])
def test_frame_path_equals_option_off_frame_then_clearing(oracle, policy, staged, frame_sync):
    import kinematic_icp_b200 as kb
    seq = _seq()
    free = (2, 0.5)
    a = _Drive(kb, oracle, seq, staged, frame_sync, free, POLICIES[policy])
    b = _Drive(kb, oracle, seq, staged, frame_sync, None, POLICIES[policy])
    l2b = np.asarray(seq["lidar_to_base"], dtype=np.float64)
    total = 0
    try:
        for k in range(len(seq["frames"])):
            oa, la, ua, fa = a.frame(k)
            ob, lb, ub, fb = b.frame(k)
            assert np.array_equal(oa[0], ob[0]), k  # pose
            assert bytes(oa[3]) == bytes(ob[3]), k  # result block
            assert np.array_equal(oa[1], ob[1]) and np.array_equal(oa[2], ob[2]), k  # clouds
            assert kb.frame_correspondences(a.ctx) == kb.frame_correspondences(b.ctx)
            assert ua == ub
            if ua == 0:  # APPLIED: the option-off frame followed by the standalone call
                down = kb.VoxelDownsample(b.ctx, np.asarray(ob[1], dtype=np.float64), 0.5)
                st = b.gm.ClearFreeSpace(down, ob[0], l2b[4:], min_misses=free[0], end_margin=free[1])
                assert fa == st, k
            else:
                assert fa == kb.FreeSpaceStats(0, 0, 0, 0, 0)
            if not frame_sync:  # the two kernels run whenever the Update's launches do (a rejected frame runs them over an unchanged map)
                assert la == lb + (0 if policy == "never" else 2), k
            total += fa.cleared_voxels
            assert _same(a.gm.export_voxels(), b.gm.export_voxels()), k
        if policy == "never":
            assert a.gm.num_points() == 0
    finally:
        a.close()
        b.close()


def test_frame_path_with_a_frozen_prior(oracle):
    import kinematic_icp_b200 as kb
    seq = _seq()
    rng = np.random.default_rng(11)
    # a prior: a wall ring around the drive and a 'van' patch near its start, frozen
    ang = rng.uniform(0, 2 * np.pi, 30000)
    ring = np.c_[60 * np.cos(ang), 60 * np.sin(ang), rng.uniform(-1, 3, 30000)]
    start = np.asarray(seq["start"], dtype=np.float64)[4:]
    van = start + np.c_[rng.uniform(3, 5, 3000), rng.uniform(-1, 1, 3000), rng.uniform(0, 1.5, 3000)]
    prior = _q(np.concatenate([ring, van]))
    a = _Drive(kb, oracle, seq, False, 0, (2, 0.5))
    b = _Drive(kb, oracle, seq, False, 0)
    l2b = np.asarray(seq["lidar_to_base"], dtype=np.float64)
    try:
        for d in (a, b):
            d.gm.AddPoints(prior)
            d.gm.freeze()
        P = a.gm.num_prior_voxels()
        prior_bytes = _bytes(a.gm.export_voxels())
        for k in range(len(seq["frames"])):
            oa, la, ua, fa = a.frame(k)
            ob, lb, ub, fb = b.frame(k)
            assert np.array_equal(oa[0], ob[0]), k
            if ua == 0:
                down = kb.VoxelDownsample(b.ctx, np.asarray(ob[1], dtype=np.float64), 0.5)
                st = b.gm.ClearFreeSpace(down, ob[0], l2b[4:], min_misses=2, end_margin=0.5)
                assert fa == st, k
                assert la == lb + 2
            ea = a.gm.export_voxels()
            assert _same(ea, b.gm.export_voxels()), k
            assert a.gm.num_prior_voxels() == P
            keys, counts, pts = ea
            pb = prior_bytes
            assert keys[:P].tobytes() == np.frombuffer(pb[0], np.int32).reshape(-1, 3)[:P].tobytes()
    finally:
        a.close()
        b.close()


def test_multi_sensor_frames_are_refused_with_the_option_on(oracle):
    import kinematic_icp_b200 as kb
    seq = _seq()
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    try:
        gm.AddPoints(np.asarray(seq["frames"][0], dtype=np.float64))
        before = _bytes(gm.export_voxels())
        ctx.set_free_space(2, 0.5)
        l2b = seq["lidar_to_base"]
        frame, stamps = seq["frames"][1], seq["stamps"][1]
        staged = kb.StageSensors(ctx, [kb.PointCloudSensor(frame, timestamps=stamps), kb.PointCloudSensor(frame, timestamps=stamps)])
        with pytest.raises(kb.KicpError) as e:
            kb.RegisterStagedSensors(gm, staged, [oracle.IDENTITY] * 2, [l2b] * 2, seq["start"], oracle.IDENTITY, 1.0, **KW)
        assert "single-sensor" in str(e.value)
        assert _bytes(gm.export_voxels()) == before
        # the staged frame was consumed
        with pytest.raises(kb.KicpError):
            kb.RegisterStagedSensors(gm, staged, [oracle.IDENTITY] * 2, [l2b] * 2, seq["start"], oracle.IDENTITY, 1.0, **KW)
        # off again: the multi-sensor call runs
        ctx.set_free_space(0, 0.0)
        staged = kb.StageSensors(ctx, [kb.PointCloudSensor(frame, timestamps=stamps), kb.PointCloudSensor(frame, timestamps=stamps)])
        kb.RegisterStagedSensors(gm, staged, [oracle.IDENTITY] * 2, [l2b] * 2, seq["start"], oracle.IDENTITY, 1.0, **KW)
    finally:
        gm.close()
        ctx.close()


def test_replay_free_space(oracle, tmp_path):
    """kicp_replay --free-space M[,E] (KinematicICP::SetFreeSpace / LastFreeSpace): the setting and the statistics summed over the
    drive in its JSON line, close to the Python frame path's on the same drive (the replay ingests float32 records); malformed values
    are refused"""
    import json
    import subprocess

    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    seq = _seq()
    n = len(seq["frames"])
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    kseq = str(tmp_path / "drive.kseq")
    S2.write_kseq(seq, kseq, header_stamps=[100.0 + 0.1 * k for k in range(n)])
    out = subprocess.run([exe, kseq, str(tmp_path / "a.tum"), "--deskew", "1", "--free-space", "2,0.5"], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stderr
    info = json.loads(out.stdout.strip().splitlines()[-1])
    assert info["free_space"] == {"min_misses": 2, "end_margin": 0.5}
    st = info["free_space_stats"]
    d = _Drive(kb, oracle, seq, False, 0, (2, 0.5))
    try:
        total = [0, 0, 0]
        for k in range(n):
            fs = d.frame(k)[3]
            total[0] += fs.rays
            total[1] += fs.visits
            total[2] += fs.cleared_voxels
    finally:
        d.close()
    assert total[0] > 0 and st["rays"] > 0
    assert abs(st["rays"] - total[0]) <= 0.01 * total[0]
    assert abs(st["visits"] - total[1]) <= 0.02 * total[1]
    assert st["cleared_voxels"] > 0 and st["prior_contradicted"] == 0
    for bad in ("0", "2,-1", "x", "2,", "2,0.5x"):
        r = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--free-space", bad], capture_output=True, text=True, timeout=300)
        assert r.returncode == 2 and "--free-space" in r.stderr, bad
