"""Occupancy evidence on the GPU (kicp_map_set_occupancy, kicp_map_export_occupancy): host and device clearing calls interleaved with
AddPoints and Update, with and without a frozen prior, against tests/occupancy_oracle.py byte for byte after every call; {1, 0, 1, 1}
against memoryless clearing; the lifecycle (growth, freeze / thaw, load_voxels, Clear, a second set call, off); the frame path in both
synchronisation orders, staged and unstaged, under ALWAYS, GATED (pass and reject), NEVER and with a frozen prior, each frame equal to the
option-off frame followed by ClearFreeSpace with the same occupancy; the launch counts; one sequence at full size; argument validation;
and kicp_replay --occupancy."""
import os

import numpy as np
import pytest

import free_space_oracle as F
import occupancy_oracle as O
from test_gpu_free_space import I7, POLICIES, POSE, ROOT, _bytes, _Drive, _q, _same, _scene, _seq

pytestmark = pytest.mark.gpu

OCC = (2, 1, 1, 3)


def _by_key(voxels, evidence):
    """(key, points, evidence) per voxel sorted by key: two maps fed the same points agree voxel by voxel (inserts race for block ids)"""
    keys, counts, pts = voxels
    starts = np.r_[0, np.cumsum(counts)[:-1]].astype(np.int64)
    order = np.lexsort(np.asarray(keys).T[::-1])
    return [(tuple(keys[v]), pts[starts[v]:starts[v] + counts[v]].tobytes(), int(evidence[v])) for v in order]


class _Expect:
    """the oracle's state beside a GPU map: its export and evidence after every call"""

    def __init__(self, gm, occ):
        self.gm, self.occ = gm, occ
        self.vox = gm.export_voxels()
        self.ev = gm.occupancy() if occ else None

    def check(self):
        assert _bytes(self.gm.export_voxels()) == _bytes(self.vox)
        if self.occ:
            assert self.gm.occupancy().tobytes() == np.ascontiguousarray(self.ev, np.int32).tobytes()

    def carried(self):
        after = self.gm.export_voxels()
        if self.occ:
            self.ev = O.carry(self.vox[0], self.ev, after[0], self.occ[0])
        self.vox = after
        self.check()

    def clear(self, oracle, pts, pose, origin, margin, mm, torch_dtype=None):
        gm = self.gm
        seen = pts
        if torch_dtype is not None:
            import torch
            seen = np.asarray(pts, np.float32).astype(np.float64) if torch_dtype == torch.float32 else pts
            pts = torch.tensor(np.asarray(pts), dtype=torch_dtype, device="cuda")
        want, wev, wst = O.clear(oracle, self.vox, self.ev, gm.num_prior_voxels(), gm.voxel_size_, gm.max_distance_, seen, pose, origin,
                                 margin, mm, self.occ)
        st = gm.ClearFreeSpace(pts, pose, origin, min_misses=mm, end_margin=margin)
        assert st._asdict() == wst
        self.vox, self.ev = want, wev
        self.check()
        assert gm.num_voxels() == len(want[1]) and gm.num_points() == len(want[2])
        return st


@pytest.mark.parametrize("variant", ["host", "f64", "f32"])
@pytest.mark.parametrize("prior", [False, True])
def test_sequences_match_the_oracle(oracle, gpu_ctx, prior, variant):
    import torch

    import kinematic_icp_b200 as kb
    td = {"host": None, "f64": torch.float64, "f32": torch.float32}[variant]
    wall, van, clutter, rays = _scene(11)
    gm = kb.VoxelHashMap(gpu_ctx, 0.5, 30.0, 20)
    try:
        gm.set_occupancy(*OCC)
        x = _Expect(gm, OCC)
        gm.AddPoints(np.concatenate([wall, clutter]))
        x.carried()
        if prior:
            gm.freeze()
        gm.AddPoints(van)
        x.carried()
        cleared = 0
        for margin, mm in ((0.5, 2), (0.0, 1)):
            cleared += x.clear(oracle, rays, POSE, [0.1, 0.0, 0.3], margin, mm, td).cleared_voxels
        gm.Update(van[::4], POSE)  # insert through a pose, then evict around its translation
        x.carried()
        x.clear(oracle, rays[::2], POSE, [0.1, 0.0, 0.3], 0.25, 2, td)
        gm.AddPoints(van[1::4])
        x.carried()
        cleared += x.clear(oracle, rays, I7, [0.0, 0.0, 0.5], 0.5, 1, td).cleared_voxels
        gm.Update(clutter[::3], [40.0, 0.0, 0.0])  # evicts the live voxels beyond 30 m of x = 40
        x.carried()
        x.clear(oracle, rays, POSE, [0.1, 0.0, 0.3], 0.5, 2, td)
        assert cleared > 0
        if not prior:  # (with the prior frozen, the wall's evidence does not move)
            assert len(set(x.ev.tolist())) > 1
        if prior:
            assert gm.occupancy()[:gm.num_prior_voxels()].tolist() == [OCC[0]] * gm.num_prior_voxels()
    finally:
        gm.close()


def test_1_0_1_1_equals_memoryless_clearing(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    wall, van, clutter, rays = _scene(12)
    for prior in (False, True):
        gm = kb.VoxelHashMap(gpu_ctx, 0.5, 30.0, 20)
        try:
            gm.set_occupancy(1, 0, 1, 1)
            gm.AddPoints(np.concatenate([wall, clutter]))
            if prior:
                gm.freeze()
            gm.AddPoints(van)
            for margin, mm in ((0.5, 2), (0.0, 1), (0.25, 3)):
                before = gm.export_voxels()
                want, wst = F.clear_free_space(oracle, before, gm.num_prior_voxels(), 0.5, 30.0, rays, POSE, [0.1, 0.0, 0.3], margin, mm)
                st = gm.ClearFreeSpace(rays, POSE, [0.1, 0.0, 0.3], min_misses=mm, end_margin=margin)
                assert st._asdict() == wst and _bytes(gm.export_voxels()) == _bytes(want)
                assert set(gm.occupancy().tolist()) <= {1}
                gm.Update(van[::3], POSE)
        finally:
            gm.close()


def test_lifecycle(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    wall, van, clutter, rays = _scene(13)
    origin = [0.1, 0.0, 0.3]
    # a small max_distance: the map is sized for 16 384 voxels (8 pi (12 / 0.5)^2 < 16 384)
    gm = kb.VoxelHashMap(gpu_ctx, 0.5, 12.0, 20)
    try:
        with pytest.raises(kb.KicpError):
            gm.occupancy()  # never set
        gm.set_occupancy(*OCC)
        x = _Expect(gm, OCC)
        gm.AddPoints(np.concatenate([wall, clutter, van]))
        x.carried()
        x.clear(oracle, rays, POSE, origin, 0.5, 2)
        x.clear(oracle, rays[::2], POSE, origin, 0.0, 1)
        assert len(set(x.ev.tolist())) > 1
        # growth past the initial capacity keeps the evidence
        rng = np.random.default_rng(3)
        grid = np.stack(np.meshgrid(np.arange(-40, 40), np.arange(-40, 40), np.arange(0, 5)), -1).reshape(-1, 3) * 0.5 + 0.25 + [60, 0, 0]
        grid = grid[rng.permutation(len(grid))]
        assert len(grid) > 16384
        gm.AddPoints(grid)
        assert gm.num_voxels() > 16384
        x.carried()
        x.clear(oracle, rays, POSE, origin, 0.5, 1)
        # freeze / thaw: the prior's evidence stays while frozen and resumes after
        gm.AddPoints(van)  # the van again, then frozen with the rest
        x.carried()
        gm.freeze()
        P = gm.num_prior_voxels()
        ev_prior = gm.occupancy()[:P].copy()
        gm.AddPoints(clutter[::2] + [0.0, 0.0, 0.26])
        x.carried()
        for _ in range(2):
            st = x.clear(oracle, rays, I7, [0.0, 0.0, 0.5], 0.0, 1)
            assert gm.occupancy()[:P].tobytes() == ev_prior.tobytes()
        assert st.prior_contradicted > 0
        gm.thaw()
        x.check()
        x.clear(oracle, rays, POSE, origin, 0.0, 1)
        # a second set call resets every voxel to initial
        gm.set_occupancy(3, 1, 2, 5)
        x.occ, x.ev = (3, 1, 2, 5), np.full(gm.num_voxels(), 3, np.int32)
        x.check()
        x.clear(oracle, rays, POSE, origin, 0.5, 2)
        # load_voxels: every loaded voxel starts at initial
        v = gm.export_voxels()
        gm.load_voxels(*v)
        x.vox, x.ev = v, np.full(len(v[1]), 3, np.int32)
        x.check()
        # Clear() keeps the setting
        gm.Clear()
        assert gm.occupancy().size == 0
        gm.AddPoints(van)
        assert set(gm.occupancy().tolist()) == {3}
        x.vox, x.ev = gm.export_voxels(), gm.occupancy()
        x.clear(oracle, rays, I7, [0.0, 0.0, 0.5], 0.5, 2)
        # off: occupancy() raises and clearing is memoryless
        gm.set_occupancy(None)
        with pytest.raises(kb.KicpError):
            gm.occupancy()
        x.occ, x.ev = None, None
        gm.AddPoints(van)
        x.carried()
        x.clear(oracle, rays, I7, [0.0, 0.0, 0.5], 0.0, 1)
    finally:
        gm.close()


def test_argument_validation_names_the_field_and_keeps_the_setting(gpu_ctx):
    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import _capi
    gm = kb.VoxelHashMap(gpu_ctx, 1.0, 100.0, 20)
    try:
        gm.AddPoints(np.array([[1.0, 2.0, 3.0], [5.0, 2.0, 3.0]]))
        gm.set_occupancy(2, 1, 1, 4)
        for bad, field in (((0, 1, 1, 4), "params->initial"), ((5, 1, 1, 4), "params->initial"), ((1, -1, 1, 4), "params->hit_gain"),
                           ((1, 1, 0, 4), "params->miss_loss"), ((1, 1, 1, 0), "params->max_evidence"),
                           ((1, 1, 1, (1 << 24) + 1), "params->max_evidence")):
            with pytest.raises(kb.KicpError) as e:
                gm.set_occupancy(*bad)
            assert e.value.status == _capi.KICP_ERR_INVALID and field in str(e.value)
            assert gm.occupancy().tolist() == [2, 2]
        import ctypes as C
        n = C.c_int64()
        out = np.zeros(1, np.int32)
        assert _capi.lib().kicp_map_export_occupancy(gm.h, out.ctypes.data_as(_capi.c_ip), 1, C.byref(n)) == _capi.KICP_ERR_CAPACITY
        assert n.value == 2
    finally:
        gm.close()


def test_full_size_cfg4_at_three_poses(oracle, gpu_ctx):
    import kinematic_icp_b200 as kb
    from oracle import workloads as W
    w4 = W.Workload(4)
    keys, counts, mpts = w4.map.export_voxels()
    scan = np.asarray(w4.scan, dtype=np.float64)
    gm = kb.VoxelHashMap(gpu_ctx, w4.voxel_size, w4.max_range, w4.max_points_per_voxel)
    try:
        gm.set_occupancy(*OCC)
        gm.load_voxels(keys, counts, mpts)
        x = _Expect(gm, OCC)
        base = np.asarray(w4.last_pose, dtype=np.float64)
        cleared = 0
        for dx in (0.0, 0.7, -0.4):
            pose = base.copy()
            pose[4] += dx
            st = x.clear(oracle, scan, pose, (0.0, 0.0, 0.0), 0.5, 2)
            assert st.rays == len(scan)
            cleared += st.cleared_voxels
        assert len(set(x.ev.tolist())) > 1
    finally:
        gm.close()


def _frames_equal(kb, a, b, free, occ, l2b, k):
    """one frame of a (the option on) against b (off), then b's standalone call with the same occupancy"""
    oa, la, ua, fa = a.frame(k)
    ob, lb, ub, fb = b.frame(k)
    assert np.array_equal(oa[0], ob[0]), k
    assert bytes(oa[3]) == bytes(ob[3]), k
    assert ua == ub
    if ua == 0:
        down = kb.VoxelDownsample(b.ctx, np.asarray(ob[1], dtype=np.float64), 0.5)
        st = b.gm.ClearFreeSpace(down, ob[0], l2b[4:], min_misses=free[0], end_margin=free[1])
        assert fa == st, k
    else:
        assert fa == kb.FreeSpaceStats(0, 0, 0, 0, 0)
    assert _by_key(a.gm.export_voxels(), a.gm.occupancy()) == _by_key(b.gm.export_voxels(), b.gm.occupancy()), k
    return la, lb, ua, fa


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("staged,frame_sync", [(False, 0), (True, 0), (False, 1), (True, 1)])
def test_frame_path_equals_option_off_frame_then_clearing(oracle, policy, staged, frame_sync):
    import kinematic_icp_b200 as kb
    seq = _seq()
    free = (2, 0.5)
    occ = (2, 1, 1, 4)
    a = _Drive(kb, oracle, seq, staged, frame_sync, free, POLICIES[policy])
    b = _Drive(kb, oracle, seq, staged, frame_sync, None, POLICIES[policy])
    l2b = np.asarray(seq["lidar_to_base"], dtype=np.float64)
    try:
        for d in (a, b):
            d.gm.set_occupancy(*occ)
        for k in range(len(seq["frames"])):
            la, lb, ua, fa = _frames_equal(kb, a, b, free, occ, l2b, k)
            if not frame_sync:  # occupancy adds no launch to the frame
                assert la == lb + (0 if policy == "never" else 2), k
        if policy in ("always", "gated"):
            assert len(set(a.gm.occupancy().tolist())) > 1
    finally:
        a.close()
        b.close()


def test_frame_path_with_a_frozen_prior(oracle):
    import kinematic_icp_b200 as kb
    seq = _seq()
    rng = np.random.default_rng(11)
    ang = rng.uniform(0, 2 * np.pi, 30000)
    ring = np.c_[60 * np.cos(ang), 60 * np.sin(ang), rng.uniform(-1, 3, 30000)]
    start = np.asarray(seq["start"], dtype=np.float64)[4:]
    van = start + np.c_[rng.uniform(3, 5, 3000), rng.uniform(-1, 1, 3000), rng.uniform(0, 1.5, 3000)]
    prior = _q(np.concatenate([ring, van]))
    free, occ = (2, 0.5), (2, 1, 1, 4)
    l2b = np.asarray(seq["lidar_to_base"], dtype=np.float64)
    for frame_sync in (0, 1):
        a = _Drive(kb, oracle, seq, False, frame_sync, free)
        b = _Drive(kb, oracle, seq, False, frame_sync)
        try:
            for d in (a, b):
                d.gm.AddPoints(prior)
                d.gm.freeze()
                d.gm.set_occupancy(*occ)
            P = a.gm.num_prior_voxels()
            head = _bytes(a.gm.export_voxels()[:2])
            for k in range(len(seq["frames"])):
                _frames_equal(kb, a, b, free, occ, l2b, k)
                ea = a.gm.export_voxels()
                assert ea[0][:P].tobytes() == np.frombuffer(head[0], np.int32).reshape(-1, 3)[:P].tobytes()
                assert a.gm.occupancy()[:P].tolist() == [occ[0]] * P
        finally:
            a.close()
            b.close()


def test_golden_drive_1_0_1_1_and_launch_counts(oracle):
    """{1, 0, 1, 1} gives memoryless clearing on the frame path; occupancy never set, set then off, and {1, 0, 1, 1} launch the same
    kernels per frame; occupancy on launches what off launches in AddPoints, the standalone call and Update, and load_voxels adds one
    fill"""
    import kinematic_icp_b200 as kb
    seq = _seq()
    free = (2, 0.5)
    for frame_sync in (0, 1):
        drives = [_Drive(kb, oracle, seq, False, frame_sync, free) for _ in range(4)]
        never, off, on, one = drives
        try:
            off.gm.set_occupancy(2, 1, 1, 4)
            off.gm.set_occupancy(None)
            on.gm.set_occupancy(2, 1, 1, 4)
            one.gm.set_occupancy(1, 0, 1, 1)
            for k in range(len(seq["frames"])):
                outs = [d.frame(k) for d in drives]
                launches = [o[1] for o in outs]
                # (`on` keeps other voxels, so its registration may take another pass: its frames are held to the option-off frame
                # with the same map in test_frame_path_equals_option_off_frame_then_clearing)
                assert launches[0] == launches[1] == launches[3], (k, launches)
                assert outs[3][3] == outs[0][3], k  # {1, 0, 1, 1}: the memoryless statistics
                assert _same(one.gm.export_voxels(), never.gm.export_voxels()), k
                assert set(one.gm.occupancy().tolist()) <= {1}
        finally:
            for d in drives:
                d.close()
    ctx = kb.Context(0)
    try:
        wall, van, clutter, rays = _scene(14)
        counts = {}
        for mode in ("never", "on"):
            gm = kb.VoxelHashMap(ctx, 0.5, 30.0, 20)
            try:
                if mode == "on":  # {1, 0, 1, 1}: the same voxels cleared, so the same compactions
                    gm.set_occupancy(1, 0, 1, 1)
                c = []
                for fn in (lambda: gm.AddPoints(np.concatenate([wall, clutter, van])),
                           lambda: gm.ClearFreeSpace(rays, POSE, [0.0, 0.0, 0.3], min_misses=1, end_margin=0.0),
                           lambda: gm.Update(van[::3], [0.0, 0.0, 0.0]),
                           lambda: gm.load_voxels(*gm.export_voxels())):
                    ctx.synchronize()
                    l0 = ctx.launch_count
                    fn()
                    c.append(ctx.launch_count - l0)
                counts[mode] = c
            finally:
                gm.close()
        assert counts["on"][:3] == counts["never"][:3]
        assert counts["on"][3] == counts["never"][3] + 1
    finally:
        ctx.close()


def test_replay_occupancy(oracle, tmp_path):
    """kicp_replay --free-space 2 --occupancy I,G,L,M (VoxelHashMap::SetOccupancy / Occupancy through KinematicICP::VoxelMap()): the
    setting in the JSON line, and the map's voxels and summed evidence close to the Python frame path's on the same drive (the replay
    ingests float32 records); --occupancy without --free-space is refused"""
    import json
    import subprocess

    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    seq = _seq()
    n = len(seq["frames"])
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    kseq = str(tmp_path / "drive.kseq")
    S2.write_kseq(seq, kseq, header_stamps=[100.0 + 0.1 * k for k in range(n)])
    occ = (2, 1, 1, 4)
    out = subprocess.run([exe, kseq, str(tmp_path / "a.tum"), "--deskew", "1", "--free-space", "2", "--occupancy", "2,1,1,4"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    info = json.loads(out.stdout.strip().splitlines()[-1])
    o = info["occupancy"]
    assert (o["initial"], o["hit_gain"], o["miss_loss"], o["max_evidence"]) == occ
    d = _Drive(kb, oracle, seq, False, 0, (2, 0.5))
    try:
        d.gm.set_occupancy(*occ)
        cleared = 0
        for k in range(n):
            cleared += d.frame(k)[3].cleared_voxels
        ev = d.gm.occupancy()
    finally:
        d.close()
    assert o["voxels"] > 0 and abs(o["voxels"] - len(ev)) <= 0.01 * len(ev)
    assert abs(o["evidence_sum"] - int(ev.sum())) <= 0.02 * int(ev.sum())
    assert abs(info["free_space_stats"]["cleared_voxels"] - cleared) <= max(5, 0.1 * cleared)
    r = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--occupancy", "2,1,1,4"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 2 and "--free-space" in r.stderr
    r = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--free-space", "2", "--occupancy", "0,1,1,4"], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0 and "initial" in r.stderr
