"""A frozen prior inside the voxel map on the GPU (kicp_map_freeze / kicp_map_thaw / kicp_map_pointcloud_layer): thaw gives the map a
never-frozen map holds; every map mutator on a frozen map matches the oracle of tests/prior_map_oracle.py (prior voxels beyond
max_distance survive, the prior prefix stays byte-identical); the golden drive against a frozen prior under ALWAYS and GATED, in both
synchronisation orders, staged and unstaged, registers against the union map and updates only the live layer with the map's six
launches, exports between frames included; growth while frozen; the layer exports; clear, load, double freeze and an empty live layer;
kicp_replay --load-map --freeze-prior; and the C++ facade against the C calls."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import map_update_rule as R
import scenes as S
from prior_map_oracle import PriorMap
from test_gpu_parity import sorted_voxels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KW = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
MAP_LAUNCHES = 6  # k_add_find_or_create, k_add_commit, k_mark_far, k_exclusive_sum, k_compact_blocks, k_table_rebuild
FAR = 400.0  # the far copy of the prior lies this far along x: beyond max_distance from every pose of the drive


def _seq():
    from oracle import sequences as S2
    return S2.unpack_sequence(np.load(os.path.join(GOLDEN, "pipeline_seq.npz")), True)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(sorted_voxels(*a), sorted_voxels(*b)))


def _bytes(v):
    return tuple(np.ascontiguousarray(a).tobytes() for a in v)


def _prefix(v, nv):
    """the first nv voxels of an export (keys, counts, points)"""
    keys, counts, pts = v
    return keys[:nv], counts[:nv], pts[:int(counts[:nv].sum())]


def _shifted(prior, dx):
    """the voxels moved by dx metres along x (dx a whole number of voxels: every key moves by dx, every point stays in its voxel)"""
    keys, counts, pts = prior
    k = keys.copy()
    k[:, 0] += int(dx)
    p = pts.copy()
    p[:, 0] += dx
    ok = np.repeat(np.floor(p[:, 0]).astype(np.int64) == np.repeat(k[:, 0], counts), 1)
    per_voxel = np.add.reduceat(ok.astype(np.int64), np.r_[0, np.cumsum(counts)[:-1]]) == counts
    keep_pts = np.repeat(per_voxel, counts)
    return k[per_voxel], counts[per_voxel], p[keep_pts]


def _concat(a, b):
    return tuple(np.concatenate([x, y]) for x, y in zip(a, b))


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

    def frame(self, k):
        """frame k: (pose, preprocessed frame in the base frame, launches)"""
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
        return pose, np.asarray(out[1], dtype=np.float64), launches

    def close(self):
        self.gm.close()
        self.ctx.close()


_PRIOR = {}


def _golden_prior(kb, ko):
    """the map a full golden drive builds (the map a previous run saved), plus a copy of it FAR metres away along x"""
    if "p" not in _PRIOR:
        d = _Drive(kb, ko, _seq())
        try:
            for k in range(len(d.seq["frames"])):
                d.frame(k)
            built = d.gm.export_voxels()
        finally:
            d.close()
        _PRIOR["p"] = _concat(built, _shifted(built, FAR))
    return _PRIOR["p"]


def _world(seed, n=4000, half=30.0):
    rng = np.random.default_rng(seed)
    return np.round(np.c_[rng.uniform(-half, half, n), rng.uniform(-half, half, n), rng.uniform(-2, 3, n)] * 1024.0) / 1024.0 + 0.0


def test_thaw_is_a_map_never_frozen(oracle, gpu_ctx):
    """freeze then thaw, then the same calls as on a map that never froze: the same voxels, and the same bytes of every export"""
    import kinematic_icp_b200 as kb
    a, b = kb.VoxelHashMap(gpu_ctx, 1.0, 30.0, 20), kb.VoxelHashMap(gpu_ctx, 1.0, 30.0, 20)
    try:
        for m in (a, b):
            m.AddPoints(_world(1))
        a.freeze()
        a.thaw()
        assert a.num_prior_voxels() == 0 and a.num_prior_points() == 0
        for m in (a, b):
            m.Update(_world(3, 3000), np.array([0.0, 0.0, np.sin(0.1), np.cos(0.1), 12.0, -4.0, 0.0]))
            m.Update(_world(4, 3000), [40.0, 0.0, 0.0])
        assert _same(a.export_voxels(), b.export_voxels())
        assert a.num_points() == b.num_points() and a.num_voxels() == b.num_voxels()
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("device", [False, True])
def test_mutators_match_the_oracle(oracle, gpu_ctx, device):
    """AddPoints, RemovePointsFarFromLocation, Update(points, origin) and Update(points, pose), host and device clouds, on a frozen map:
    the oracle's map after every call, the prior prefix byte-identical, the prior's far voxels kept"""
    import kinematic_icp_b200 as kb
    torch = pytest.importorskip("torch") if device else None
    ko = oracle
    gm = kb.VoxelHashMap(gpu_ctx, 1.0, 30.0, 20)
    try:
        base = _world(10, 6000)
        far = _world(11, 2000, 5.0) + np.array([200.0, 0.0, 0.0])  # beyond max_distance from every origin below
        gm.AddPoints(np.concatenate([base, far]))
        gm.freeze()
        prior = gm.export_voxels()
        P = len(prior[1])
        assert gm.num_prior_voxels() == P and gm.num_prior_points() == len(prior[2])
        om = PriorMap(ko, prior, 1.0, 30.0, 20)

        def pts(x):
            return torch.from_numpy(np.ascontiguousarray(x)).cuda() if device else x

        pose = np.array([0.0, 0.0, np.sin(0.2), np.cos(0.2), 7.0, 3.0, 0.0])
        steps = [("add", _world(12, 3000, 40.0)), ("update_origin", (_world(13, 3000, 40.0), [20.0, 0.0, 0.0])),
                 ("update_pose", (_world(14, 3000, 40.0), pose)), ("remove_far", [-35.0, 0.0, 0.0]),
                 ("update_pose", (_world(15, 3000, 40.0), np.array([0.0, 0.0, 0.0, 1.0, -30.0, 0.0, 0.0])))]
        for name, arg in steps:
            if name == "add":
                gm.AddPoints(pts(arg))
                om.add_points(arg)
            elif name == "update_origin":
                gm.Update(pts(arg[0]), arg[1])
                om.update_origin(*arg)
            elif name == "update_pose":
                gm.Update(pts(arg[0]), arg[1])
                om.update_pose(*arg)
            else:
                gm.RemovePointsFarFromLocation(arg)
                om.remove_far(arg)
            got = gm.export_voxels()
            assert _same(got, om.export_voxels()), name
            assert _bytes(_prefix(got, P)) == _bytes(prior), name
            assert gm.num_points() == om.num_points() and gm.num_voxels() == om.num_voxels(), name
        assert om.live.num_voxels() > 0
    finally:
        gm.close()


@pytest.mark.parametrize("mode", [R.ALWAYS, R.GATED])
@pytest.mark.parametrize("frame_sync", [0, 1])
@pytest.mark.parametrize("staged", [False, True])
def test_drive_against_a_frozen_prior(oracle, mode, frame_sync, staged):
    """the golden drive against its own saved map plus a far copy, frozen, under ALWAYS or GATED: every pose is bit for bit the pose a
    context registers with the same union map re-loaded before the frame; after every frame the map is the oracle's (the prior, then
    the live layer fed the points outside the prior's voxels), the prior prefix is byte-identical and the far copy is still there; the
    outcome follows the rule; in the single-synchronisation order the frame launches the map's six kernels more than under NEVER.
    The exports of every frame (Pointcloud, export_voxels, the layers) come between two frames: the spare arrays' prior copy survives."""
    import kinematic_icp_b200 as kb
    ko = oracle
    seq = _seq()
    prior = _golden_prior(kb, ko)
    P = len(prior[1])
    a = _Drive(kb, ko, seq, staged=staged, frame_sync=frame_sync, correspondences=1)
    b = _Drive(kb, ko, seq, staged=staged, frame_sync=frame_sync, correspondences=1)
    try:
        a.gm.load_voxels(*prior)
        a.gm.freeze()
        gate = (R.GATED, 50, 0.3, 0.5)
        if mode == R.GATED:
            a.ctx.set_map_update(*gate[:1], min_inliers=gate[1], min_fitness=gate[2], max_inlier_rmse=gate[3])
        b.ctx.set_map_update(R.NEVER)
        om = PriorMap(ko, prior, 1.0, 100.0, 20)
        applied = 0
        for k in range(len(seq["frames"])):
            union = a.gm.export_voxels()
            b.gm.load_voxels(*union)
            pa, fa, la = a.frame(k)
            pb, fb, lb = b.frame(k)
            assert S.same_bits(pa, pb), k
            outcome = kb.frame_map_update(a.ctx)
            expect = R.rule_stats(gate if mode == R.GATED else (R.ALWAYS, 0, 0.0, np.inf), R.KICP_OK, False, kb.frame_correspondences(a.ctx))
            assert outcome == expect, (k, outcome, expect)
            if outcome == R.APPLIED:
                om.update_pose(ko.voxel_downsample(fa, 0.5), pa)
                applied += 1
            if frame_sync == 0:
                assert la == lb + MAP_LAUNCHES + (1 if mode == R.GATED else 0), (k, la, lb)
            got = a.gm.export_voxels()
            assert _same(got, om.export_voxels()), k
            assert _bytes(_prefix(got, P)) == _bytes(prior), k
            assert a.gm.num_prior_voxels() == P
            # the exports between two frames (the pitfall: the host packing must not use the spare arrays' prior copy as scratch)
            assert a.gm.Pointcloud().tobytes() == got[2].tobytes()
            assert a.gm.Pointcloud(layer="prior").tobytes() == prior[2].tobytes()
            a.gm.PointcloudF32(layer="live")
        assert applied > 0
        assert np.any(prior[2][:, 0] > FAR / 2) and om.live.num_voxels() > 0
    finally:
        a.close()
        b.close()


def test_growth_while_frozen(oracle, monkeypatch):
    """KICP_MAP_VOXELS at its minimum, a prior that fills most of it: the storage and the table grow during the frozen drive, and every
    pose and map equals the drive's on a roomy map"""
    import kinematic_icp_b200 as kb
    ko = oracle
    seq = _seq()
    prior = _golden_prior(kb, ko)
    n_first = len(seq["frames"][0])
    assert len(prior[1]) + n_first > 16384, "the drive must outgrow the small map"
    monkeypatch.setenv("KICP_MAP_VOXELS", "16384")
    small = _Drive(kb, ko, seq)
    monkeypatch.delenv("KICP_MAP_VOXELS")
    roomy = _Drive(kb, ko, seq)
    try:
        for d in (small, roomy):
            d.gm.load_voxels(*prior)
            d.gm.freeze()
        for k in range(len(seq["frames"])):
            ps, _, _ = small.frame(k)
            pr, _, _ = roomy.frame(k)
            assert S.same_bits(ps, pr), k
            vs, vr = small.gm.export_voxels(), roomy.gm.export_voxels()
            assert _same(vs, vr), k
            assert _bytes(_prefix(vs, len(prior[1]))) == _bytes(prior), k
    finally:
        small.close()
        roomy.close()


@pytest.mark.parametrize("f32", [False, True])
def test_layer_exports(oracle, gpu_ctx, f32):
    """ALL is PRIOR followed by LIVE, byte for byte, from the host calls and into device memory; ALL is the whole-map export"""
    import kinematic_icp_b200 as kb
    torch = pytest.importorskip("torch")
    gm = kb.VoxelHashMap(gpu_ctx, 1.0, 30.0, 20)
    try:
        gm.AddPoints(_world(20, 5000))
        gm.freeze()
        gm.Update(_world(21, 3000, 45.0), [10.0, 0.0, 0.0])
        get = gm.PointcloudF32 if f32 else gm.Pointcloud
        whole, al, pr, lv = get(), get(layer="all"), get(layer="prior"), get(layer="live")
        assert len(pr) == gm.num_prior_points() and len(lv) == gm.num_points() - gm.num_prior_points() > 0
        assert whole.tobytes() == al.tobytes() == np.concatenate([pr, lv]).tobytes()
        dt = torch.float32 if f32 else torch.float64
        for layer, ref in (("all", al), ("prior", pr), ("live", lv), (None, whole)):
            out = torch.full((len(ref) + 5, 3), -1.0, dtype=dt, device="cuda")
            n = gm.PointcloudInto(out, layer=layer)
            torch.cuda.synchronize()
            assert n == len(ref) and out[:n].cpu().numpy().tobytes() == ref.tobytes(), layer
        small = torch.zeros((1, 3), dtype=dt, device="cuda")
        with pytest.raises(kb.KicpError):
            gm.PointcloudInto(small, layer="live")
        with pytest.raises(kb.KicpError, match="layer"):
            gm.Pointcloud(layer=3)
    finally:
        gm.close()


def test_edges(oracle, gpu_ctx):
    """clear and load_voxels end the prior; a second freeze takes in the live voxels; a live layer that stays empty (every point in a
    prior voxel) leaves the map as it was; freezing an empty map freezes nothing"""
    import kinematic_icp_b200 as kb
    gm = kb.VoxelHashMap(gpu_ctx, 1.0, 30.0, 20)
    try:
        gm.freeze()
        assert gm.num_prior_voxels() == 0
        base = _world(30, 4000, 20.0)
        gm.AddPoints(base)
        gm.freeze()
        before = gm.export_voxels()
        gm.Update(base + 0.01, [0.0, 0.0, 0.0])  # every point falls in a prior voxel (or in none of the map's, at a voxel face)
        inside = PriorMap(oracle, before, 1.0, 30.0, 20).not_prior(base + 0.01)
        if len(inside) == 0:
            assert _bytes(gm.export_voxels()) == _bytes(before)
        assert len(gm.Pointcloud(layer="live")) == gm.num_points() - gm.num_prior_points()
        gm.Update(_world(31, 2000, 28.0), [0.0, 0.0, 0.0])
        nv = gm.num_voxels()
        assert nv > gm.num_prior_voxels()
        gm.freeze()
        assert gm.num_prior_voxels() == nv and len(gm.Pointcloud(layer="live")) == 0
        gm.Clear()
        assert gm.num_prior_voxels() == 0 and gm.num_prior_points() == 0
        gm.AddPoints(base)
        gm.freeze()
        gm.load_voxels(*before)
        assert gm.num_prior_voxels() == 0
        gm.Update(base, [100.0, 0.0, 0.0])  # not frozen any more: everything evicted
        assert gm.num_voxels() == 0
    finally:
        gm.close()


def test_replay_freeze_prior(oracle, tmp_path):
    """kicp_replay --load-map F --freeze-prior --map-update always: the poses of the Python frame path on the same frozen prior, the
    prior and live sizes at the end in its JSON line; --freeze-prior without --load-map is refused"""
    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    ko = oracle
    seq = _seq()
    n = len(seq["frames"])
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    prior = _golden_prior(kb, ko)
    from test_map_update_cpu import _hooks, write_map
    kseq, mp = str(tmp_path / "drive.kseq"), str(tmp_path / "prior.kmap")
    S2.write_kseq(seq, kseq, header_stamps=[100.0 + 0.1 * k for k in range(n)])
    write_map(_hooks(), mp, 1.0, 20, *prior)
    tum = str(tmp_path / "a.tum")
    out = subprocess.run([exe, kseq, tum, "--deskew", "1", "--load-map", mp, "--freeze-prior", "--map-update", "always"],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    info = json.loads(out.stdout.strip().splitlines()[-1])
    d = _Drive(kb, ko, seq)
    try:
        d.gm.load_voxels(*prior)
        d.gm.freeze()
        poses = [d.frame(k)[0] for k in range(n)]
        assert info["prior_voxels"] == d.gm.num_prior_voxels() == len(prior[1])
        assert info["prior_points"] == d.gm.num_prior_points() == len(prior[2])
        assert info["live_voxels"] == d.gm.num_voxels() - len(prior[1])
        assert info["live_points"] == d.gm.num_points() - len(prior[2])
    finally:
        d.close()
    assert info["map_update_outcomes"]["applied"] == n
    got = np.loadtxt(tum, ndmin=2)
    assert got.shape == (n, 8)
    for row, p in zip(got, poses):
        dt, ang = ko.pose_delta(np.r_[row[4:8], row[1:4]], p)
        assert dt <= 2e-6 and ang <= 1e-5, (dt, ang)
    bad = subprocess.run([exe, kseq, str(tmp_path / "x.tum"), "--freeze-prior"], capture_output=True, text=True, timeout=300)
    assert bad.returncode == 2 and "--load-map" in bad.stderr


def test_facade_agrees_with_the_c_calls(oracle):
    """kiss_icp::VoxelHashMap::Freeze / Thaw / PriorVoxels / PriorPoints / Pointcloud(layer) against the C calls on a map of the same
    context fed the same points"""
    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import _capi
    H = C.CDLL(os.path.join(ROOT, "tests", "hooks", "_build", "libkicp_prior_map_hooks.so"))
    H.kpm_create.restype = C.c_void_p
    H.kpm_create.argtypes = [C.c_double, C.c_double, C.c_uint32]
    for f in (H.kpm_destroy, H.kpm_freeze, H.kpm_thaw, H.kpm_clear):
        f.argtypes = [C.c_void_p]
    H.kpm_handle.restype = C.c_void_p
    H.kpm_handle.argtypes = [C.c_void_p]
    for f in (H.kpm_prior_voxels, H.kpm_prior_points):
        f.restype, f.argtypes = C.c_int64, [C.c_void_p]
    H.kpm_update_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    H.kpm_pointcloud.restype = C.c_int64
    H.kpm_pointcloud.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_char_p, C.c_int64]
    L = _capi.lib()
    fm = C.c_void_p(H.kpm_create(1.0, 30.0, 20))
    h = C.c_void_p(H.kpm_handle(fm))
    try:
        base = _world(40, 4000, 20.0)
        L.kicp_map_add_points(h, base.ctypes.data_as(_capi.c_dp), len(base))
        H.kpm_freeze(fm)
        v, p = C.c_int64(), C.c_int64()
        assert L.kicp_map_prior_size(h, C.byref(v), C.byref(p)) == 0
        assert H.kpm_prior_voxels(fm) == v.value > 0 and H.kpm_prior_points(fm) == p.value > 0
        fr = _world(41, 2000, 40.0)
        pose = np.array([0.0, 0.0, np.sin(0.1), np.cos(0.1), 3.0, 1.0, 0.0])
        H.kpm_update_pose(fm, fr.ctypes.data, len(fr), pose.ctypes.data)
        err = C.create_string_buffer(256)
        for layer in (0, 1, 2):
            nm = C.c_int64()
            total = C.c_int64()
            L.kicp_map_num_points(h, C.byref(total))
            out_c = np.zeros((max(total.value, 1), 3))
            assert L.kicp_map_pointcloud_layer(h, layer, 0, out_c.ctypes.data, total.value, C.byref(nm)) == 0
            out_f = np.zeros((max(total.value, 1), 3))
            assert H.kpm_pointcloud(fm, layer, out_f.ctypes.data, total.value, err, 256) == nm.value
            assert out_f[:nm.value].tobytes() == out_c[:nm.value].tobytes(), layer
        assert H.kpm_pointcloud(fm, 7, None, 0, err, 256) == -1 and b"layer" in err.value
        H.kpm_thaw(fm)
        assert H.kpm_prior_voxels(fm) == 0 and H.kpm_prior_points(fm) == 0
        H.kpm_freeze(fm)
        H.kpm_clear(fm)
        assert H.kpm_prior_voxels(fm) == 0
    finally:
        H.kpm_destroy(fm)
