"""The correspondence report on the GPU: kicp_map_correspondences and its device variant against the oracle's composition
(tests/corr_oracle.py), and option "correspondences" of the frame calls on the golden drive, a staged LaserScan, a two-sensor frame and
a segments frame: every frame's pose, clouds and map bit for bit those with the option off, its statistics the oracle's evaluation of
the frame's source at the returned pose against the map before the frame's Update, two more launches per frame with the option on and
none with it off."""
import os

import numpy as np
import pytest

import laser_projection as LP
import scenes as S
from corr_oracle import check_stats, oracle_corr
from test_gpu_parity import sorted_voxels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
IDENT = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def _oracle_map(ko, voxels, vs=1.0, cap=20, max_distance=100.0):
    """an oracle map holding exactly the exported voxels (each voxel's points re-added in its insertion order)"""
    om = ko.OracleMap(vs, max_distance, cap)
    if len(voxels[2]):
        om.add_points(voxels[2])
    return om


def _check_points(got, want):
    pts, dist, inl = (np.asarray(a) for a in got)
    po, do, io = want
    assert S.same_bits(dist, do) and S.same_bits(pts, po)
    assert np.array_equal(inl.astype(bool), io) and set(np.unique(inl)) <= {0, 1}


def test_standalone_host_and_device(oracle, workload):
    """cfg2's map: its scan at the prior (host, device float64, device float32 records) and far points; an empty map."""
    import torch

    import kinematic_icp_b200 as kb
    ko = oracle
    w = workload(2)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    try:
        gm.load_voxels(*w.map.export_voxels())
        rng = np.random.default_rng(2)
        src = np.concatenate([w.scan, rng.uniform(-150, 150, (500, 3))])
        po, do, io, want = oracle_corr(ko, w.map, src, w.prior, w.tau)
        assert 0 < want["n_inliers"] < len(src)
        *pts, st = gm.Correspondences(src, w.prior, w.tau)
        _check_points(pts, (po, do, io))
        check_stats(st_c(st), want)
        *pts, st2 = gm.Correspondences(torch.from_numpy(src).cuda(), w.prior, w.tau)
        _check_points([t.cpu().numpy() for t in pts], (po, do, io))
        assert st2 == st  # same inputs, same bits
        f32 = src.astype(np.float32)
        po, do, io, want = oracle_corr(ko, w.map, f32.astype(np.float64), w.prior, w.tau)
        rec = np.zeros((len(f32), 4), np.float32)
        rec[:, :3] = f32
        dev = torch.from_numpy(rec.view(np.uint8).reshape(-1)).cuda()
        *pts, st = gm.Correspondences(dev, w.prior, w.tau, point_step=16, offsets=(0, 4, 8),
                                      out=(torch.empty((len(f32), 3), dtype=torch.float64, device="cuda"),
                                           torch.empty(len(f32), dtype=torch.float64, device="cuda"),
                                           torch.empty(len(f32), dtype=torch.uint8, device="cuda")))
        _check_points([t.cpu().numpy() for t in pts], (po, do, io))
        check_stats(st_c(st), want)
        gm.Clear()
        *pts, st = gm.Correspondences(src, w.prior, w.tau)
        assert (pts[1] == np.finfo(np.float64).max).all() and st.n_inliers == 0 and st.fitness == 0.0 and st.n_points == len(src)
    finally:
        gm.close()
        ctx.close()


def st_c(st):
    """a CorrespondenceStats as the ctypes mirror check_stats takes"""
    from corr_oracle import CorrStats
    c = CorrStats()
    c.n_points, c.n_inliers, c.fitness, c.inlier_rmse, c.sum_sq = st.n_points, st.n_inliers, st.fitness, st.inlier_rmse, st.sum_sq
    c.jtj[:], c.jtr[:] = list(st.jtj), list(st.jtr)
    return c


def _frame_report(kb, ctx):
    import torch
    pts, dist, inl = (torch.as_tensor(a, device="cuda").cpu().numpy() for a in kb.frame_correspondences_device(ctx))
    return pts, dist, inl, st_c(kb.frame_correspondences(ctx))


class _Twin:
    """two contexts and maps driven with the same frames: option "correspondences" off and on"""

    def __init__(self, kb, frame_sync=0):
        self.kb = kb
        self.ctx = [kb.Context(0), kb.Context(0)]
        for c, on in zip(self.ctx, (0, 1)):
            c.set_option("frame_sync", frame_sync)
            c.set_option("correspondences", on)
        self.gm = [kb.VoxelHashMap(c, 1.0, 100.0, 20) for c in self.ctx]

    def frame(self, ko, run, tau):
        """run(ctx, gm) -> (pose, frame, source, result) on both; asserts everything equal and the report the oracle's; returns
        (pose, the on-side report's statistics)"""
        before = self.gm[1].export_voxels()
        outs, launches = [], []
        for c, g in zip(self.ctx, self.gm):
            l0 = c.launch_count
            outs.append(run(c, g))
            launches.append(c.launch_count - l0)
        assert launches[1] == launches[0] + 2, launches
        (p0, f0, s0, r0), (p1, f1, s1, r1) = outs
        assert S.same_bits(p0, p1) and S.same_bits(f0, f1) and S.same_bits(s0, s1) and bytes(r0) == bytes(r1)
        off = self.kb.frame_correspondences(self.ctx[0])
        assert off.n_points == 0 and off.n_inliers == 0 and len(self.kb.frame_correspondences_device(self.ctx[0])[0]) == 0
        pts, dist, inl, st = _frame_report(self.kb, self.ctx[1])
        po, do, io, want = oracle_corr(ko, _oracle_map(ko, before), s1, p1, tau)
        _check_points((pts, dist, inl), (po, do, io))
        check_stats(st, want)
        return p1, want

    def same_maps(self):
        """the same voxels with the same points in the same per-voxel order (the block order follows the device's atomics)"""
        a, b = (sorted_voxels(*g.export_voxels()) for g in self.gm)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))

    def close(self):
        for g in self.gm:
            g.close()
        for c in self.ctx:
            c.close()


@pytest.mark.parametrize("frame_sync", [0, 1])
@pytest.mark.parametrize("staged", [False, True])
def test_golden_drive(oracle, frame_sync, staged):
    """tests/golden/pipeline_seq.npz with de-skew, through RegisterFrame or StageFrame + RegisterStagedFrame, in both synchronisation
    orders: the first frame has no inliers (empty map), every later one has some."""
    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    ko = oracle
    seq = S2.unpack_sequence(np.load(os.path.join(GOLDEN, "pipeline_seq.npz")), True)
    tw = _Twin(kb, frame_sync)
    threshold = ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
    l2b = seq["lidar_to_base"]
    last = np.array(seq["start"], dtype=np.float64)
    kw = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
    try:
        fits = []
        for frame, stamps, odom in zip(seq["frames"], seq["stamps"], seq["odoms"]):
            motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
            tau = threshold.compute()

            def run(c, g):
                if staged:
                    return kb.RegisterStagedFrame(g, kb.StageFrame(c, frame, timestamps=stamps), motion, l2b, last, odom, tau, **kw)
                return kb.RegisterFrame(g, frame, stamps, motion, l2b, last, odom, tau, **kw)

            pose, want = tw.frame(ko, run, tau)
            fits.append(want["n_inliers"] / max(want["n_points"], 1))
            threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(last, odom)), pose))
            last = pose
        assert fits[0] == 0.0 and min(fits[1:]) > 0.0, fits
        tw.same_maps()
    finally:
        tw.close()


def test_laser_scan_two_sensor_and_segments_frames(oracle):
    """On a map built by two 3D frames: a staged 2D LaserScan frame, a frame of two sensors and a segments frame, each with the option
    on and off."""
    import kinematic_icp_b200 as kb
    ko = oracle
    rng = np.random.default_rng(11)
    tw = _Twin(kb)
    kw = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
    world = np.c_[rng.uniform(-20, 20, 30000), rng.uniform(-20, 20, 30000), rng.uniform(-1, 3, 30000)]
    world = np.round(world * 4096.0) / 4096.0 + 0.0
    l2b = IDENT.copy()
    last = IDENT.copy()
    odom = np.array([0.0, 0.0, np.sin(0.002), np.cos(0.002), 0.02, 0.0, 0.0])
    try:
        for k in range(2):
            stamps = np.linspace(0.0, 0.1, len(world))
            pose, _ = tw.frame(ko, lambda c, g: kb.RegisterFrame(g, world, stamps, odom, l2b, last, odom, 1.0, **kw), 1.0)
            last = pose
        ranges = rng.uniform(0.5, 25.0, 1081).astype(np.float32)
        pose, _ = tw.frame(ko, lambda c, g: kb.RegisterStagedFrame(g, kb.StageLaserScan(c, ranges, **LP.SCAN), odom, l2b, last, odom, 1.0,
                                                                   **kw), 1.0)
        last = pose
        halves = [world[::2], world[1::2]]
        t = [1.7e9 + np.linspace(0.0, 0.1, len(h)) for h in halves]
        l2bs = [IDENT, np.array([0.0, 0.0, 0.0, 1.0, 0.1, 0.0, 0.0])]

        def two(c, g):
            st = kb.StageSensors(c, [kb.PointCloudSensor(h, timestamps=s, time_offset=0.002 * i) for i, (h, s) in enumerate(zip(halves, t))])
            motions = [ko.se3_compose(ko.se3_compose(ko.se3_inverse(l), odom), l) for l in l2bs]
            return kb.RegisterStagedSensors(g, st, motions, l2bs, last, odom, 1.0, **kw)

        pose, _ = tw.frame(ko, two, 1.0)
        last = pose

        def segments(c, g):
            st = kb.StageFrame(c, world, timestamps=1.7e9 + np.linspace(0.0, 0.1, len(world)))
            w0, w1 = st.stamp_range
            mid = 0.5 * (w0 + w1)
            half = ko.se3_exp(0.5 * ko.se3_log(odom))
            table = np.array([np.concatenate([[w0, mid], half, half]), np.concatenate([[mid, w1], half, IDENT])])
            return kb.RegisterStagedFrameSegments(g, st, table, l2b, last, odom, 1.0, **kw)

        pose, want = tw.frame(ko, segments, 1.0)
        assert want["n_inliers"] > 0
        tw.same_maps()
    finally:
        tw.close()


def test_option_values(oracle):
    import kinematic_icp_b200 as kb
    from kinematic_icp_b200 import KicpError
    ctx = kb.Context(0)
    try:
        for v in (-1, 2):
            with pytest.raises(KicpError):
                ctx.set_option("correspondences", v)
        ctx.set_option("correspondences", 1)
        ctx.set_option("correspondences", 0)
    finally:
        ctx.close()


def _drive_python(kb, ko, seq):
    """the golden drive through RegisterFrame with option "correspondences" 1, the threshold as the C++ facade keeps it: per frame the
    statistics (frame_correspondences) and the pose"""
    ctx = kb.Context(0)
    ctx.set_option("correspondences", 1)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    threshold = ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
    l2b = seq["lidar_to_base"]
    last = np.array(seq["start"], dtype=np.float64)
    stats, poses = [], []
    try:
        for frame, stamps, odom in zip(seq["frames"], seq["stamps"], seq["odoms"]):
            motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
            pose, _, _, _ = kb.RegisterFrame(gm, frame, stamps, motion, l2b, last, odom, threshold.compute(), max_range=100.0,
                                             min_range=0.0, deskew=True, voxel_size=1.0, want_clouds=False)
            threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(last, odom)), pose))
            last = pose
            stats.append(kb.frame_correspondences(ctx)), poses.append(pose)
    finally:
        gm.close()
        ctx.close()
    return stats, poses


def test_replay_writes_one_line_per_frame(oracle, tmp_path):
    """kicp_replay --correspondences on the golden drive (the C++ facade's KinematicICP::LastCorrespondenceStats after every frame):
    one CSV line per frame with the TUM file's stamp, and the values frame_correspondences gives for the same drive through the Python
    binding of kicp_frame_correspondences (counts exactly, the doubles to 1e-9: the two drives' thresholds are computed by two
    restatements of CorrespondenceThreshold)."""
    import subprocess

    import kinematic_icp_b200 as kb
    from oracle import sequences as S2
    ko = oracle
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    seq = S2.unpack_sequence(np.load(os.path.join(GOLDEN, "pipeline_seq.npz")), True)
    header = [100.0 + 0.1 * k for k in range(len(seq["frames"]))]
    kseq, tum, csv = str(tmp_path / "drive.kseq"), str(tmp_path / "out.tum"), str(tmp_path / "corr.csv")
    S2.write_kseq(seq, kseq, header_stamps=header)
    out = subprocess.run([exe, kseq, tum, "--deskew", "1", "--correspondences", csv], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    got = np.loadtxt(csv, delimiter=",", ndmin=2)
    assert got.shape == (len(seq["frames"]), 10)
    assert np.allclose(got[:, 0], header, rtol=0, atol=1e-9)  # the header stamps, as the TUM lines of a version-1 drive
    stats, poses = _drive_python(kb, ko, seq)
    for k, (row, st) in enumerate(zip(got, stats)):
        assert row[1] == st.n_points and row[2] == st.n_inliers, (k, row, st)
        want = np.array([st.fitness, st.inlier_rmse, *st.jtj, *st.jtr])
        assert np.allclose(row[3:], want, rtol=1e-9, atol=1e-9 * np.abs(want).max()), (k, row, want)
    assert got[0, 2] == 0 and (got[1:, 2] > 0).all()
    # without the flag no file and the same trajectory
    tum2 = str(tmp_path / "off.tum")
    out = subprocess.run([exe, kseq, tum2, "--deskew", "1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert open(tum2).read() == open(tum).read()


FACADE_PROGRAM = r"""
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "kinematic_icp/pipeline/KinematicICP.hpp"
#include "kicp/runtime.hpp"
int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    try {
        if (mode == "set") kinematic_icp::pipeline::KinematicICP::SetCorrespondences(true);
        kinematic_icp::pipeline::Config config;
        config.deskew = false;
        kinematic_icp::pipeline::KinematicICP pipeline(config);
        for (int f = 0; f < 3; ++f) {
            std::vector<Eigen::Vector3d> frame;
            for (int i = 0; i < 60; ++i)
                for (int j = 0; j < 60; ++j)
                    for (int k = 0; k < 4; ++k) frame.emplace_back(-15.0 + 0.5 * i + 0.01 * f, -15.0 + 0.5 * j, -1.0 + 1.3 * k + 0.1 * ((i * j) % 5));
            const auto [pre, source] = pipeline.RegisterFrame(frame, {}, Sophus::SE3d(), Sophus::SE3d());
            const kicp_corr_stats st = pipeline.LastCorrespondenceStats();
            kicp_corr_stats c{};
            kicp_frame_correspondences(kicp::default_context(), &c);
            std::printf("%zu %lld %lld %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d\n", source.size(), (long long)st.n_points,
                        (long long)st.n_inliers, st.fitness, st.inlier_rmse, st.sum_sq, st.jtj[0], st.jtj[1], st.jtj[2], st.jtr[0], st.jtr[1],
                        std::memcmp(&st, &c, sizeof(st)) == 0 ? 1 : 0);
        }
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 3;
    }
    return 0;
}
"""


def test_facade_stats_and_switches(tmp_path):
    """A C++ facade program: KinematicICP::LastCorrespondenceStats equals kicp_frame_correspondences of the process-wide context after
    every frame; KICP_CORRESPONDENCES=1 and SetCorrespondences(true) switch the report on alike (the same stats, the first frame
    without inliers, the later ones with), no switch or KICP_CORRESPONDENCES=0 leave it off (all zero), any other value throws."""
    import subprocess
    cpp = os.path.join(ROOT, "kinematic-icp_b200", "cpp")
    lib = os.path.join(ROOT, "kinematic-icp_b200", "lib")
    src, exe = tmp_path / "facade_corr.cpp", tmp_path / "facade_corr"
    src.write_text(FACADE_PROGRAM)
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", cpp, "-I", os.path.join(cpp, "compat"), "-I", os.path.join(ROOT, "include"), str(src),
                    "-o", str(exe), "-L", lib, "-lkinematic_icp_b200", "-lkicp_b200", "-Wl,-rpath," + lib], check=True)

    def run(mode, env_value):
        env = {k: v for k, v in os.environ.items() if k != "KICP_CORRESPONDENCES"}
        if env_value is not None:
            env["KICP_CORRESPONDENCES"] = env_value
        return subprocess.run([str(exe), mode], capture_output=True, text=True, env=env, timeout=120)

    outs = {}
    for name, mode, value in [("env", "", "1"), ("set", "set", None), ("off", "", None), ("zero", "", "0")]:
        r = run(mode, value)
        assert r.returncode == 0, (name, r.stderr)
        outs[name] = np.array([[float(x) for x in l.split()] for l in r.stdout.splitlines()])
        assert outs[name].shape == (3, 12) and (outs[name][:, -1] == 1).all(), name  # the facade's stats are the C entry point's
    assert np.array_equal(outs["env"], outs["set"])
    on = outs["env"]
    assert (on[:, 1] == on[:, 0]).all()  # n_points: the registration source RegisterFrame returned
    assert on[0, 2] == 0 and (on[1:, 2] > 0).all() and (on[1:, 3] > 0.5).all()
    for name in ("off", "zero"):
        assert not outs[name][:, 1:11].any(), name
    assert run("", "2").returncode == 3
