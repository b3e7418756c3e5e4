"""kicp_replay on version-3 .kseq drives (tests/kseq3.py): a one-slot drive is bit for bit the version-2 replay of the same records, a
LaserScan slot is the replay of projectLaser's records and reproduces the 2D golden drive, multi-slot drives and drives with odometry
samples are the facade run frame by frame (tests/hooks/sensor_hooks.cpp, segment_hooks.cpp) and follow the oracle compositions, a frame
whose samples miss its sweep is refused, and the publication modes agree.  Every replay is one kicp_replay process."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import deskew_segments_oracle as DO
import kseq2
import kseq3 as K
import laser_projection as LP
import multi_sensor_oracle as MO
from test_gpu_deskew_segments import register_preprocessed, segment_hooks
from test_gpu_multi_sensor import MAX_RANGE, TOL_R, TOL_T, sensor_hooks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
START = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
# the keys of a KSEQ1 / KSEQ2 line (bench.py parses them); a KSEQ3 line adds the slots
KEYS = {"harness", "frames", "points_per_frame", "seconds", "frames_per_s", "ms_per_frame", "frames_per_s_best", "repetition_seconds",
        "host_buffers", "deskew", "publish", "map_points", "tum_file"}
KEYS3 = KEYS | {"slots", "slot_kinds", "odometry_samples_per_frame"}


def replay(kseq, tum, *extra, ok=True):
    """(TUM text, JSON line) of one kicp_replay run; with ok False the finished process"""
    r = subprocess.run([EXE, str(kseq), str(tum)] + [str(x) for x in extra], capture_output=True, text=True, timeout=600)
    if not ok:
        return r
    assert r.returncode == 0, r.stderr
    return open(tum).read(), json.loads(r.stdout.strip().splitlines()[-1])


def pose_columns(text):
    return [line.split(" ", 1)[1] for line in text.splitlines()]


def tum_text(stamps, poses7):
    """what kicp::write_poses_tum writes for these poses ({qx, qy, qz, qw, tx, ty, tz})"""
    return "".join("%.6f %.6f %.6f %.6f %.6f %.6f %.6f %.6f\n" % (t, p[4], p[5], p[6], p[0], p[1], p[2], p[3]) for t, p in zip(stamps, poses7))


def tum_poses(text):
    """the TUM file's poses as pose7"""
    v = np.array([[float(x) for x in line.split()] for line in text.splitlines()])
    return v[:, 0], np.column_stack([v[:, 4:8], v[:, 1:4]])


def kseq2_frames(slots, frames, project=False):
    """a one-slot drive as version-2 frames (a LaserScan slot as projectLaser's records)"""
    out = []
    for fr in frames:
        m = fr["messages"][0]
        m = K.projected_message(m) if project else m
        out.append((m["records"], m["point_step"], m["offsets"], m["stamp_datatype"], m["stamp_offset"], m["header"], fr["odom"]))
    return out


# ------------------------------------------------------------------------------------------------ the facade frame by frame
def facade_drive(ko, slots, frames):
    """the drive through KinematicICP::StageSensors and RegisterStagedSensors (with the frame's samples, when it has them), as the
    test hooks run them: per frame (sweep, window-free pose7)"""
    Hf, Hs = sensor_hooks(), segment_hooks()
    pipe = ko.facade_pipeline(deskew=True)
    k = len(slots)
    l2bs = np.ascontiguousarray([s[2] for s in slots], dtype=np.float64)
    last = np.array([min(m["header"] for m in frames[0]["messages"])])
    out = []
    try:
        for fr in frames:
            keep, data, n = [], [], np.zeros(k, np.int64)
            step, xyz, t_type, t_off = np.zeros(k, np.uint32), np.zeros(3 * k, np.uint32), np.zeros(k, np.uint8), np.zeros(k, np.uint32)
            laser6, header, offset = np.zeros((k, 6), np.float32), np.zeros(k), np.zeros(k)
            kind = np.array([s[0] for s in slots], np.int32)
            for i, (s, m) in enumerate(zip(slots, fr["messages"])):
                header[i], offset[i] = m["header"], K.offset(s, m)
                if s[0] == K.LASER_SCAN:
                    buf = np.ascontiguousarray(m["ranges"], np.float32)
                    n[i], laser6[i] = len(buf), [m[q] for q in K.SCAN_KEYS]
                else:
                    buf = np.ascontiguousarray(m["records"], np.uint8)
                    n[i], step[i], xyz[3 * i:3 * i + 3] = len(buf) // m["point_step"], m["point_step"], m["offsets"]
                    t_type[i], t_off[i] = m["stamp_datatype"], m["stamp_offset"]
                keep.append(buf)
                data.append(buf.ctypes.data if len(buf) else None)
            ptrs = (C.c_void_p * k)(*data)
            be = np.zeros(2)
            assert Hf.kfac_pipeline_stage_sensors(pipe.h, k, kind.ctypes.data, ptrs, n.ctypes.data, step.ctypes.data, xyz.ctypes.data,
                                                  t_type.ctypes.data, t_off.ctypes.data, laser6.ctypes.data, header.ctypes.data,
                                                  offset.ctypes.data, np.zeros(k, np.int32).ctypes.data, last.ctypes.data, be.ctypes.data) == 0
            cap = max(int(n.sum()), 1)
            pose, buf_f, buf_s, nf = np.zeros(7), np.zeros((cap, 3)), np.zeros((cap, 3)), np.zeros(1, np.int64)
            odom = np.ascontiguousarray(fr["odom"], np.float64)
            if fr["samples"]:
                st = np.ascontiguousarray([s[0] for s in fr["samples"]], np.float64)
                sp = np.ascontiguousarray([s[1] for s in fr["samples"]], np.float64)
                ns = Hs.kseg_pipeline_register_samples(pipe.h, 1, k, l2bs.ctypes.data, odom.ctypes.data, len(st), st.ctypes.data, sp.ctypes.data,
                                                       pose.ctypes.data, buf_f.ctypes.data, buf_s.ctypes.data, cap, nf.ctypes.data)
            else:
                ns = Hf.kfac_pipeline_register_staged_sensors(pipe.h, k, l2bs.ctypes.data, odom.ctypes.data, 0, pose.ctypes.data,
                                                              buf_f.ctypes.data, buf_s.ctypes.data, cap, nf.ctypes.data)
            assert ns >= 0
            out.append((be.copy(), pose))
    finally:
        pipe.close()
    return out


def oracle_sensors(slots, messages):
    """the messages as multi_sensor_oracle takes them: points, stamps on their own clock, offset"""
    out = []
    for s, m in zip(slots, messages):
        if s[0] == K.LASER_SCAN:
            proj = LP.LaserProjector().project(m["ranges"], **{q: m[q] for q in K.SCAN_KEYS})
            pts = proj["points"]
        else:
            pts = K.records_points(m)
        st = K.message_stamps(s[0], m)
        out.append(dict(points=pts, stamps=st if len(st) else None, offset=K.offset(s, m)))
    return out


# ------------------------------------------------------------------------------------------------------------ 1. one records slot
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("deskew", [0, 1])
def test_one_records_slot_is_the_kseq2_replay(oracle, tmp_path, device, deskew):
    """pose columns byte-identical to the version-2 replay of the same records; the stamp column is the end of each sweep"""
    ko = oracle
    slots, frames, _ = K.sensors_drive(ko, 8, ["rel"], 3, world="3d")
    K.write_kseq3(str(tmp_path / "d3.kseq"), START, slots, frames)
    kseq2.write_kseq2(str(tmp_path / "d2.kseq"), slots[0][2], START, kseq2_frames(slots, frames))
    extra = ["--deskew", deskew] + (["--device-input"] if device else [])
    t3, j3 = replay(tmp_path / "d3.kseq", tmp_path / "d3.tum", *extra)
    t2, j2 = replay(tmp_path / "d2.kseq", tmp_path / "d2.tum", *extra)
    assert len(t3.splitlines()) == len(frames) and pose_columns(t3) == pose_columns(t2)
    assert [line.split()[0] for line in t3.splitlines()] == ["%.6f" % e for _, e in K.sweeps(slots, frames)]
    assert [line.split()[0] for line in t2.splitlines()] == ["%.6f" % fr["messages"][0]["header"] for fr in frames]
    assert set(j2) == KEYS and set(j3) == KEYS3 and j3["slots"] == 1 and j3["slot_kinds"] == ["records"]
    assert j3["odometry_samples_per_frame"] == 0 and j3["points_per_frame"] == j2["points_per_frame"]
    assert j3["map_points"] == j2["map_points"] and j3["host_buffers"] == j2["host_buffers"]


# ------------------------------------------------------------------------------------------------------------ 2. one LaserScan slot
def test_one_laser_scan_slot_is_the_projected_replay(oracle, tmp_path):
    """pose columns byte-identical to the version-2 replay of projectLaser's records, staged and from device memory"""
    l2b, scans = LP.drive_2d(frames=12)
    slots = [(K.LASER_SCAN, 0, l2b)]
    frames = [dict(odom=odom, samples=[], messages=[K.scan_message(r, header, **kw)]) for r, kw, header, odom in scans]
    K.write_kseq3(str(tmp_path / "d3.kseq"), START, slots, frames)
    kseq2.write_kseq2(str(tmp_path / "d2.kseq"), l2b, START, kseq2_frames(slots, frames, project=True))
    t2, j2 = replay(tmp_path / "d2.kseq", tmp_path / "d2.tum")
    for extra in ([], ["--device-input"]):
        t3, j3 = replay(tmp_path / "d3.kseq", tmp_path / "d3.tum", *extra)
        assert pose_columns(t3) == pose_columns(t2) and j3["map_points"] == j2["map_points"]
        assert j3["slot_kinds"] == ["laser_scan"] and j3["points_per_frame"] == j2["points_per_frame"]


@pytest.mark.parametrize("deskew", [False, True])
def test_golden_2d_drive_from_laser_scans(oracle, tmp_path, deskew):
    """tests/golden/pipeline_2d.npz (the reference's KinematicICP fed projectLaser's clouds) replayed from its LaserScans: the poses
    within test_gpu_laserscan's 1e-6 m / 1e-7 rad plus the TUM file's rounding (half a unit of the sixth decimal per value), and the
    final map size"""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden_2d as G
    ko = oracle
    z = np.load(os.path.join(ROOT, "tests", "golden", "pipeline_2d.npz"))
    l2b, start, scans = G.unpack(z)
    frames = [dict(odom=odom, samples=[], messages=[K.scan_message(r, header, **kw)]) for r, kw, header, odom in scans]
    K.write_kseq3(str(tmp_path / "g.kseq"), start, [(K.LASER_SCAN, 0, l2b)], frames)
    text, j = replay(tmp_path / "g.kseq", tmp_path / "g.tum", "--deskew", int(deskew))
    tag = "deskew" if deskew else "plain"
    _, poses = tum_poses(text)
    rounding_t, rounding_r = np.sqrt(3) * 5e-7, 4 * np.sqrt(3) * 5e-7  # a unit quaternion off by 5e-7 per component turns by <= 4 * that
    for k, p in enumerate(poses):
        dt, ang = ko.pose_delta(p, z[tag + "_poses"][k])
        assert dt <= 1e-6 + rounding_t and ang <= 1e-7 + rounding_r, (k, dt, ang)
    assert j["map_points"] == z[tag + "_n_map"][-1]


# ------------------------------------------------------------------------------------------------------------ 3. several slots
LAYOUTS = [(["rel", "scan"], None), (["abs", "scan", "scan"], (2, 1)), (["rel", "abs", "scan"], (4, 0))]


@pytest.mark.parametrize("layout,empty", LAYOUTS)
def test_several_slots_are_the_facade_and_the_oracle(oracle, tmp_path, layout, empty):
    """2 and 3 slots (records with absolute and relative stamps, LaserScans, one empty message): the TUM file is the facade's
    StageSensors + RegisterStagedSensors run frame by frame, whose poses follow multi_sensor_oracle's composition"""
    ko = oracle
    slots, frames, _ = K.sensors_drive(ko, 8, layout, 20 + len(layout), empty=empty)
    K.write_kseq3(str(tmp_path / "d.kseq"), START, slots, frames)
    text, j = replay(tmp_path / "d.kseq", tmp_path / "d.tum")
    got = facade_drive(ko, slots, frames)
    assert [tuple(be) for be, _ in got] == K.sweeps(slots, frames)
    assert text == tum_text([be[1] for be, _ in got], [p for _, p in got])
    assert j["slots"] == len(layout) and j["slot_kinds"] == ["laser_scan" if x == "scan" else "records" for x in layout]
    comp = MO.Pipeline(ko, deskew=True)
    l2bs = [s[2] for s in slots]
    for f, (fr, (_, pose)) in enumerate(zip(frames, got)):
        p_ref, _, _ = comp.register_frame(oracle_sensors(slots, fr["messages"]), l2bs, fr["odom"])
        dt, ang = ko.pose_delta(pose, p_ref)
        assert dt <= TOL_T and ang <= TOL_R, (f, dt, ang)
    assert j["map_points"] == comp.num_map_points()


# ------------------------------------------------------------------------------------------------------------ 4. samples
@pytest.mark.parametrize("layout", [["rel"], ["rel", "scan"]])
def test_two_samples_are_the_one_motion_replay(oracle, tmp_path, layout):
    """samples {(begin, identity), (end, relative_odometry)} on every frame: the TUM file of the drive without samples, byte for byte"""
    ko = oracle
    slots, frames, _ = K.sensors_drive(ko, 8, layout, 30)
    two = [dict(fr, samples=[(b, START), (e, fr["odom"])]) for fr, (b, e) in zip(frames, K.sweeps(slots, frames))]
    K.write_kseq3(str(tmp_path / "a.kseq"), START, slots, frames)
    K.write_kseq3(str(tmp_path / "b.kseq"), START, slots, two)
    ta, _ = replay(tmp_path / "a.kseq", tmp_path / "a.tum")
    tb, jb = replay(tmp_path / "b.kseq", tmp_path / "b.tum")
    assert ta == tb and jb["odometry_samples_per_frame"] == 2


def turning_drive(ko):
    """two 3D records slots with relative stamps over a path that turns and brakes inside its sweeps, odometry every 10 ms"""
    slots, frames, traj = K.sensors_drive(ko, 10, ["rel", "rel"], 40, world="3d")
    t_s, P, _ = traj
    out = []
    for fr, (b, e) in zip(K.with_samples(ko, traj, slots, frames, 0), K.sweeps(slots, frames)):
        sel = np.nonzero((t_s > b - 0.01) & (t_s < e + 0.01))[0]
        out.append(dict(fr, samples=[(float(t_s[i]), P[i]) for i in sel]))
    return slots, out, traj


def test_samples_follow_the_facade_and_the_oracle(oracle, tmp_path):
    """several samples per frame: the TUM file is the facade's RegisterStagedSensors with samples run frame by frame, its poses follow
    deskew_segments_oracle's composition, and they are not the one-motion replay's"""
    from test_deskew_segments_emu_cpu import compose
    ko = oracle
    slots, frames, _ = turning_drive(ko)
    assert all(len(fr["samples"]) >= 11 for fr in frames)
    K.write_kseq3(str(tmp_path / "s.kseq"), START, slots, frames)
    K.write_kseq3(str(tmp_path / "m.kseq"), START, slots, [dict(fr, samples=[]) for fr in frames])
    text, j = replay(tmp_path / "s.kseq", tmp_path / "s.tum")
    got = facade_drive(ko, slots, frames)
    assert text == tum_text([be[1] for be, _ in got], [p for _, p in got])
    Hs = segment_hooks()
    comp = MO.Pipeline(ko, deskew=True)
    l2bs = [s[2] for s in slots]
    for f, (fr, (be, pose)) in enumerate(zip(frames, got)):
        win = K.window(slots, fr["messages"])
        t_s = [s[0] for s in fr["samples"]]
        P = [s[1] for s in fr["samples"]]
        tables = [compose(Hs, t_s, P, l2b, be, win) for l2b in l2bs]
        assert all(tb is not None and len(tb) >= 10 for tb in tables)
        sensors = [dict(points=s["points"], stamps=s["stamps"] + s["offset"]) for s in oracle_sensors(slots, fr["messages"])]
        ref_frame = DO.preprocess_segments(ko, sensors, tables, l2bs, MAX_RANGE, 0.0, True)
        p_ref, _, _ = register_preprocessed(comp, ref_frame, fr["odom"])
        dt, ang = ko.pose_delta(pose, p_ref)
        assert dt <= TOL_T and ang <= TOL_R, (f, dt, ang)
    assert j["map_points"] == comp.num_map_points() and j["odometry_samples_per_frame"] == np.mean([len(fr["samples"]) for fr in frames])
    one, _ = replay(tmp_path / "m.kseq", tmp_path / "m.tum")
    _, a = tum_poses(text)
    _, b = tum_poses(one)
    worst = max(ko.pose_delta(x, y)[0] for x, y in zip(a, b))
    assert worst > 100 * TOL_T, worst


def test_samples_that_miss_the_sweep_are_refused(oracle, tmp_path):
    """a frame whose samples begin after its sweep does: non-zero exit naming the frame, no TUM file"""
    ko = oracle
    slots, frames, _ = turning_drive(ko)
    frames[3] = dict(frames[3], samples=frames[3]["samples"][2:])
    K.write_kseq3(str(tmp_path / "bad.kseq"), START, slots, frames)
    r = replay(tmp_path / "bad.kseq", tmp_path / "bad.tum", ok=False)
    assert r.returncode != 0 and "frame 3" in r.stderr and "cover" in r.stderr, r.stderr
    assert not (tmp_path / "bad.tum").exists()


# ------------------------------------------------------------------------------------------------------------ 5. publication
def test_publication_modes_agree(oracle, tmp_path):
    """a three-slot drive with samples: --publish host and device write the same digests, live and no publication the same poses"""
    ko = oracle
    slots, frames, traj = K.sensors_drive(ko, 6, ["rel", "scan", "scan"], 50)
    frames = K.with_samples(ko, traj, slots, frames, 5)
    K.write_kseq3(str(tmp_path / "d.kseq"), START, slots, frames)
    texts, digests = {}, {}
    for mode in ("none", "host", "device", "live"):
        extra = [] if mode == "none" else ["--publish", mode, "--publish-digest", tmp_path / (mode + ".digest")]
        texts[mode], j = replay(tmp_path / "d.kseq", tmp_path / (mode + ".tum"), *extra)
        assert j["publish"] == mode
        if mode != "none":
            digests[mode] = (tmp_path / (mode + ".digest")).read_text()
            assert len(digests[mode].splitlines()) == len(frames)
    assert digests["host"] == digests["device"] == digests["live"]
    assert texts["host"] == texts["device"] == texts["live"] == texts["none"]
