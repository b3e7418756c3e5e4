"""The version-3 .kseq reader (kinematic-icp_b200/cpp/kicp/kseq.hpp) on the CPU, through tests/hooks/kseq_hooks.cpp: files written by
tests/kseq3.py with mixed slots, empty messages and odometry samples come back with the same counts, headers, layouts and bytes, and
every malformed file is refused with a message that names the frame and the slot."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import kseq3 as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")


@pytest.fixture(scope="module")
def hooks():
    import __graft_entry__ as g
    g.build()
    L = C.CDLL(os.path.join(ROOT, "tests", "hooks", "_build", "libkicp_kseq_hooks.so"))
    L.kseq3_rewrite.restype = C.c_int32
    L.kseq3_rewrite.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32]
    L.kseq3_offsets.restype = C.c_int64
    L.kseq3_offsets.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_int32]
    return L


def read_error(L, path):
    """the reader's message for the file at path, None when it reads"""
    err = C.create_string_buffer(512)
    out = str(path) + ".out"
    r = L.kseq3_rewrite(str(path).encode(), out.encode(), err, 512)
    return None if r == 0 else err.value.decode()


def pose(rng):
    q = rng.normal(size=4)
    return np.concatenate([q / np.linalg.norm(q), rng.normal(size=3)])


def records(rng, n, layout):
    """n records of one of three layouts: (point_step, offsets, stamp_datatype, stamp_offset)"""
    step, offs, dt, t_off = layout
    raw = rng.integers(0, 256, n * step, dtype=np.uint8)
    return dict(records=raw, point_step=step, offsets=offs, stamp_datatype=dt, stamp_offset=t_off, header=float(rng.uniform(10, 20)))


LAYOUTS = [(24, (0, 4, 8), K.FLOAT64, 16), (20, (8, 12, 16), K.UINT32, 0), (13, (9, 1, 5), 0, 0), (16, (0, 4, 8), K.FLOAT32, 12)]


def mixed_drive(rng, frames=5):
    """four slots (three records layouts, one LaserScan, one slot sharing another's extrinsic), empty messages, 0 to 4 samples"""
    l2b = pose(rng)
    slots = [(K.RECORDS, 1, l2b), (K.LASER_SCAN, 0, pose(rng)), (K.RECORDS, 0, pose(rng)), (K.RECORDS, 1, l2b)]
    out = []
    for f in range(frames):
        msgs = []
        for i, (kind, _, _) in enumerate(slots):
            n = 0 if (f + i) % 4 == 3 else int(rng.integers(1, 300))
            if kind == K.LASER_SCAN:
                msgs.append(K.scan_message(rng.uniform(0, 30, n).astype(np.float32), float(rng.uniform(10, 20)),
                                           time_increment=float(rng.uniform(1e-5, 1e-4))))
            else:
                msgs.append(records(rng, n, LAYOUTS[(f + i) % len(LAYOUTS)]))
        t = np.sort(rng.uniform(0, 100, f % 5))
        out.append(dict(odom=pose(rng), samples=[(float(s), pose(rng)) for s in t], messages=msgs))
    return slots, out


def test_round_trip(hooks, tmp_path):
    """read and written back: the same bytes; the views' time offsets follow the slot table"""
    rng = np.random.default_rng(1)
    slots, frames = mixed_drive(rng)
    path = tmp_path / "drive.kseq"
    K.write_kseq3(str(path), pose(rng), slots, frames)
    err = C.create_string_buffer(512)
    assert hooks.kseq3_rewrite(str(path).encode(), str(tmp_path / "back.kseq").encode(), err, 512) == 0, err.value
    assert (tmp_path / "back.kseq").read_bytes() == path.read_bytes()
    n = len(frames) * len(slots)
    offsets, is_scan = np.zeros(n), np.zeros(n, np.int32)
    assert hooks.kseq3_offsets(str(path).encode(), offsets.ctypes.data, is_scan.ctypes.data, n, err, 512) == n
    for f, fr in enumerate(frames):
        for s, ((kind, rel, _), m) in enumerate(zip(slots, fr["messages"])):
            assert is_scan[f * len(slots) + s] == (kind == K.LASER_SCAN)
            assert offsets[f * len(slots) + s] == (m["header"] if kind == K.LASER_SCAN or rel else 0.0)
    # one slot, no samples, no frames at all
    for fr in ([], frames[:1]):
        K.write_kseq3(str(path), pose(rng), slots[1:2], [dict(f, messages=f["messages"][1:2]) for f in fr])
        assert read_error(hooks, path) is None
        assert (tmp_path / "drive.kseq.out").read_bytes() == path.read_bytes()


# ---------------------------------------------------------------------------------------------------------- malformed
def small_drive():
    """two slots (records FLOAT64 stamps, LaserScan), two frames, frame 1 with three samples; and the byte offsets of its parts"""
    rng = np.random.default_rng(2)
    slots = [(K.RECORDS, 0, np.array([0, 0, 0, 1.0, 0, 0, 0])), (K.LASER_SCAN, 0, np.array([0, 0, 0, 1.0, 0.5, 0, 0]))]
    frames = []
    for f in range(2):
        msgs = [records(rng, 10, LAYOUTS[0]), K.scan_message(rng.uniform(0, 30, 7).astype(np.float32), 10.0 + f)]
        samples = [(1.0, pose(rng)), (2.0, pose(rng)), (3.0, pose(rng))] if f == 1 else []
        frames.append(dict(odom=pose(rng), samples=samples, messages=msgs))
    at = {"n_frames": 8, "n_slots": 12, "start": 16}
    o = 72
    for s in range(2):
        at[("slot", s)] = o
        o += 64
    for f, fr in enumerate(frames):
        at[("frame", f)] = o
        o += 64
        at[("samples", f)] = o
        o += 64 * len(fr["samples"])
        at[("msg", f, 0)] = o
        o += 40 + 10 * 24
        at[("msg", f, 1)] = o
        o += 40 + 4 * 7
    at["end"] = o
    return slots, frames, at


def patched(path, at, fmt, *values):
    b = bytearray(path.read_bytes())
    struct.pack_into(fmt, b, at, *values)
    out = path.parent / "bad.kseq"
    out.write_bytes(bytes(b))
    return out


def test_malformed_files_are_refused(hooks, tmp_path):
    slots, frames, at = small_drive()
    path = tmp_path / "drive.kseq"
    K.write_kseq3(str(path), np.array([0, 0, 0, 1.0, 0, 0, 0]), slots, frames)
    assert len(path.read_bytes()) == at["end"] and read_error(hooks, path) is None
    nan, inf = float("nan"), float("inf")
    m1, m11, fr0, fr1, smp = at[("msg", 1, 0)], at[("msg", 1, 1)], at[("frame", 0)], at[("frame", 1)], at[("samples", 1)]
    cases = [
        ((0, "8s", b"KSEQ9\0\0\0"), "bad magic"),
        ((0, "8s", b"KSEQ2\0\0\0"), "version-2"),
        ((at["n_slots"], "<i", 0), "slot count 0"),
        ((at["n_slots"], "<i", 9), "slot count 9"),
        ((at[("slot", 1)], "<i", 2), "slot 1: kind 2"),
        ((at[("slot", 1)] + 4, "<i", 2), "slot 1: stamps_relative 2"),
        ((at[("slot", 0)] + 8 + 8 * 4, "<d", nan), "slot 0: non-finite lidar_to_base"),
        ((at["start"] + 8, "<d", inf), "non-finite start pose"),
        ((at["n_frames"], "<i", -1), "implausible frame count"),
        ((at["n_frames"], "<i", 1 << 20), "implausible frame count"),
        ((fr0 + 8 * 5, "<d", nan), "frame 0: non-finite relative_odometry"),
        ((fr0 + 56, "<i", -1), "frame 0: implausible sample count"),
        ((fr1 + 56, "<i", 1 << 28), "frame 1: implausible sample count"),
        ((smp + 64, "<d", nan), "frame 1: sample 1: non-finite stamp"),
        ((smp + 128 + 8 + 8 * 2, "<d", -inf), "frame 1: sample 2: non-finite pose"),
        ((smp + 128, "<d", 1.5), "frame 1: sample 2: stamps do not increase"),
        ((smp + 64, "<d", 1.0), "frame 1: sample 1: stamps do not increase"),
        ((m1, "<i", -3), "frame 1, slot 0: negative point count"),
        ((m1 + 4, "<i", 0), "frame 1, slot 0: point_step 0"),
        ((m1 + 4, "<i", -24), "frame 1, slot 0: point_step -24"),
        ((m1 + 16, "<i", 21), "frame 1, slot 0: z outside point_step"),
        ((m1 + 8, "<i", -1), "frame 1, slot 0: x outside point_step"),
        ((m1 + 20, "<i", 5), "frame 1, slot 0: stamp_datatype 5"),
        ((m1 + 24, "<i", 17), "frame 1, slot 0: time field outside point_step"),
        ((m1 + 32, "<d", nan), "frame 1, slot 0: non-finite header stamp"),
        ((m1, "<i", 1 << 30), "frame 1, slot 0: truncated"),
        ((m11, "<i", -7), "frame 1, slot 1: negative beam count"),
        ((m11, "<i", 8), "frame 1, slot 1: truncated"),
        ((m11 + 8, "<d", inf), "frame 1, slot 1: non-finite header stamp"),
    ]
    for (off, fmt, value), text in cases:
        err = read_error(hooks, patched(path, off, fmt, value))
        assert err is not None and text in err, (text, err)
    raw = path.read_bytes()
    for cut, text in [(at[("msg", 1, 1)] + 50, "frame 1, slot 1: truncated while reading the ranges"),
                      (at[("msg", 1, 0)] + 45, "frame 1, slot 0: truncated while reading the records"),
                      (at[("msg", 0, 1)] + 20, "frame 0, slot 1: truncated while reading the message header"),
                      (smp + 70, "frame 1: truncated while reading the odometry samples"), (fr1 + 10, "frame 1: truncated"),
                      (at[("slot", 1)] + 10, "slot 1: truncated"), (5, "truncated while reading the magic")]:
        (tmp_path / "cut.kseq").write_bytes(raw[:cut])
        err = read_error(hooks, tmp_path / "cut.kseq")
        assert err is not None and text in err, (text, err)
    (tmp_path / "long.kseq").write_bytes(raw + b"\0" * 3)
    assert "3 bytes after the last frame" in read_error(hooks, tmp_path / "long.kseq")


def test_replay_refuses_host_stamps_for_kseq3(hooks, tmp_path):
    """--host-stamps has no multi-sensor entry point: refused before the replay starts"""
    slots, frames, _ = small_drive()
    K.write_kseq3(str(tmp_path / "d.kseq"), np.array([0, 0, 0, 1.0, 0, 0, 0]), slots, frames)
    r = subprocess.run([EXE, str(tmp_path / "d.kseq"), str(tmp_path / "o.tum"), "--host-stamps"], capture_output=True, text=True)
    assert r.returncode == 2 and "--host-stamps" in r.stderr and "KSEQ3" in r.stderr
    assert not (tmp_path / "o.tum").exists()


def test_sweeps_follow_the_stamp_rules():
    """kseq3.sweeps: the first sweep begins at the earliest header stamp; a message stamped at its end ends there, one whose stamps
    are relative or begin at the header ends a sweep duration later; the latest message ends the frame"""
    a = K.records_message(np.zeros((3, 3)), np.array([5.0, 5.05, 5.1]), 5.1)  # absolute, header at the end
    b = K.records_message(np.zeros((3, 3)), np.array([0.0, 0.02, 0.08]), 5.03)  # relative to a header at the beginning
    slots = [(K.RECORDS, 0, None), (K.RECORDS, 1, None)]
    sw = K.sweeps(slots, [dict(messages=[a, b]), dict(messages=[dict(a, header=5.2), dict(b, header=5.3)])])
    assert sw[0][0] == 5.03 and abs(sw[0][1] - 5.11) < 1e-12 and sw[1][0] == sw[0][1] and abs(sw[1][1] - 5.38) < 1e-12
    assert K.sweeps(slots[:1], [dict(messages=[dict(a, records=a["records"][:0])])]) == [(5.1, 5.1)]
