"""TEST INFRASTRUCTURE — writer of version-3 .kseq drives (message streams of PointCloud2 records or LaserScans with their extrinsics,
odometry samples per frame; the layout kinematic-icp_b200/cpp/tools/kicp_replay.cpp documents), the sweep intervals the replay stages
them over, and synthetic drives built from the existing scenes (oracle's synth_scan world, tests/laser_projection.py's 2D world).

A slot is (kind, stamps_relative, lidar_to_base pose7).  A frame is dict(odom=pose7, samples=[(stamp, pose7)] (empty: one motion),
messages=[one per slot]); a records message is dict(records=uint8 array, point_step, offsets=(x, y, z), stamp_datatype, stamp_offset,
header), a LaserScan message dict(ranges=float32 array, header, angle_min, angle_max, angle_increment, time_increment, range_min,
range_max)."""
import struct

import numpy as np

import laser_projection as LP

RECORDS, LASER_SCAN = 0, 1
UINT32, FLOAT32, FLOAT64 = 6, 7, 8
SCAN_KEYS = ("angle_min", "angle_max", "angle_increment", "time_increment", "range_min", "range_max")


def write_kseq3(path, start, slots, frames):
    with open(path, "wb") as f:
        f.write(b"KSEQ3\0\0\0")
        f.write(struct.pack("<ii", len(frames), len(slots)))
        f.write(np.asarray(start, dtype="<f8").tobytes())
        for kind, rel, l2b in slots:
            f.write(struct.pack("<ii", kind, rel))
            f.write(np.asarray(l2b, dtype="<f8").tobytes())
        for fr in frames:
            f.write(np.asarray(fr["odom"], dtype="<f8").tobytes())
            samples = fr.get("samples") or []
            f.write(struct.pack("<ii", len(samples), 0))
            for stamp, pose in samples:
                f.write(struct.pack("<d", float(stamp)))
                f.write(np.asarray(pose, dtype="<f8").tobytes())
            assert len(fr["messages"]) == len(slots)
            for (kind, _, _), m in zip(slots, fr["messages"]):
                if kind == LASER_SCAN:
                    r = np.ascontiguousarray(m["ranges"], dtype="<f4").reshape(-1)
                    f.write(struct.pack("<ii", len(r), 0))
                    f.write(struct.pack("<d", float(m["header"])))
                    f.write(np.array([m[k] for k in SCAN_KEYS], dtype="<f4").tobytes())
                    f.write(r.tobytes())
                    continue
                raw = np.ascontiguousarray(m["records"], dtype=np.uint8).reshape(-1)
                step = m["point_step"]
                assert raw.size % step == 0
                f.write(struct.pack("<8i", raw.size // step, step, *m["offsets"], m["stamp_datatype"], m["stamp_offset"], 0))
                f.write(struct.pack("<d", float(m["header"])))
                f.write(raw.tobytes())


# ------------------------------------------------------------------------------------------------------------ sweeps
def message_stamps(kind, m):
    """the stamps the staging call decodes for a message, on its own clock (NaN included)"""
    if kind == LASER_SCAN:
        return LP.LaserProjector().project(m["ranges"], **{k: m[k] for k in SCAN_KEYS})["stamps"]
    if m["stamp_datatype"] == 0 or len(m["records"]) == 0:
        return np.zeros(0)
    fmt = {UINT32: "<u4", FLOAT32: "<f4", FLOAT64: "<f8"}[m["stamp_datatype"]]
    rec = np.frombuffer(np.ascontiguousarray(m["records"], np.uint8).tobytes(), dtype=np.dtype({"names": ["t"], "formats": [fmt],
                                                                                                "offsets": [m["stamp_offset"]],
                                                                                                "itemsize": m["point_step"]}))
    return np.array([LP.stamp_seconds(v) for v in rec["t"]], dtype=np.float64)


def offset(slot, m):
    kind, rel, _ = slot
    return float(m["header"]) if kind == LASER_SCAN or rel else 0.0


def window(slots, messages):
    """(T0, T1): the staged window, the stamps of all messages on the common clock (stamp + offset), None without stamps"""
    ts = [message_stamps(s[0], m) + offset(s, m) for s, m in zip(slots, messages)]
    t = np.concatenate(ts) if ts else np.zeros(0)
    t = t[~np.isnan(t)]
    return (float(t.min()), float(t.max())) if len(t) else None


def sweeps(slots, frames):
    """[(begin, end)] per frame as kicp_replay stages them: the first sweep begins at the earliest header stamp of the first frame, each
    frame's sweep at the end of the previous one; it ends at the latest of its messages' ends, each by process_timestamps' rule on the
    message's own clock (one slot: StageFrame / StageLaserScan; several: StageSensors, which takes the stamps back from the common
    clock)"""
    out = []
    last = min(float(m["header"]) for m in frames[0]["messages"]) if frames else 0.0
    for fr in frames:
        end = None
        for s, m in zip(slots, fr["messages"]):
            t = message_stamps(s[0], m)
            t = t[~np.isnan(t)]
            e = float(m["header"])
            if len(t):
                lo, hi = float(t.min()), float(t.max())
                if len(slots) > 1:
                    off = offset(s, m)
                    lo, hi = (lo + off) - off, (hi + off) - off
                if abs(e - hi) > 1e-8:
                    e = e + (hi - lo)
            end = e if end is None or e > end else end
        out.append((last, end))
        last = end
    return out


# ------------------------------------------------------------------------------------------------------------ messages
def records_message(pts, stamps, header, datatype=FLOAT64):
    """float32 x, y, z at 0, 4, 8 and the time field at 12 (UINT32 / FLOAT32) or 16 (FLOAT64), point_step 24"""
    fmt = {UINT32: "<u4", FLOAT32: "<f4", FLOAT64: "<f8"}[datatype]
    off = 16 if datatype == FLOAT64 else 12
    rec = np.zeros(len(pts), dtype=np.dtype({"names": ["x", "y", "z", "t"], "formats": ["<f4"] * 3 + [fmt], "offsets": [0, 4, 8, off],
                                             "itemsize": 24}))
    if len(pts):
        rec["x"], rec["y"], rec["z"], rec["t"] = pts[:, 0], pts[:, 1], pts[:, 2], stamps
    return dict(records=np.frombuffer(rec.tobytes(), dtype=np.uint8).copy(), point_step=24, offsets=(0, 4, 8), stamp_datatype=datatype,
                stamp_offset=off, header=header)


def records_points(m):
    """x, y, z of a records message widened to float64 (what the device ingests)"""
    rec = np.frombuffer(np.ascontiguousarray(m["records"], np.uint8).tobytes(),
                        dtype=np.dtype({"names": ["x", "y", "z"], "formats": ["<f4"] * 3, "offsets": list(m["offsets"]), "itemsize": m["point_step"]}))
    return np.stack([rec["x"], rec["y"], rec["z"]], 1).astype(np.float64)


def scan_message(ranges, header, **scan_kw):
    kw = {k: scan_kw.get(k, LP.SCAN[k]) for k in SCAN_KEYS}
    return dict(ranges=np.asarray(ranges, dtype=np.float32), header=header, **kw)


def projected_message(m):
    """the records projectLaser makes of a LaserScan message (x, y, z, stamps FLOAT32 at 0, 4, 8, 12), header kept"""
    proj = LP.LaserProjector().project(m["ranges"], **{k: m[k] for k in SCAN_KEYS})
    return dict(records=proj["records"], point_step=16, offsets=(0, 4, 8), stamp_datatype=FLOAT32, stamp_offset=12, header=m["header"])


# ------------------------------------------------------------------------------------------------------------ synthetic drives
def pose_at(ko, traj, t):
    """the base pose at t on a trajectory (t_s, poses, twists) sampled with constant velocity between samples"""
    t_s, P, tw = traj
    k = min(max(int(np.searchsorted(t_s, t, side="right")) - 1, 0), len(t_s) - 2)
    u = (t - t_s[k]) / (t_s[k + 1] - t_s[k])
    return ko.se3_compose(P[k], ko.se3_exp(u * tw[k]))


def trajectory(ko, duration, seed, dt=0.01, turn=0.8):
    """base poses every dt over [-0.05, duration + 0.05]: speed and yaw rate change at every sample (accelerating, braking, turning)"""
    rng = np.random.default_rng(seed)
    n = int(round((duration + 0.1) / dt)) + 1
    t = -0.05 + dt * np.arange(n)
    poses, twists = [ko.IDENTITY.copy()], []
    for k in range(n - 1):
        v = 2.0 + 1.5 * np.sin(0.15 * k) + rng.normal(0, 0.2)
        w = turn * np.sin(0.07 * k) + rng.normal(0, 0.1)
        twists.append(np.array([dt * v, 0.0, 0.0, 0.0, 0.0, dt * w]))
        poses.append(ko.se3_compose(poses[-1], ko.se3_exp(twists[-1])))
    return t, np.array(poses), np.array(twists)


def samples_over(ko, traj, begin, end, n):
    """n >= 2 samples of the trajectory evenly spread from just before begin to just after end: n - 1 de-skew segments"""
    margin = 1e-3 * (end - begin)
    return [(float(t), pose_at(ko, traj, t)) for t in np.linspace(begin - margin, end + margin, n)]


def with_samples(ko, traj, slots, frames, n):
    """the frames with n samples each over their sweeps and relative_odometry T(begin)^-1 T(end) (n 0: no samples)"""
    out = []
    for fr, (b, e) in zip(frames, sweeps(slots, frames)):
        odom = ko.se3_compose(ko.se3_inverse(pose_at(ko, traj, b)), pose_at(ko, traj, e))
        out.append(dict(fr, odom=odom, samples=samples_over(ko, traj, b, e, n) if n else []))
    return out


def sensor_pose(ko, traj, l2b, t):
    return ko.se3_compose(pose_at(ko, traj, t), l2b)


def world_3d(ko, traj, l2b, t, seed, beams=16, n_az=720):
    """a scan of the oracle's synthetic world from the sensor at time t, in the sensor's frame"""
    sp = sensor_pose(ko, traj, l2b, t)
    return ko.synth_scan(beams, -0.26, 0.26, n_az, sp[4], sp[5], 2.0 * np.arctan2(sp[2], sp[3]), seed)


def world_2d_ranges(ko, traj, l2b, t, rng, n=1081):
    """a LaserScan of tests/laser_projection.py's 2D world from the sensor at time t"""
    sp = sensor_pose(ko, traj, l2b, t)
    return LP.raycast(sp[4], sp[5], 2.0 * np.arctan2(sp[2], sp[3]), n, LP.SCAN["angle_min"], LP.SCAN["angle_increment"], rng)


def walls_3d(ko, traj, l2b, t, rng, rings=(-0.6, -0.2, 0.2, 0.6), n=1440):
    """a 3D sensor in the 2D world: its walls and pillars are vertical, so each ring sees the projected scan's x, y at its own height"""
    inc = 2 * 2.3561945 / (n - 1)
    sp = sensor_pose(ko, traj, l2b, t)
    r = LP.raycast(sp[4], sp[5], 2.0 * np.arctan2(sp[2], sp[3]), n, LP.SCAN["angle_min"], inc, rng)
    pts = LP.LaserProjector().project(r, LP.SCAN["angle_min"], LP.SCAN["angle_max"], inc, 0.0, 0.1, 30.0)["points"]
    return np.concatenate([np.column_stack([pts[:, :2], np.full(len(pts), z)]) for z in rings])


def sensors_drive(ko, frames, layout, seed, period=0.1, empty=None, l2bs=None, world="2d"):
    """A drive of len(layout) slots: "abs" / "rel" records slots (absolute stamps, or stamps relative to the header) and "scan"
    LaserScan slots, every slot sweeping [t0 + 4 ms i, t0 + 4 ms i + period) of frame t0 = period f.  world "2d": the records are
    walls_3d of the 2D world (the LaserScans' world); "3d": the oracle's 3D world (world_3d), LaserScans of random ranges.
    empty = (frame, slot): that message has no points.  Returns (slots, frames, trajectory) with no samples; add them with
    with_samples."""
    rng = np.random.default_rng(seed)
    traj = trajectory(ko, period * frames, seed)
    if l2bs is None:
        l2bs = [ko.se3_exp([0.8 * np.cos(2.1 * i), 0.5 * np.sin(2.1 * i), 0.0, 0.0, 0.0, 2.1 * i + 0.2]) for i in range(len(layout))]
    slots = [(LASER_SCAN if kind == "scan" else RECORDS, 1 if kind == "rel" else 0, l2b) for kind, l2b in zip(layout, l2bs)]
    out = []
    for f in range(frames):
        t0 = period * f
        msgs = []
        for i, kind in enumerate(layout):
            start = t0 + 0.004 * i
            if kind == "scan":
                r = world_2d_ranges(ko, traj, l2bs[i], start + period, rng) if world == "2d" else rng.uniform(0.2, 30.0, 1081).astype(np.float32)
                if empty == (f, i):
                    r = r[:0]
                msgs.append(scan_message(r, start, time_increment=period / len(r) if len(r) else LP.SCAN["time_increment"]))
                continue
            pts = walls_3d(ko, traj, l2bs[i], start + period, rng) if world == "2d" else world_3d(ko, traj, l2bs[i], start + period, 31 * f + i)
            if empty == (f, i):
                pts = pts[:0]
            rel = rng.uniform(0.0, period, len(pts))
            if len(pts) > 1:
                rel[0], rel[1] = 0.0, period * (1 - 1e-6)
            msgs.append(records_message(pts, rel if kind == "rel" else start + rel, start))
        out.append(dict(odom=ko.IDENTITY.copy(), samples=[], messages=msgs))
    return slots, with_samples(ko, traj, slots, out, 0), traj
