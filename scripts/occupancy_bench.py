"""Occupancy evidence in free-space clearing (kicp_map_set_occupancy), measured on one GPU.

1. Per-frame time of the frame call in three modes, alternated over rounds (one fresh context and map per mode and round): clearing
   off, memoryless clearing {min_misses 2, end_margin 0.5}, and the same clearing with occupancy at the Python defaults (or --occupancy).
   On the golden drive and on free_space_bench.py's synthetic street of 131 k and 262 k points.  Host clock around each frame call (the
   call ends in its synchronisation); the first two frames of a drive are left out.  Median over all rounds.
2. The standalone call on cfg4's scan against cfg4's map (oracle/workloads.py), occupancy off and on, the map reloaded before every call.
3. "The van leaves": prior_map_bench.py's van present in the first half of two drives and gone after: the golden drive, and a 40-frame
   drive of oracle/sequences.make_sequence.  Per frame, the van's voxels left in the map: clearing off, memoryless, and a small grid of
   occupancy settings, at min_misses 1 and 2 (end_margin 0.5).
4. Erosion: the same drives unchanged, voxels in the map at the end for the same settings.

A setting QUALIFIES on a drive and min_misses when it erodes less than memoryless {2, 0.5} and leaves no more van voxels at the last
frame than memoryless {2, 0.5}.  Prints the card's name, power limit and maximum SM clock (read in the same run) and one JSON line.

    python scripts/occupancy_bench.py [--rounds 3] [--occupancy I,G,L,M]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kinematic-icp_b200", "python"), os.path.join(ROOT, "scripts")):
    sys.path.insert(0, p)

from free_space_bench import _street  # noqa: E402
from prior_map_bench import KW, _van, card  # noqa: E402

MEMORYLESS = (2, 0.5)
# (initial, hit_gain, miss_loss, max_evidence); (1, 0, 1, 1) is the memoryless rule
GRID = [(1, 1, 1, 2), (1, 1, 1, 4), (2, 1, 1, 4), (2, 1, 1, 8), (3, 1, 1, 3), (1, 2, 1, 6)]


def _drive(kb, ko, seq, free, occ, frames=None, times=None, poses=None, per_frame=None):
    """`seq` (or `frames` in its place) on a fresh context and map: clearing `free` (None: off), occupancy `occ` (None: off)"""
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    if free:
        ctx.set_free_space(*free)
    if occ:
        gm.set_occupancy(*occ)
    l2b = seq["lidar_to_base"]
    threshold = ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
    last = np.array(seq["start"], dtype=np.float64)
    frames = frames if frames is not None else seq["frames"]
    for k, frame in enumerate(frames):
        odom = seq["odoms"][k]
        motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
        tau = threshold.compute()
        stamps = seq["stamps"][k] if len(seq["stamps"][k]) == len(frame) else np.linspace(0, 1, len(frame))
        t0 = time.perf_counter()
        pose = kb.RegisterFrame(gm, frame, stamps, motion, l2b, last, odom, tau, want_clouds=False, **KW)[0]
        dt = time.perf_counter() - t0
        if times is not None and k >= 2:
            times.append(dt)
        if poses is not None:
            poses.append(np.array(pose))
        if per_frame is not None:
            per_frame(k, gm, ctx)
        threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(last, odom)), pose))
        last = pose
    gm.close()
    ctx.close()


def _synthetic(kb, n, free, occ, frames=12):
    I7 = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    pts = _street(n, 7)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    if free:
        ctx.set_free_space(*free)
    if occ:
        gm.set_occupancy(*occ)
    t = []
    for k in range(frames):
        t0 = time.perf_counter()
        kb.RegisterFrame(gm, pts, np.zeros(0), I7, I7, I7, I7, 2.0, want_clouds=False, max_range=100.0, min_range=0.0, deskew=False,
                         voxel_size=1.0)
        if k >= 2:
            t.append(time.perf_counter() - t0)
    gm.close()
    ctx.close()
    return t


def _van_keys(ko, seq, gt):
    sensor = ko.se3_compose(gt[0], seq["lidar_to_base"])
    van_local = _van(seq, gt, 0)[len(seq["frames"][0]):]
    return {tuple(k) for k in np.floor(ko.se3_transform(sensor, van_local)).astype(np.int64).tolist()}


def _drives(ko):
    from oracle import sequences as S2
    golden = S2.unpack_sequence(np.load(os.path.join(ROOT, "tests", "golden", "pipeline_seq.npz")), True)
    return {"golden": golden, "long40": S2.make_sequence(n_frames=40, deskew=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--occupancy", default=None, help="I,G,L,M timed in sections 1 and 2 (default: the Python defaults)")
    args = ap.parse_args()
    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle import workloads as W
    ko.build()
    occ = tuple(int(x) for x in args.occupancy.split(",")) if args.occupancy else \
        (kb.OCCUPANCY_INITIAL, kb.OCCUPANCY_HIT_GAIN, kb.OCCUPANCY_MISS_LOSS, kb.OCCUPANCY_MAX_EVIDENCE)
    print("card:", card(), flush=True)
    drives = _drives(ko)
    result = {"bench": "occupancy", "card": card(), "rounds": args.rounds, "memoryless": list(MEMORYLESS), "occupancy": list(occ),
              "frames": {k: len(v["frames"]) for k, v in drives.items()}}
    modes = {"off": (None, None), "memoryless": (MEMORYLESS, None), "occupancy": (MEMORYLESS, occ)}
    # 1. per-frame time, the three modes alternated
    per = {}
    for name in ("golden", "synthetic_131k", "synthetic_262k"):
        times = {m: [] for m in modes}
        for r in range(args.rounds):
            for mode, (free, o) in modes.items():
                if name == "golden":
                    _drive(kb, ko, drives["golden"], free, o, times=times[mode])
                else:
                    times[mode] += _synthetic(kb, 131072 if name.endswith("131k") else 262144, free, o)
        per[name] = {m: 1e3 * float(np.median(times[m])) for m in times}
        per[name]["spread_ms"] = {m: 1e3 * float(np.percentile(times[m], 75) - np.percentile(times[m], 25)) for m in times}
        print(json.dumps({"frame_ms": name, **per[name]}), flush=True)
    result["frame_ms"] = per
    # 2. the standalone call against cfg4's map, occupancy off and on (alternated)
    w4 = W.Workload(4)
    keys, counts, mpts = w4.map.export_voxels()
    scan = np.asarray(w4.scan, dtype=np.float64)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w4.voxel_size, w4.max_range, w4.max_points_per_voxel)
    t = {"off": [], "on": []}
    for r in range(args.rounds + 1):
        for mode in ("off", "on"):
            gm.set_occupancy(*occ) if mode == "on" else gm.set_occupancy(None)
            gm.load_voxels(keys, counts, mpts)
            ctx.synchronize()
            t0 = time.perf_counter()
            gm.ClearFreeSpace(scan, w4.last_pose, (0.0, 0.0, 0.0), min_misses=MEMORYLESS[0], end_margin=MEMORYLESS[1])
            if r:
                t[mode].append(time.perf_counter() - t0)
    gm.close()
    ctx.close()
    result["standalone_ms"] = {m: 1e3 * float(np.median(v)) for m, v in t.items()}
    result["standalone_points"], result["standalone_map_points"] = int(len(scan)), int(len(mpts))
    print(json.dumps({"standalone_ms": result["standalone_ms"]}), flush=True)
    # 3 and 4. the van and the erosion, per drive, for off, memoryless and the grid at min_misses 1 and 2
    settings = [("off", None, None)]
    for mm in (1, 2):
        settings.append(("memoryless,%d" % mm, (mm, 0.5), None))
        settings += [("%d,%d,%d,%d,%d" % (o + (mm,)), (mm, 0.5), o) for o in GRID]
    van, ero, qual = {}, {}, {}
    for dname, seq in drives.items():
        gt = []
        _drive(kb, ko, seq, None, None, poses=gt)
        half = len(seq["frames"]) // 2
        frames = [_van(seq, gt, k) if k < half else seq["frames"][k] for k in range(len(seq["frames"]))]
        vk = _van_keys(ko, seq, gt)
        van[dname], ero[dname] = {}, {}
        for label, free, o in settings:
            left = []

            def count(k, gm, ctx, left=left):
                left.append(sum(1 for x in gm.export_voxels()[0].tolist() if tuple(x) in vk))

            _drive(kb, ko, seq, free, o, frames=frames, per_frame=count)
            van[dname][label] = left
            end = []
            _drive(kb, ko, seq, free, o, per_frame=lambda k, gm, ctx, end=end: end.append(gm.num_voxels()))
            ero[dname][label] = end[-1]
        print(json.dumps({"van": dname, "per_frame": van[dname]}), flush=True)
        print(json.dumps({"erosion": dname, "voxels_at_end": ero[dname]}), flush=True)
        ref_end, ref_van = ero[dname]["memoryless,2"], van[dname]["memoryless,2"][-1]
        qual[dname] = [label for label, free, o in settings if o and ero[dname][label] > ref_end and van[dname][label][-1] <= ref_van]
    result["van_voxels_per_frame"], result["voxels_at_end"] = van, ero
    result["qualifying"] = sorted(set(qual["golden"]) & set(qual["long40"]))
    print(json.dumps({"qualifying": qual}), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
