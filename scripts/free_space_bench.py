"""Free-space clearing (kicp_map_clear_free_space, kicp_ctx_set_free_space), measured on one GPU.

1. Per-frame time of the frame call with the option off and on ({min_misses 2, end_margin 0.5}), alternated over rounds (one fresh
   context and map per mode and round): the golden drive (tests/golden/pipeline_seq.npz, de-skewed), and synthetic frames of 131 k and
   262 k points (a street: two walls, a floor, clutter; seeded) registered repeatedly at the identity.  Host clock around each frame
   call (the call ends in its synchronisation); the first two frames of a drive are left out.  Median over all rounds.
2. The standalone call: 131 k points (cfg4's scan, oracle/workloads.py) against cfg4's map of about 1 M points, the map reloaded before
   every call; median over rounds.
3. "The van leaves": prior_map_bench.py's van (a 5 m x 2 m x 2 m box) present in the scans of the first half of the golden drive and gone
   after.  Per frame, the van's voxels left in the map with the option off and on, and the pose error against the unchanged drive.
4. Erosion on a static scene: the unchanged drive with the option on for a grid of (min_misses, end_margin); voxels cleared per frame
   and the map's size at the end against the option off.

Prints the card's name, power limit and maximum SM clock (read in the same run) and one JSON line.

    python scripts/free_space_bench.py [--rounds 5]
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

from prior_map_bench import KW, _built, _seq, _van, card  # noqa: E402

ON = (2, 0.5)


def _drive(kb, ko, seq, free, frames=None, times=None, poses=None, per_frame=None):
    """the golden drive (or `frames` in its place) on a fresh context and map with free-space clearing `free` (None: off)"""
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    if free:
        ctx.set_free_space(*free)
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


def _street(n, seed):
    rng = np.random.default_rng(seed)
    m = n // 4
    x = rng.uniform(-60, 60, (4, m))
    walls = [np.c_[x[0], np.full(m, 8.0) + rng.normal(0, 0.05, m), rng.uniform(-1, 6, m)],
             np.c_[x[1], np.full(m, -8.0) + rng.normal(0, 0.05, m), rng.uniform(-1, 6, m)],
             np.c_[x[2], rng.uniform(-8, 8, m), np.full(m, -1.5) + rng.normal(0, 0.02, m)],
             np.c_[x[3], rng.uniform(-7, 7, m), rng.uniform(-1.5, 2.5, m)]]
    return np.concatenate(walls)


def _synthetic(kb, n, free, frames=12):
    """the same synthetic frame registered `frames` times at the identity; per-frame seconds (the first two left out)"""
    I7 = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    pts = _street(n, 7)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    if free:
        ctx.set_free_space(*free)
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


def _van_keys(seq, gt):
    from oracle import kicp_oracle_py as ko
    l2b = seq["lidar_to_base"]
    sensor = ko.se3_compose(gt[0], l2b)
    frame0 = _van(seq, gt, 0)
    van_local = frame0[len(seq["frames"][0]):]
    world = ko.se3_transform(sensor, van_local)
    return {tuple(k) for k in np.floor(world).astype(np.int64).tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle import workloads as W
    ko.build()
    print("card:", card(), flush=True)
    seq = _seq()
    result = {"bench": "free_space", "card": card(), "frames": len(seq["frames"]), "rounds": args.rounds, "on": list(ON)}
    # 1. per-frame time, off and on, alternated
    per = {}
    for name in ("golden", "synthetic_131k", "synthetic_262k"):
        times = {"off": [], "on": []}
        for r in range(args.rounds):
            for mode in ("off", "on"):
                free = ON if mode == "on" else None
                if name == "golden":
                    _drive(kb, ko, seq, free, times=times[mode])
                else:
                    times[mode] += _synthetic(kb, 131072 if name.endswith("131k") else 262144, free)
        per[name] = {m: 1e3 * float(np.median(times[m])) for m in times}
        print(json.dumps({"frame_ms": name, **per[name]}), flush=True)
    result["frame_ms"] = per
    # 2. the standalone call against cfg4's map
    w4 = W.Workload(4)
    keys, counts, mpts = w4.map.export_voxels()
    scan = np.asarray(w4.scan, dtype=np.float64)
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w4.voxel_size, w4.max_range, w4.max_points_per_voxel)
    t = []
    for r in range(args.rounds + 1):
        gm.load_voxels(keys, counts, mpts)
        ctx.synchronize()
        t0 = time.perf_counter()
        st = gm.ClearFreeSpace(scan, w4.last_pose, (0.0, 0.0, 0.0), min_misses=ON[0], end_margin=ON[1])
        if r:
            t.append(time.perf_counter() - t0)
    gm.close()
    ctx.close()
    result["standalone"] = {"points": int(len(scan)), "map_points": int(len(mpts)), "median_ms": 1e3 * float(np.median(t)),
                            "stats": st._asdict()}
    print(json.dumps({"standalone": result["standalone"]}), flush=True)
    # 3. the van leaves
    _, gt = _built(kb, ko, seq)
    half = len(seq["frames"]) // 2
    frames = [_van(seq, gt, k) if k < half else seq["frames"][k] for k in range(len(seq["frames"]))]
    vk = _van_keys(seq, gt)
    van = {}
    for mode in ("off", "on"):
        left, poses = [], []

        def count(k, gm, ctx, left=left):
            keys = gm.export_voxels()[0]
            left.append(sum(1 for x in keys.tolist() if tuple(x) in vk))

        _drive(kb, ko, seq, ON if mode == "on" else None, frames=frames, poses=poses, per_frame=count)
        d = [ko.pose_delta(p, g) for p, g in zip(poses, gt)]
        van[mode] = {"van_voxels_per_frame": left, "max_pose_err_m": max(x[0] for x in d), "max_pose_err_rad": max(x[1] for x in d)}
    result["van"] = van
    print(json.dumps({"van": van}), flush=True)
    # 4. erosion on the unchanged drive
    ero = {}
    sizes = []
    _drive(kb, ko, seq, None, per_frame=lambda k, gm, ctx: sizes.append(gm.num_voxels()) if k == len(seq["frames"]) - 1 else None)
    ero["off"] = {"voxels_at_end": sizes[-1]}
    for mm in (1, 2, 4):
        for em in (0.0, 0.5, 1.0):
            cl, end = [], []

            def rec(k, gm, ctx, cl=cl, end=end):
                cl.append(kb.frame_free_space(ctx).cleared_voxels)
                if k == len(seq["frames"]) - 1:
                    end.append(gm.num_voxels())

            _drive(kb, ko, seq, (mm, em), per_frame=rec)
            ero["%d,%g" % (mm, em)] = {"cleared_per_frame_mean": float(np.mean(cl)), "cleared_total": int(np.sum(cl)),
                                       "voxels_at_end": end[-1]}
    result["erosion"] = ero
    print(json.dumps({"erosion": ero}), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
