"""A frozen prior inside the voxel map (kicp_map_freeze), timed on one GPU.

1. Per-frame cost with a large prior.  Priors of about 0.25 M, 1 M and 4 M voxels: the map the golden drive
   (tests/golden/pipeline_seq.npz, de-skewed) builds, in the middle, and copies of cfg4's map (oracle/workloads.py, seeded; its points
   re-inserted into 1 m voxels) tiled on a square lattice around it, each copy moved by a whole number of voxels so that the copies never share a voxel.  The golden drive is
   registered frame after frame against each prior under four modes, alternated over rounds (one fresh context and map per mode and
   round, the prior loaded before the drive):
     never          the prior as it is, no Update (kicp_ctx_set_map_update NEVER);
     frozen_always  the prior frozen, ALWAYS: the Update compacts and re-inserts the live layer only;
     frozen_gated   the prior frozen, GATED with thresholds that pass every frame (the report's and the gate's launches on top);
     unfrozen       the prior NOT frozen, ALWAYS, on a map whose max_distance (1e9 m) evicts nothing: what keeping the prior costs
                    without freezing it (every frame compacts and re-inserts every voxel).
   Host clock around each frame call (the call ends in its synchronisation); the first two frames of a drive are left out (they
   allocate).  Reported: the median over all timed frames of all rounds, and the spread of the per-round medians.
2. A changed scene: a box of points (a parked van, 5 m x 2 m x 2 m, 51 x 51 points on each face) added to every scan of the golden drive
   at a fixed place in the world, after the prior was built from the unchanged drive.  The changed drive is registered under NEVER
   and under frozen prior + ALWAYS; the pose error of each is taken against the poses of the unchanged drive's own ALWAYS run (the
   ground truth of this synthetic drive).  Reported without a threshold.

Prints the card's name, power limit and maximum SM clock (read in the same run) and one JSON line.

    python scripts/prior_map_bench.py [--rounds 3] [--sizes 250000,1000000,4000000]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kinematic-icp_b200", "python")):
    sys.path.insert(0, p)

KW = dict(max_range=100.0, min_range=0.0, deskew=True, voxel_size=1.0)
MODES = ("never", "frozen_always", "frozen_gated", "unfrozen")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def _seq():
    from oracle import sequences as S2
    return S2.unpack_sequence(np.load(os.path.join(ROOT, "tests", "golden", "pipeline_seq.npz")), True)


def _drive(kb, ko, gm, ctx, seq, frames=None, times=None, poses=None):
    """the golden drive (or `frames` in its place) on gm; per-frame times appended to `times`, poses to `poses`"""
    l2b = seq["lidar_to_base"]
    threshold = ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0)
    last = np.array(seq["start"], dtype=np.float64)
    frames = frames if frames is not None else seq["frames"]
    for k, frame in enumerate(frames):
        odom = seq["odoms"][k]
        motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
        tau = threshold.compute()
        t0 = time.perf_counter()
        pose = kb.RegisterFrame(gm, frame, seq["stamps"][k] if len(seq["stamps"][k]) == len(frame) else np.linspace(0, 1, len(frame)),
                                motion, l2b, last, odom, tau, want_clouds=False, **KW)[0]
        dt = time.perf_counter() - t0
        if times is not None and k >= 2:
            times.append(dt)
        if poses is not None:
            poses.append(np.array(pose))
        threshold.update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(last, odom)), pose))
        last = pose
    return last


def _built(kb, ko, seq):
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
    poses = []
    _drive(kb, ko, gm, ctx, seq, poses=poses)
    v = gm.export_voxels()
    gm.close()
    ctx.close()
    return v, poses


def _tiled(centre, tile, target):
    """`centre` plus copies of `tile` on a square lattice around it until about `target` voxels"""
    ck, cc, cp = centre
    tk, tc, tp = tile
    lo = np.minimum(ck.min(0), tk.min(0)).astype(np.int64)
    hi = np.maximum(ck.max(0), tk.max(0)).astype(np.int64)
    step = int(max(hi[0] - lo[0], hi[1] - lo[1])) + 8
    keys, counts, pts = [ck], [cc], [cp]
    n, ring = len(cc), 1
    while n < target:
        for i in range(-ring, ring + 1):
            for j in range(-ring, ring + 1):
                if max(abs(i), abs(j)) != ring or n >= target:
                    continue
                off = np.array([i * step, j * step, 0], dtype=np.int64)
                keys.append((tk + off).astype(np.int32))
                counts.append(tc)
                pts.append(tp + off.astype(np.float64))  # whole metres (= whole voxels of 1 m): every point stays in its voxel
                n += len(tc)
        ring += 1
    return np.concatenate(keys), np.concatenate(counts), np.concatenate(pts)


def _van(seq, gt_poses, k):
    """frame k of the changed scene: the van's faces, in the sensor frame of that frame's ground-truth pose, after the scan's points"""
    from oracle import kicp_oracle_py as ko
    g = np.arange(0.0, 1.0 + 1e-9, 0.02)
    a, b = np.meshgrid(g, g)
    a, b = a.ravel(), b.ravel()
    size = np.array([5.0, 2.0, 2.0])
    faces = []
    for ax in range(3):
        o = [d for d in range(3) if d != ax]
        for side in (0.0, 1.0):
            f = np.zeros((len(a), 3))
            f[:, ax] = side
            f[:, o[0]], f[:, o[1]] = a, b
            faces.append(f * size)
    start = np.array(seq["start"])[4:]
    van = np.concatenate(faces) + np.array([start[0] + 12.0, start[1] + 4.0, -1.0])
    l2b = seq["lidar_to_base"]
    sensor = ko.se3_compose(gt_poses[k], l2b)
    local = ko.se3_transform(ko.se3_inverse(sensor), van)
    local = local[np.linalg.norm(local, axis=1) < 60.0]
    return np.concatenate([seq["frames"][k], local])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="250000,1000000,4000000")
    args = ap.parse_args()
    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle import workloads as W
    ko.build()
    print("card:", card(), flush=True)
    seq = _seq()
    centre, gt = _built(kb, ko, seq)
    w4 = W.Workload(4)  # cfg4's map has 0.5 m voxels: its points, re-inserted into a map of the drive's 1 m voxels
    t = ko.OracleMap(1.0, 1e9, 20)
    t.add_points(w4.map.pointcloud())
    tile = t.export_voxels()
    result = {"bench": "prior_map", "card": card(), "frames": len(seq["frames"]), "rounds": args.rounds, "sizes": {}}
    for target in [int(s) for s in args.sizes.split(",")]:
        prior = _tiled(centre, tile, target)
        times = {m: [] for m in MODES}
        round_medians = {m: [] for m in MODES}
        for r in range(args.rounds):
            for mode in MODES:
                ctx = kb.Context(0)
                gm = kb.VoxelHashMap(ctx, 1.0, 1e9 if mode == "unfrozen" else 100.0, 20)
                gm.load_voxels(*prior)
                if mode.startswith("frozen"):
                    gm.freeze()
                ctx.set_map_update(1 if mode == "never" else 2 if mode == "frozen_gated" else 0, min_inliers=0, min_fitness=0.0,
                                   max_inlier_rmse=math.inf)
                t = []
                _drive(kb, ko, gm, ctx, seq, times=t)
                times[mode] += t
                round_medians[mode].append(float(np.median(t)))
                gm.close()
                ctx.close()
        entry = {"voxels": int(len(prior[1])), "points": int(len(prior[2]))}
        for m in MODES:
            entry[m] = {"median_ms": 1e3 * float(np.median(times[m])), "round_median_ms_min": 1e3 * min(round_medians[m]),
                        "round_median_ms_max": 1e3 * max(round_medians[m])}
        result["sizes"][str(target)] = entry
        print(json.dumps({"size": target, **entry}), flush=True)
    # 2. the changed scene
    changed = [_van(seq, gt, k) for k in range(len(seq["frames"]))]
    err = {}
    for mode in ("never", "frozen_always"):
        ctx = kb.Context(0)
        gm = kb.VoxelHashMap(ctx, 1.0, 100.0, 20)
        gm.load_voxels(*centre)
        if mode == "frozen_always":
            gm.freeze()
        ctx.set_map_update(1 if mode == "never" else 0)
        poses = []
        _drive(kb, ko, gm, ctx, seq, frames=changed, poses=poses)
        d = [ko.pose_delta(p, g) for p, g in zip(poses, gt)]
        err[mode] = {"max_m": max(x[0] for x in d), "mean_m": float(np.mean([x[0] for x in d])), "max_rad": max(x[1] for x in d),
                     "live_voxels_at_end": int(gm.num_voxels() - gm.num_prior_voxels())}
        gm.close()
        ctx.close()
    result["changed_scene"] = err
    print(json.dumps(result))


if __name__ == "__main__":
    main()
