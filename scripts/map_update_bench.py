"""The frame path's map-update policy, timed on one GPU.

1. Per-frame time of kicp_register_frame under ALWAYS, GATED (thresholds (0, 0.0, inf): every frame applied, option "correspondences"
   off, so the report's two launches and the gate's one are the whole difference) and NEVER (against the map the drive built), on
   three contexts driven with the same frames in alternated rounds: the golden drive (tests/golden/pipeline_seq.npz, de-skewed) and
   cfg4's scan (261 675 points) registered frame after frame at the pose it was taken from.  Host clock around each call (the call ends
   in its synchronisation).
2. Localising on a prior map: the golden drive replayed under NEVER against the map its own ALWAYS run built, its poses against the
   ALWAYS run's (maximum translation and rotation difference).

Prints the card's name and power limit (read in the same run) and one JSON line.

    python scripts/map_update_bench.py [--rounds 5] [--frames 30]
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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


MODES = ("always", "gated", "never")


def _contexts(kb, vs=1.0):
    out = {}
    for m, code in zip(MODES, (0, 2, 1)):
        ctx = kb.Context(0)
        gm = kb.VoxelHashMap(ctx, vs, 100.0, 20)
        out[m] = (ctx, gm, code)
    return out


def golden(kb, ko, rounds):
    from oracle import sequences as S2
    seq = S2.unpack_sequence(np.load(os.path.join(ROOT, "tests", "golden", "pipeline_seq.npz")), True)
    l2b = seq["lidar_to_base"]
    cs = _contexts(kb)
    times = {m: [] for m in MODES}
    poses = {m: [] for m in MODES}
    prior = None
    for r in range(rounds + 1):
        for m in MODES:
            ctx, gm, code = cs[m]
            ctx.set_map_update(0)
            gm.Clear()
            if m == "never" and prior is not None:
                gm.load_voxels(*prior)
            ctx.set_map_update(code)
        last = {m: np.array(seq["start"], dtype=np.float64) for m in MODES}
        thr = {m: ko.OracleThreshold(1.0 / np.sqrt(20), 100.0, True, 1.0) for m in MODES}
        for m in MODES:
            poses[m] = []
        for frame, stamps, odom in zip(seq["frames"], seq["stamps"], seq["odoms"]):
            motion = ko.se3_compose(ko.se3_compose(ko.se3_inverse(l2b), odom), l2b)
            for m in MODES:
                ctx, gm, _ = cs[m]
                tau = thr[m].compute()
                t0 = time.perf_counter()
                pose = kb.RegisterFrame(gm, frame, stamps, motion, l2b, last[m], odom, tau, max_range=100.0, min_range=0.0, deskew=True,
                                        voxel_size=1.0, want_clouds=False)[0]
                dt = time.perf_counter() - t0
                if r > 0 and (m != "never" or prior is not None):
                    times[m].append(dt)
                thr[m].update(ko.se3_compose(ko.se3_inverse(ko.se3_compose(last[m], odom)), pose))
                last[m] = pose
                poses[m].append(pose)
        if prior is None:
            prior = cs["always"][1].export_voxels()
    worst = (0.0, 0.0)
    for a, b in zip(poses["never"], poses["always"]):
        d = ko.pose_delta(a, b)
        worst = (max(worst[0], d[0]), max(worst[1], d[1]))
    for ctx, gm, _ in cs.values():
        gm.close()
        ctx.close()
    return {m: 1e3 * float(np.median(times[m])) for m in MODES}, worst, len(seq["frames"])


def cfg4(kb, Workload, rounds, frames):
    w = Workload(4)
    cs = _contexts(kb, w.voxel_size)
    ident = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    for m in MODES:  # warm-up frames build every map (NEVER's is built under ALWAYS first)
        ctx, gm, code = cs[m]
        for _ in range(3):
            kb.RegisterFrame(gm, w.scan, np.zeros(0), ident, ident, w.true_pose, ident, w.tau, max_range=100.0, min_range=0.0, deskew=False,
                             voxel_size=w.voxel_size, want_clouds=False)
        ctx.set_map_update(code)
    times = {m: [] for m in MODES}
    for _ in range(rounds):
        for m in MODES:
            ctx, gm, _ = cs[m]
            for _ in range(frames):
                t0 = time.perf_counter()
                kb.RegisterFrame(gm, w.scan, np.zeros(0), ident, ident, w.true_pose, ident, w.tau, max_range=100.0, min_range=0.0,
                                 deskew=False, voxel_size=w.voxel_size, want_clouds=False)
                times[m].append(time.perf_counter() - t0)
    for ctx, gm, _ in cs.values():
        gm.close()
        ctx.close()
    return {m: 1e3 * float(np.median(times[m])) for m in MODES}, len(w.scan)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=30)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import kinematic_icp_b200 as kb
    from oracle import kicp_oracle_py as ko
    from oracle.workloads import Workload
    print("card:", card())
    gold, worst, n = golden(kb, ko, a.rounds)
    big, npts = cfg4(kb, Workload, a.rounds, a.frames)
    print(json.dumps({"golden_ms_per_frame": gold, "golden_frames": n, "never_vs_always_max_dt_m": worst[0],
                      "never_vs_always_max_rot_rad": worst[1], "cfg4_ms_per_frame": big, "cfg4_scan_points": npts}))


if __name__ == "__main__":
    main()
