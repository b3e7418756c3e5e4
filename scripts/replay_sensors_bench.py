"""kicp_replay's frame rate on version-3 .kseq drives, on one GPU:

  kseq2      : one 131k-point 3D sensor (float32 x, y, z + float64 stamps relative to the header), as a version-2 drive
  kseq3      : the same records as a one-slot version-3 drive (the format path should cost nothing)
  3d+2scans  : that sensor plus two 1081-beam LaserScans, three slots
  segments N : that three-slot drive de-skewed along N + 1 odometry samples per frame (N = 1, 10, 64 segments)

A 12-frame drive of the synthetic world (the oracle's synth_scan, a planar path that turns and brakes), de-skew on.  Each run is one
kicp_replay process with --repeat 3 and reports its fastest repetition after the first; the drives alternate for --rounds rounds and
each figure is the fastest round.  Prints one JSON line with the card's name and power limit.

    python scripts/replay_sensors_bench.py [--frames 12] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "kinematic-icp_b200", "python")):
    sys.path.insert(0, p)
EXE = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import kseq2
    import kseq3 as K
    from oracle import kicp_oracle_py as ko
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    rng = np.random.default_rng(0)
    period = 0.1
    traj = K.trajectory(ko, period * args.frames, 1)
    l2bs = [ko.se3_exp([0.8, 0.0, 0.3, 0.0, 0.0, 0.0]), ko.se3_exp([-0.8, 0.1, 0.3, 0.0, 0.0, np.pi]), ko.se3_exp([0.0, 0.4, 0.5, 0.0, 0.0, 1.5])]
    slots = [(K.RECORDS, 1, l2bs[0]), (K.LASER_SCAN, 0, l2bs[1]), (K.LASER_SCAN, 0, l2bs[2])]
    frames = []
    for f in range(args.frames):
        t0 = period * f
        pts = K.world_3d(ko, traj, l2bs[0], t0 + period, 7 * f, beams=64, n_az=2048)
        msgs = [K.records_message(pts, rng.uniform(0.0, period, len(pts)), t0)]
        for i in (1, 2):
            msgs.append(K.scan_message(rng.uniform(0.2, 30.0, 1081).astype(np.float32), t0 + 0.01 * i, time_increment=period / 1081))
        frames.append(dict(odom=ko.IDENTITY.copy(), samples=[], messages=msgs))
    one = [dict(fr, messages=fr["messages"][:1]) for fr in frames]
    with tempfile.TemporaryDirectory() as d:
        path = lambda name: os.path.join(d, name + ".kseq")  # noqa: E731
        one = K.with_samples(ko, traj, slots[:1], one, 0)
        kseq2.write_kseq2(path("kseq2"), l2bs[0], ko.IDENTITY, [(m["records"], m["point_step"], m["offsets"], m["stamp_datatype"],
                                                               m["stamp_offset"], m["header"], fr["odom"]) for fr in one
                                                              for m in fr["messages"]])
        K.write_kseq3(path("kseq3"), ko.IDENTITY, slots[:1], one)
        K.write_kseq3(path("3d+2scans"), ko.IDENTITY, slots, K.with_samples(ko, traj, slots, frames, 0))
        runs = ["kseq2", "kseq3", "3d+2scans"]
        for n in (1, 10, 64):
            K.write_kseq3(path("segments %d" % n), ko.IDENTITY, slots, K.with_samples(ko, traj, slots, frames, n + 1))
            runs.append("segments %d" % n)
        best, lines = {}, {}
        for _ in range(args.rounds):
            for name in runs:
                r = subprocess.run([EXE, path(name), os.path.join(d, "out.tum"), "--repeat", "3"], capture_output=True, text=True,
                                   check=True)
                j = json.loads(r.stdout.strip().splitlines()[-1])
                best.setdefault(name, []).append(j["frames_per_s_best"])
                lines[name] = j
    result = {"harness": "scripts/replay_sensors_bench.py", "gpu": gpu, "frames": args.frames, "rounds": args.rounds, "drives": []}
    for name in runs:
        j = lines[name]
        result["drives"].append({"name": name, "frames_per_s_rounds": best[name], "frames_per_s": max(best[name]),
                                 "points_per_frame": j["points_per_frame"], "slot_kinds": j.get("slot_kinds"),
                                 "odometry_samples_per_frame": j.get("odometry_samples_per_frame", 0)})
    print(json.dumps(result))


if __name__ == "__main__":
    main()
