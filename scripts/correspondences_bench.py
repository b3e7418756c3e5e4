"""The correspondence report, timed on one GPU.

1. Per-frame time of kicp_register_frame with option "correspondences" 0 and 1, on two contexts driven with the same frames in
   alternated rounds: cfg4's scan (261 675 points) and its first half (~131k points), registered frame after frame at the pose that
   scan was taken from, after warm-up frames that built each map.  Host clock around each call (the call ends in its synchronisation).
2. kicp_map_correspondences_device_async on cfg4 (its 261 675 scan points at the prior against its 1 001 499-point map): CUDA events
   around each call on the context stream, per-point outputs and the statistics in device memory.

Prints the card's name and power limit (read in the same run) and one JSON line.

    python scripts/correspondences_bench.py [--frames 30] [--warmup 5] [--calls 200]
"""
import argparse
import json
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


def frame_times(kb, scan, frames, warmup):
    """median / p90 per-frame ms with the option off and on (alternated frame by frame), and the last on-frame's statistics"""
    ctxs = [kb.Context(0), kb.Context(0)]
    ctxs[1].set_option("correspondences", 1)
    maps = [kb.VoxelHashMap(c, 1.0, 100.0, 20) for c in ctxs]
    ident = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    times = [[], []]
    poses = [ident.copy(), ident.copy()]
    for k in range(warmup + frames):
        for j in (0, 1) if k % 2 == 0 else (1, 0):
            t0 = time.perf_counter()
            pose, nf, ns, _ = kb.RegisterFrame(maps[j], scan, np.zeros(0), ident, ident, poses[j], ident, 1.0, deskew=False, want_clouds=False)
            dt = (time.perf_counter() - t0) * 1e3
            poses[j] = pose
            if k >= warmup:
                times[j].append(dt)
    st = kb.frame_correspondences(ctxs[1])
    for m in maps:
        m.close()
    for c in ctxs:
        c.close()
    q = lambda t, p: float(np.percentile(t, p))
    return dict(points=len(scan), source=int(ns), off_ms=q(times[0], 50), on_ms=q(times[1], 50), off_p90_ms=q(times[0], 90),
                on_p90_ms=q(times[1], 90), delta_us=1e3 * (q(times[1], 50) - q(times[0], 50)), fitness=st.fitness, n_inliers=st.n_inliers)


def standalone(kb, w, calls):
    import torch
    from kinematic_icp_b200 import _capi
    ctx = kb.Context(0)
    gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
    gm.load_voxels(*w.map.export_voxels())
    src = torch.from_numpy(np.ascontiguousarray(w.scan)).cuda()
    n = len(src)
    pts, dist = torch.empty((n, 3), dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda")
    inl, stats = torch.empty(n, dtype=torch.uint8, device="cuda"), torch.empty(10, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    pose = _capi.as_pose(w.prior)
    L = _capi.lib()
    stream = torch.cuda.ExternalStream(ctx.stream)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def call():
        _capi.check(L.kicp_map_correspondences_device_async(gm.h, src.data_ptr(), n, _capi.KICP_DTYPE_F64, 0, 0, 0, 0, _capi.dp(pose),
                                                            float(w.tau), pts.data_ptr(), dist.data_ptr(), inl.data_ptr(),
                                                            stats.data_ptr()), "kicp_map_correspondences_device_async")

    for _ in range(10):
        call()
    ctx.synchronize()
    ev[0].record(stream)
    for _ in range(calls):
        call()
    ev[1].record(stream)
    ev[1].synchronize()
    us = ev[0].elapsed_time(ev[1]) * 1e3 / calls
    n_inl = int(inl.sum().item())
    gm.close()
    ctx.close()
    return dict(points=n, map_points=int(w.map.num_points()), us_per_call=us, n_inliers=n_inl)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--calls", type=int, default=200)
    a = ap.parse_args()
    import kinematic_icp_b200 as kb
    from oracle import workloads as W
    w = W.Workload(4)
    name = card()
    print("card:", name, flush=True)
    out = {"card": name, "frames": []}
    for scan in (np.ascontiguousarray(w.scan[: len(w.scan) // 2]), np.ascontiguousarray(w.scan)):
        r = frame_times(kb, scan, a.frames, a.warmup)
        print(r, flush=True)
        out["frames"].append(r)
    out["standalone_cfg4"] = standalone(kb, w, a.calls)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
