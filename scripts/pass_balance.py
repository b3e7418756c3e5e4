"""Load balance of the search phase, pass by pass (needs a -DKR_PROFILE build: KICP_LIB=kinematic-icp_b200/lib/ab/libkicp_prof.so).
For every pass: the end of the last window on each CTA, the windows that finish last (tasks, lines), and how well a window's task
and line counts predict its duration; plus the per-pass device timings of the same launch (ctx.last_timing(), all passes).
usage: python scripts/pass_balance.py [CFG [OUTDIR]]   -> OUTDIR/balance_cfgN.npy (raw window log; OUTDIR defaults to .) + a printed report"""
import os, sys, ctypes as C
sys.path.insert(0, "."); sys.path.insert(0, "kinematic-icp_b200/python")
import numpy as np
import torch
import kinematic_icp_b200 as kb
from kinematic_icp_b200 import _capi
from oracle import workloads as W

KR_WARPS = 8
cfg = int(sys.argv[1]) if len(sys.argv) > 1 else 4
outdir = sys.argv[2] if len(sys.argv) > 2 else "."
w = W.Workload(cfg)
ctx = kb.Context(0)
gm = kb.VoxelHashMap(ctx, w.voxel_size, w.max_range, w.max_points_per_voxel)
gm.load_voxels(*w.map.export_voxels())
reg = kb.KinematicRegistration()
scan = kb.Scan(ctx, w.N); scan.upload(w.scan)
res = kb.pinned_result()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
L = _capi.lib()
L.kicp_debug_window_log.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_int64, C.POINTER(C.c_int64)]
print("lib", os.environ.get("KICP_LIB", "default"), torch.cuda.get_device_name(0), flush=True)


def one(rep):
    flush.fill_(rep & 255); torch.cuda.synchronize()  # L2 flushed, as bench.py does before every step
    reg.enqueue(scan, gm, w.last_pose, w.rel_odom, w.tau, res)
    ctx.synchronize()
    out = np.zeros((65536, 4), dtype=np.uint64); n = C.c_int64(0)
    assert L.kicp_debug_window_log(ctx.h, out.ctypes.data_as(C.POINTER(C.c_uint64)), 65536, C.byref(n)) == 0
    return out[: n.value], np.array(ctx.last_timing())[: res.iterations] / 1e3


for rep in range(3):
    one(rep)
os.makedirs(outdir, exist_ok=True)
logs = []
for rep in range(5):
    log, tim = one(rep)
    logs.append(log)
    print("rep %d iterations %d  per pass [cert, its barrier, search, wait, reduce, solve] us:" % (rep, res.iterations))
    for p, row in enumerate(tim):
        print("   pass %d: %s" % (p, " ".join("%6.1f" % x for x in row)))
np.save(os.path.join(outdir, "balance_cfg%d.npy" % cfg), np.concatenate([np.c_[np.full(len(l), r, np.uint64), l] for r, l in enumerate(logs)]))

log = logs[-1]
t0 = log[:, 0].min()
ts = (log[:, 0] - t0).astype(np.float64) / 1e3; te = (log[:, 1] - t0).astype(np.float64) / 1e3
kind = (log[:, 2] >> np.uint64(56)).astype(int); it = ((log[:, 2] >> np.uint64(48)) & np.uint64(0xFF)).astype(int)
warp = (log[:, 2] & np.uint64(0xFFFFFFFF)).astype(int); cta = warp // KR_WARPS
a = (log[:, 3] >> np.uint64(32)).astype(np.int64); lines = (log[:, 3] & np.uint64(0xFFFFFFFF)).astype(np.int64)
tasks = a >> 8; npts = a & 0xFF
for p in range(1, int(it.max()) + 1):
    Wn = (kind == 0) & (it == p)
    if not Wn.any(): continue
    s0 = ts[Wn].min(); d = te[Wn] - ts[Wn]
    last = np.full(cta.max() + 1, np.nan); np.fmax.at(last, cta[Wn], te[Wn] - s0)
    last = last[~np.isnan(last)]
    print("pass %d: %d windows, pts/window %.1f, tasks/window %.1f, lines/window %.1f" % (p, Wn.sum(), npts[Wn].mean(), tasks[Wn].mean(), lines[Wn].mean()))
    print("   last window end per CTA (us after the phase starts): min %.1f p10 %.1f p50 %.1f p90 %.1f max %.1f" %
          tuple([last.min()] + [np.percentile(last, q) for q in (10, 50, 90)] + [last.max()]))
    print("   window duration: p10 %.1f p50 %.1f p90 %.1f max %.1f ; corr(dur, tasks) %.2f  corr(dur, lines) %.2f  corr(dur, pts) %.2f" %
          (np.percentile(d, 10), np.median(d), np.percentile(d, 90), d.max(), np.corrcoef(d, tasks[Wn])[0, 1], np.corrcoef(d, lines[Wn])[0, 1],
           np.corrcoef(d, npts[Wn])[0, 1]))
    for i in np.where(Wn)[0][np.argsort(te[Wn])[-8:]]:
        print("      finishes late: cta %3d start %.1f end %.1f dur %.1f pts %d tasks %d lines %d" % (cta[i], ts[i] - s0, te[i] - s0, te[i] - ts[i], npts[i], tasks[i], lines[i]))
gm.close()
