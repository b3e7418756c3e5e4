"""The rule of free-space clearing (include/kicp.h, kicp_map_clear_free_space) in vectorised numpy (test infrastructure).

The map is given as its export in block order, (keys, counts, points), with its first P voxels a frozen prior (prior_map_oracle.py).
Every cast ray is traversed by the DDA of the rule, one step of all rays at a time; a ray visits each voxel at most once, so the misses
of a voxel are the number of visits to it by rays that do not end in it.  The result is the export with the cleared live voxels
removed (the others in their order) and the statistics (rays, visits, cleared_voxels, cleared_points, prior_contradicted)."""
import numpy as np

INT_MIN = -(1 << 31)


def voxel_key(x, voxel_size):
    """the map's voxel key per axis: floor(x / v), INT_MIN for a non-finite value or a floor outside [-2^31, 2^31)"""
    f = np.floor(np.asarray(x, dtype=np.float64) / voxel_size)
    with np.errstate(invalid="ignore"):
        ok = (f >= -2147483648.0) & (f < 2147483648.0)
    return np.where(ok, np.where(ok, f, 0.0).astype(np.int64), INT_MIN)


def transform(ko, pose, pts):
    """T * p by the oracle's Sophus transform (kicp_map_update_pose's bits)"""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    if len(pts) == 0:
        return pts.copy()
    return np.asarray(ko.se3_transform(np.asarray(pose, dtype=np.float64), pts), dtype=np.float64).reshape(-1, 3)


def dda_visits(o, q, voxel_size, end_margin, max_distance):
    """The traversal of step 4 for rays from the point o (3,) to the points q (n, 3), every ray assumed cast.  Returns (ray index,
    visited key (m, 3)) of every visit, in traversal order per ray."""
    o = np.asarray(o, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64).reshape(-1, 3)
    v = float(voxel_size)
    ko = voxel_key(o, v)
    kq = voxel_key(q, v)
    d = q - o
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        L = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        cut = L - end_margin
        t_end = np.where(cut < max_distance, cut, max_distance) / L
        live = (L != 0.0) & (t_end > 0.0)
        k = np.broadcast_to(ko, d.shape).copy()
        kf = k.astype(np.float64)
        step = np.where(d > 0, 1, np.where(d < 0, -1, 0)).astype(np.int64)
        tmax = np.where(d > 0, ((kf + 1.0) * v - o) / d, np.where(d < 0, (kf * v - o) / d, np.inf))
        tdelta = np.where(d > 0, v / d, np.where(d < 0, -v / d, 0.0))
    steps = np.abs(kq - ko).sum(axis=1)
    rays, keys = [], []
    idx = np.nonzero(live)[0]
    rays.append(idx)
    keys.append(k[idx].copy())
    s = 0
    while len(idx):
        idx = idx[steps[idx] > s]
        if not len(idx):
            break
        tm = tmax[idx]
        j = np.argmin(tm, axis=1)  # the first minimum: the lowest index on ties
        tj = tm[np.arange(len(idx)), j]
        go = tj < t_end[idx]
        idx, j = idx[go], j[go]
        k[idx, j] += step[idx, j]
        tmax[idx, j] += tdelta[idx, j]
        rays.append(idx)
        keys.append(k[idx].copy())
        s += 1
    return np.concatenate(rays).astype(np.int64), np.concatenate(keys).reshape(-1, 3)


def clear_free_space(ko, voxels, prior_blocks, voxel_size, max_distance, points, pose, origin, end_margin, min_misses):
    """The rule on a map export `voxels` = (keys, counts, points) whose first `prior_blocks` voxels are prior.  Returns (the export
    after the call, stats dict)."""
    keys, counts, vpts = (np.asarray(a) for a in voxels)
    keys = keys.reshape(-1, 3).astype(np.int64)
    counts = counts.astype(np.int64)
    nb = len(counts)
    o = transform(ko, pose, np.asarray(origin, dtype=np.float64).reshape(1, 3))[0]
    q = transform(ko, pose, points)
    ko_key = voxel_key(o, voxel_size)
    kq = voxel_key(q, voxel_size)
    cast = np.zeros(len(q), bool) if (ko_key == INT_MIN).any() else ~(kq == INT_MIN).any(axis=1)
    ci = np.nonzero(cast)[0]
    where = {tuple(k): b for b, k in enumerate(keys.tolist())}

    def lookup(ks):
        return np.fromiter((where.get(tuple(k), -1) for k in ks.tolist()), np.int64, len(ks))

    hits = np.zeros(nb, np.int64)
    misses = np.zeros(nb, np.int64)
    hb = lookup(kq[ci])
    np.add.at(hits, hb[hb >= 0], 1)
    ray, vk = dda_visits(o, q[ci], voxel_size, end_margin, max_distance) if len(ci) else (np.zeros(0, np.int64), np.zeros((0, 3), np.int64))
    not_end = ~(vk == kq[ci][ray]).all(axis=1)
    if len(vk):
        uk, inv = np.unique(vk, axis=0, return_inverse=True)
        vb = lookup(uk)[inv.reshape(-1)]
        sel = not_end & (vb >= 0)
        np.add.at(misses, vb[sel], 1)
    free = (misses >= min_misses) & (hits == 0)
    P = int(prior_blocks)
    cleared = free.copy()
    cleared[:P] = False
    keep_pts = np.repeat(~cleared, counts)
    out = (keys[~cleared].astype(np.int32), counts[~cleared].astype(np.int32), np.asarray(vpts, np.float64).reshape(-1, 3)[keep_pts])
    stats = dict(rays=int(len(ci)), visits=int(len(vk)), cleared_voxels=int(cleared.sum()), cleared_points=int(counts[cleared].sum()),
                 prior_contradicted=int(free[:P].sum()))
    return out, stats


def brute_visits(o, q, voxel_size, end_margin, max_distance, pad=1):
    """Every voxel whose closed cube the segment o + t (q - o), t in [0, t_end], meets: the slab test over the voxels of the segment's
    bounding box.  For rays whose coordinates stay away from voxel faces this is the DDA's visit set."""
    o, q = np.asarray(o, float), np.asarray(q, float)
    d = q - o
    L = np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    cut = L - end_margin
    t_end = min(cut, max_distance) / L
    if L == 0 or not t_end > 0:
        return set()
    e = o + t_end * d
    lo = np.floor(np.minimum(o, e) / voxel_size).astype(int) - pad
    hi = np.floor(np.maximum(o, e) / voxel_size).astype(int) + pad
    out = set()
    for x in range(lo[0], hi[0] + 1):
        for y in range(lo[1], hi[1] + 1):
            for z in range(lo[2], hi[2] + 1):
                k = np.array([x, y, z], float)
                t0, t1 = 0.0, t_end
                ok = True
                for j in range(3):
                    a, b = k[j] * voxel_size, (k[j] + 1) * voxel_size
                    if d[j] == 0:
                        if not (a <= o[j] <= b):
                            ok = False
                            break
                    else:
                        u, w = (a - o[j]) / d[j], (b - o[j]) / d[j]
                        t0, t1 = max(t0, min(u, w)), min(t1, max(u, w))
                if ok and t0 < t1:
                    out.add((x, y, z))
    return out
