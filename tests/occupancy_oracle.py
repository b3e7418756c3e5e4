"""The rule of occupancy evidence (include/kicp.h, kicp_map_set_occupancy) in numpy (test infrastructure).

The map is its export in block order, (keys, counts, points), with its first P voxels a frozen prior, and the evidence is one int per
voxel in the same order.  A clearing call counts every voxel's hits and misses as free_space_oracle.py does (its transform, voxel keys and
DDA), then applies step 5 with the evidence.  `carry` gives the evidence after a call that does not clear (an insert, an eviction): a
voxel that was in the map keeps its evidence, a new one starts at `initial`."""
import numpy as np

import free_space_oracle as F


def counts(ko, keys, voxel_size, max_distance, points, pose, origin, end_margin):
    """Steps 1-4 of the rule: (hits (nb,), misses (nb,), rays, visits) for the map's keys (nb, 3)."""
    keys = np.asarray(keys).reshape(-1, 3).astype(np.int64)
    nb = len(keys)
    o = F.transform(ko, pose, np.asarray(origin, dtype=np.float64).reshape(1, 3))[0]
    q = F.transform(ko, pose, points)
    kq = F.voxel_key(q, voxel_size)
    cast = np.zeros(len(q), bool) if (F.voxel_key(o, voxel_size) == F.INT_MIN).any() else ~(kq == F.INT_MIN).any(axis=1)
    ci = np.nonzero(cast)[0]
    where = {tuple(k): b for b, k in enumerate(keys.tolist())}

    def lookup(ks):
        return np.fromiter((where.get(tuple(k), -1) for k in ks.tolist()), np.int64, len(ks))

    hits = np.zeros(nb, np.int64)
    misses = np.zeros(nb, np.int64)
    hb = lookup(kq[ci])
    np.add.at(hits, hb[hb >= 0], 1)
    if len(ci):
        ray, vk = F.dda_visits(o, q[ci], voxel_size, end_margin, max_distance)
    else:
        ray, vk = np.zeros(0, np.int64), np.zeros((0, 3), np.int64)
    if len(vk):
        not_end = ~(vk == kq[ci][ray]).all(axis=1)
        uk, inv = np.unique(vk, axis=0, return_inverse=True)
        vb = lookup(uk)[inv.reshape(-1)]
        sel = not_end & (vb >= 0)
        np.add.at(misses, vb[sel], 1)
    return hits, misses, int(len(ci)), int(len(vk))


def clear(ko, voxels, evidence, prior_blocks, voxel_size, max_distance, points, pose, origin, end_margin, min_misses, occ):
    """One clearing call on the export `voxels` with `evidence` (None when occupancy is off) and occ = (initial, hit_gain, miss_loss,
    max_evidence).  Returns (the export after the call, the evidence after it (None when off), stats dict)."""
    keys, cnt, vpts = (np.asarray(a) for a in voxels)
    keys = keys.reshape(-1, 3)
    cnt = cnt.astype(np.int64)
    nb = len(cnt)
    hits, misses, rays, visits = counts(ko, keys, voxel_size, max_distance, points, pose, origin, end_margin)
    free = (misses >= min_misses) & (hits == 0)
    P = int(prior_blocks)
    live = np.arange(nb) >= P
    if evidence is None:
        cleared = free & live
        ev = None
    else:
        _, gain, loss, top = (int(v) for v in occ)
        ev = np.asarray(evidence, np.int64).copy()
        hit = live & (hits > 0)
        ev[hit] = np.minimum(ev[hit] + gain, top)
        dec = live & free
        ev[dec] -= loss
        cleared = dec & (ev <= 0)
        ev = ev[~cleared].astype(np.int32)
    keep_pts = np.repeat(~cleared, cnt)
    out = (keys[~cleared].astype(np.int32), cnt[~cleared].astype(np.int32), np.asarray(vpts, np.float64).reshape(-1, 3)[keep_pts])
    stats = dict(rays=rays, visits=visits, cleared_voxels=int(cleared.sum()), cleared_points=int(cnt[cleared].sum()),
                 prior_contradicted=int(free[:P].sum()))
    return out, ev, stats


def carry(before_keys, before_evidence, after_keys, initial):
    """The evidence after a call that does not clear: by key, a voxel of `before_keys` keeps its evidence, a new voxel gets `initial`."""
    where = {tuple(k): int(e) for k, e in zip(np.asarray(before_keys).reshape(-1, 3).tolist(), np.asarray(before_evidence).tolist())}
    return np.fromiter((where.get(tuple(k), int(initial)) for k in np.asarray(after_keys).reshape(-1, 3).tolist()), np.int32,
                       len(np.asarray(after_keys).reshape(-1, 3)))


def calls_to_clear(e, miss_loss):
    """the number of free calls a voxel at evidence e survives before the one that clears it: ceil(e / miss_loss) - 1"""
    return -(-int(e) // int(miss_loss)) - 1
