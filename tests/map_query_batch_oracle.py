"""The pose search's oracle (tests/pose_search_oracle.py) vectorised over hypotheses (test infrastructure, shared by
tests/test_map_query_batch_oracle_cpu.py and tests/test_gpu_map_query_scale.py), for lattices of millions of hypotheses or scans of
hundreds of thousands of points, where PO.search's one pose and one kernel_sum per hypothesis in Python is too slow.  The same
arithmetic in the same order: one rotation per yaw (PO.rotation) and one translation per (x, y) (PO.translation), the query points
R p + t in quat_rotate's order, one om.nearest over all queries of a yaw, kernel_sum batched over hypotheses, and the ranking by
PO.key through np.lexsort.  Counts, kernel-order sums and the kept lists are therefore PO.search's bit for bit."""
import numpy as np

import pose_search_oracle as PO


def quat_rotate(q, p):
    """R_q p for q = (x, y, z, w) and p (..., 3), in kicp_device.cuh quat_rotate's operation order"""
    qx, qy, qz, qw = (float(v) for v in q)
    px, py, pz = p[..., 0], p[..., 1], p[..., 2]
    with np.errstate(invalid="ignore", over="ignore"):  # non-finite points stay non-finite, as on the device
        ux, uy, uz = qy * pz - qz * py, qz * px - qx * pz, qx * py - qy * px
        ux, uy, uz = ux + ux, uy + uy, uz + uz
        return np.stack([px + qw * ux + (qy * uz - qz * uy), py + qw * uy + (qz * ux - qx * uz), pz + qw * uz + (qx * uy - qy * ux)],
                        -1)


def kernel_sums(v):
    """PO.kernel_sum of every row of v (H, n): thread t adds points t, t + 256, ... in turn; lane l adds threads l, l + 32, ...,
    l + 224; then the xor tree over the 32 lanes, read on lane 0"""
    v = np.asarray(v, dtype=np.float64)
    H, n = v.shape
    rows = np.concatenate([v, np.zeros((H, -n % PO.THREADS))], 1).reshape(H, -1, PO.THREADS)
    per = np.zeros((H, PO.THREADS))
    for r in range(rows.shape[1]):
        per = per + rows[:, r]
    lanes = np.zeros((H, 32))
    for k in range(PO.THREADS // 32):
        lanes = lanes + per[:, 32 * k:32 * k + 32]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0].copy()


def score(ko, om, src, prior, u, Ls, tau, max_queries=1 << 22):
    """(n_inliers, kernel-order sum_sq, plain sum_sq) arrays of the lattice points Ls (H, 3): PO.score_many of their PO.pose"""
    src = np.ascontiguousarray(src, dtype=np.float64).reshape(-1, 3)
    Ls = np.asarray(Ls, dtype=np.int64).reshape(-1, 3)
    H, n = len(Ls), len(src)
    cnt, ssq, plain = np.zeros(H, np.int64), np.zeros(H), np.zeros(H)
    if n == 0 or H == 0:
        return cnt, ssq, plain
    prior = np.asarray(prior, dtype=np.float64)
    xy, t_of = np.unique(Ls[:, :2], axis=0, return_inverse=True)
    trans = np.array([PO.translation(prior, int(ix) * u[0], int(iy) * u[1]) for ix, iy in xy])
    yaws, r_of = np.unique(Ls[:, 2], return_inverse=True)
    step = max(1, max_queries // n)
    for r, ipsi in enumerate(yaws):
        rs = quat_rotate(PO.rotation(prior, int(ipsi) * u[2]), src)
        hyp = np.flatnonzero(r_of.reshape(-1) == r)
        for b in range(0, len(hyp), step):
            h = hyp[b:b + step]
            q = rs[None, :, :] + trans[t_of.reshape(-1)[h]][:, None, :]
            _, d = om.nearest(q.reshape(-1, 3))
            d = d.reshape(len(h), n)
            inl = d < tau
            dd = np.where(inl, d, 0.0)
            sq = dd * dd
            cnt[h] = inl.sum(1)
            ssq[h] = kernel_sums(sq)
            plain[h] = sq.sum(1)
    return cnt, ssq, plain


def rank(Ls, cnt, ssq):
    """indices of the hypotheses in PO.key order (best first)"""
    L = np.asarray(Ls, dtype=np.int64).reshape(-1, 3)
    return np.lexsort((L[:, 1], L[:, 0], L[:, 2], L[:, 0] * L[:, 0] + L[:, 1] * L[:, 1], np.abs(L[:, 2]), ssq, -cnt))


def level0(half_extent, step, levels):
    """level 0's lattice points in PO.search's order"""
    k, scale, _ = PO.plan(half_extent, step, levels)
    ip, ix, iy = np.meshgrid(*[np.arange(-k[a], k[a] + 1) * scale for a in (2, 0, 1)], indexing="ij")
    return np.stack([ix.reshape(-1), iy.reshape(-1), ip.reshape(-1)], 1)


def search(ko, om, src, prior, tau, half_extent, step, levels, keep):
    """PO.search's result for the kept hypotheses: dict(kept, level_kept, n_scored, u, and scores {L: (n, sum_sq, plain, level)} of
    every lattice point kept at some level)"""
    k, scale, u = PO.plan(half_extent, step, levels)
    L0 = level0(half_extent, step, levels)
    c0, s0, p0 = score(ko, om, src, prior, u, L0, tau)
    Ls, cnt, ssq, plain, lev = [L0], [c0], [s0], [p0], [np.zeros(len(L0), np.int64)]
    refined = set()

    def best():
        L, c, s = np.concatenate(Ls), np.concatenate(cnt), np.concatenate(ssq)
        return rank(L, c, s)[:keep]

    def at(i):
        j = int(i)
        for a, L in enumerate(Ls):
            if j < len(L):
                return tuple(int(x) for x in L[j]), int(cnt[a][j]), float(ssq[a][j]), float(plain[a][j]), int(lev[a][j])
            j -= len(L)

    def in0(L):
        return all(L[a] % scale == 0 and abs(L[a]) <= k[a] * scale for a in range(3))

    kept = [at(i) for i in best()]
    level_kept = [[e[0] for e in kept]]
    scores = {e[0]: e[1:] for e in kept}
    for level in range(1, levels):
        s = 2 ** (levels - 1 - level)
        kids = []
        for e in kept:
            c = e[0]
            for dp in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    for dy in (-1, 0, 1):
                        L = (c[0] + dx * s, c[1] + dy * s, c[2] + dp * s)
                        if (dp or dx or dy) and not in0(L) and L not in refined:
                            refined.add(L)
                            kids.append(L)
        if kids:
            ck, sk, pk = score(ko, om, src, prior, u, kids, tau)
            Ls.append(np.array(kids, dtype=np.int64)), cnt.append(ck), ssq.append(sk), plain.append(pk)
            lev.append(np.full(len(kids), level, np.int64))
        kept = [at(i) for i in best()]
        level_kept.append([e[0] for e in kept])
        scores.update({e[0]: e[1:] for e in kept})
    return dict(kept=[(e[0], e[1], e[2], e[4]) for e in kept], scores=scores, level_kept=level_kept, n_scored=len(L0) + len(refined), u=u)
