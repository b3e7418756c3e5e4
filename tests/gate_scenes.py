"""Scenes on the registration kernel's gate and on its non-finite inputs (test infrastructure, shared by
tests/test_gate_emu_cpu.py and tests/test_gpu_gate.py), built with the helpers of tests/scenes.py.

The gate of Registration.cpp:75, (neighbor - query).norm() < tau: the reference's norm is sqrt((dx dx + dy dy) + dz dz), every
operation rounded.  A kernel that squares r with an FMA sees another square in the last bit or two, and a point whose norm is
within an ulp of tau may then fall on the other side.  The gate scenes are made of such points: every query has exactly one map
point in its 27 voxels, at a reference norm of exactly prev(tau), tau or next(tau)."""
import math

import numpy as np

from scenes import (FAR, IDENTITY, INF, Scene, _dyadic, _lattice, _oracle_map, _scan_for, floor_key, map_shape, ref_sq, rotated_prior,
                    with_nonfinite)

def _fast_fma():
    f = getattr(math, "fma", None)  # (Python >= 3.13)
    if f is None:
        import ctypes
        import ctypes.util
        f = ctypes.CDLL(ctypes.util.find_library("m")).fma
        f.restype, f.argtypes = ctypes.c_double, [ctypes.c_double] * 3
    return f


FMA = _fast_fma()  # one rounding of a b + c (correctly rounded, as _fma; checked against it by the gate tests)

# every contraction of (dx dx + dy dy) + dz dz a compiler may choose, by the products it fuses (nvcc and GCC: x, then z)
CONTRACTIONS = {
    "x": lambda x, y, z: FMA(x, x, y * y) + z * z,
    "y": lambda x, y, z: FMA(y, y, x * x) + z * z,
    "z": lambda x, y, z: FMA(z, z, x * x + y * y),
    "x,z": lambda x, y, z: FMA(z, z, FMA(x, x, y * y)),
    "y,z": lambda x, y, z: FMA(z, z, FMA(y, y, x * x)),
}


def gate_flips(c, q, tau):
    """The contractions (keys of CONTRACTIONS) under which the pair (c, q) would be gated otherwise than the reference gates it."""
    dx, dy, dz = float(c[0]) - float(q[0]), float(c[1]) - float(q[1]), float(c[2]) - float(q[2])
    accept = math.sqrt(ref_sq(c, q)) < tau
    return [k for k, f in CONTRACTIONS.items() if (math.sqrt(f(dx, dy, dz)) < tau) != accept]


def _gate_point(rng, q, u, t, tau, vs, f, want, tries=24):
    """A map point c in q's 27 voxels with sqrt(ref_sq(c, q)) == t exactly, roughly in direction u.  The two axes other than f
    take their share of t first; c[f] is then solved for and walked ulp by ulp onto t (|q[f]| <= |c[f] - q[f]|, so an ulp of c[f]
    moves the square by about an ulp at most).  Among such points, one that the contraction `want` gates otherwise than the
    reference is preferred; `tries` jittered directions are looked at."""
    q = np.asarray(q, dtype=np.float64)
    qv = [floor_key(x, vs) for x in q]
    o = [a for a in range(3) if a != f]
    ks = np.arange(-64, 65, dtype=np.float64)
    first = None
    for k in range(tries):
        v = u + (0.02 * rng.normal(size=3) if k else 0.0)
        v = v / np.linalg.norm(v)
        c = q + t * v
        d = c - q
        s = d[o[0]] * d[o[0]] + d[o[1]] * d[o[1]]
        if s >= t * t:
            continue
        cf = q[f] + math.copysign(math.sqrt(t * t - s), v[f])
        cand = np.repeat(c[None], len(ks), 0)
        cand[:, f] = cf + ks * math.ulp(cf)
        dd = cand - q
        sq = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
        for j in np.flatnonzero(np.sqrt(sq) == t):
            cj = cand[j]
            if any(abs(floor_key(cj[a], vs) - qv[a]) > 1 for a in range(3)) or math.sqrt(ref_sq(cj, q)) != t:
                continue
            if first is None:
                first = cj.copy()
            if want is None or want in gate_flips(cj, q, tau):
                return cj.copy()
    return first


def _gate_offset(rng, t, vs, f, crossed):
    """(direction u, q's position): u[f] carries 30 to 58 % of t, no axis more than 1.9 voxels; q + t u leaves q's voxel along
    the axes in `crossed` (and along any it cannot stay within), into a neighbouring voxel.  Along the other axes the position is
    in voxels within q's lattice voxel; along f it is relative to the voxel face at 0, and |q[f]| <= |t u[f]|."""
    while True:
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        if 0.3 <= abs(u[f]) <= 0.577 and np.all(np.abs(t * u) < 1.9 * vs):
            break
    pos = np.empty(3)
    for a in range(3):
        da = t * u[a] / vs  # the offset in voxels along a; positions for da > 0, mirrored for da < 0
        m = abs(da)
        cross = a in crossed or m >= 1.0
        if a == f:
            lo, hi = (max(-1.0, -m), min(0.0, 1.0 - m)) if cross else (0.0, min(1.0 - m, 0.5 * m))
        else:
            lo, hi = (max(0.0, 1.0 - m), min(1.0, 2.0 - m)) if cross else (0.0, 1.0 - m)
        p = lo + (hi - lo) * rng.uniform(0.05, 0.95)
        pos[a] = p if da > 0 else (-p if a == f else 1.0 - p)
    return u, pos


def gate_scene(ko, tau, vs, n=300, rotated=False, origin=None, f32=False, seed=21, cap=20, **kw):
    """n queries, each alone with one map point in its 27 voxels at a reference norm of exactly prev(tau), tau or next(tau) (in
    turn), the point in q's own voxel or across a face, an edge or a corner (in turn, where tau / vs allows).  Query i has its
    fine axis f = i mod 3 near 0 (with `origin`: z, the others far out) and sits on the lattice of the other two axes, 4 voxels or
    more from 0 and from each other.  Points are chosen to flip under each of CONTRACTIONS in turn; `traps` is the smallest count
    over the contractions.  rotated: the prior of rotated_prior(); origin: the identity rotation and the translation `origin`
    (queries far out, q = p + t rounds); f32: float32-representable scan, identity prior."""
    rng = np.random.default_rng(seed)
    if rotated:
        last, odom = rotated_prior(ko, rng)
    elif origin is not None:
        last, odom = np.r_[0.0, 0.0, 0.0, 1.0, origin], IDENTITY.copy()
    else:
        last, odom = IDENTITY.copy(), IDENTITY.copy()
    lattice = np.array([-20, -16, -12, -8, -4, 4, 8, 12, 16, 20])
    prev_t, next_t = np.nextafter(tau, 0.0), np.nextafter(tau, INF)
    plan, local = [], []
    for i in range(n):
        f = 2 if origin is not None else i % 3
        j = i if origin is not None else i // 3
        o = [a for a in range(3) if a != f]
        cls = (i // 3) % 4  # own voxel, face, edge, corner
        crossed = list(rng.permutation(3)[:cls])
        u, pos = _gate_offset(rng, [prev_t, tau, next_t][i % 3], vs, f, crossed)
        v = np.zeros(3)
        v[o[0]], v[o[1]] = lattice[j % 10], lattice[(j // 10) % 10] + (0 if j < 100 else 4 * 11 * (j // 100))
        x = (v + pos) * vs
        if f32:
            x = _dyadic(x, 2.0 ** -16)
        plan.append((f, u, [prev_t, tau, next_t][i % 3]))
        local.append(x)
    local = np.array(local)
    scan, qs = _scan_for(ko, local, last, odom) if origin is None else (local, None)
    if origin is not None:
        qs = ko.se3_transform(ko.se3_compose(last, odom), scan)
    if f32:
        assert np.array_equal(scan.astype(np.float32).astype(np.float64), scan)
    flips = {k: 0 for k in CONTRACTIONS}
    pts, classes = [], [0] * 4
    for i, (q, (f, u, t)) in enumerate(zip(qs, plan)):
        want = min(flips, key=flips.get)  # the contraction with the fewest flips so far
        c = _gate_point(rng, q, u, t, tau, vs, f, want)
        assert c is not None, "no point at norm %r from query %d" % (t, i)
        for k in gate_flips(c, q, tau):
            flips[k] += 1
        shift = tuple(floor_key(c[a], vs) - floor_key(q[a], vs) for a in range(3))
        classes[sum(s != 0 for s in shift)] += 1
        pts.append(c)
    pts = np.array(pts)
    om = _oracle_map(ko, vs, cap, pts)
    name = "gate-tau%g-vs%g%s%s%s" % (tau, vs, "-rotated" if rotated else "", "-far" if origin is not None else "", "-f32" if f32 else "")
    sc = Scene(name, om, scan.astype(np.float32) if f32 else scan, last, odom, tau, traps=min(flips.values()), **kw)
    sc.flips, sc.classes, sc.cands = flips, classes, pts
    # the reference's N of the first pass, counted here: every query's only candidate, gated by its norm
    sc.expected_n = sum(int(math.sqrt(ref_sq(c, q)) < tau) for c, q in zip(pts, qs))
    return sc


def dyadic_gate_scene(ko, k=-4, vs=1.0, above=False, n=96, **kw):
    """Exact gate cases: offsets (3, 4, 12) 2^k, every permutation and sign, at norm exactly 13 2^k, and half as far, from dyadic
    queries.  tau = 13 2^k rejects the far ones (the gate is a strict <), tau = next(13 2^k) (`above`) accepts them.  Every
    square is exact, so no contraction changes a decision here: this is the strictness of the gate."""
    import itertools
    base = np.array([3.0, 4.0, 12.0]) * 2.0 ** k
    offs = [np.array(p) * s for p in itertools.permutations(base) for s in itertools.product((1, -1), repeat=3)]
    tau = 13.0 * 2.0 ** k
    if above:
        tau = float(np.nextafter(tau, INF))
    assert 12.0 * 2.0 ** k < vs
    qs, pts = [], []
    for i in range(n):
        q = (_lattice(i) + 0.5) * vs
        d = offs[i % len(offs)] * (0.5 if i % 2 else 1.0)
        qs.append(q)
        pts.append(q + d)
    qs, pts = np.array(qs), np.array(pts)
    om = _oracle_map(ko, vs, 20, pts)
    sc = Scene("gate-dyadic-13x2^%d%s" % (k, "-next" if above else ""), om, qs, IDENTITY.copy(), IDENTITY.copy(), tau, **kw)
    sc.expected_n = sum(int(math.sqrt(ref_sq(c, q)) < tau) for c, q in zip(pts, qs))
    assert sc.expected_n == (n if above else n // 2)
    sc.flips, sc.cands = None, pts
    return sc


def gate_scenes(ko):
    """The gate scenes of the suite: tau 0.05 / 0.3 / 1.0 / 2.9 on voxels of 0.5 / 0.37 / 1.0, the rotated prior, queries near
    (4.2e5, 5.8e6, 0), a float32 scan; adaptive and fixed regularisation; and the exact (3, 4, 12) 2^k cases.  One pass each
    (max_iter 1): only the first pass's N is defined bit for bit."""
    fixed = dict(max_iter=1, adaptive=False, fixed_reg=0.5)
    return [gate_scene(ko, 0.05, 0.5, max_iter=1), gate_scene(ko, 0.3, 0.37, seed=22, **fixed),
            gate_scene(ko, 1.0, 1.0, seed=23, max_iter=1), gate_scene(ko, 0.3, 0.5, rotated=True, seed=24, max_iter=1),
            gate_scene(ko, 0.3, 1.0, origin=(4.2e5, 5.8e6, 0.0), seed=25, max_iter=1),
            gate_scene(ko, 1.0, 1.0, f32=True, seed=26, **fixed), gate_scene(ko, 2.9, 1.0, seed=27, max_iter=1),
            dyadic_gate_scene(ko, max_iter=1), dyadic_gate_scene(ko, above=True, max_iter=1)]


def nonfinite_reg_scenes(ko):
    """Registrations with NaN, +-Inf and +-3e9 vs among the scan points (the rows of nonfinite_rows()) and in the map, where voxels
    (INT_MIN, 0, 0) and (INT_MIN, INT_MIN, INT_MIN) get a NaN first point — the reference's min_element then returns that point,
    so the whole voxel hides.  Full IRLS runs (every pass's N is defined: no point sits on a decision).  The last scene gates with
    tau = 1e12, and the INT_MIN voxel's first point is -3e9 vs: the +huge queries are accepted against it.  Its residuals are of
    the order of 1e9, so only the first pass's N and sums are held to the oracle."""
    out = []
    for vs, cap, seed in ((0.75, 24, 7), (0.6, 25, 8)):
        base = map_shape(ko, vs, cap, seed=seed)
        pts = with_nonfinite(base.om.export_voxels()[2], vs, seed=seed)
        om = ko.OracleMap(vs, FAR, cap)
        om.add_points(pts)
        scan = with_nonfinite(base.scan, vs, seed=seed + 1)
        out.append(Scene("nonfinite-vs%g-cap%d" % (vs, cap), om, scan, base.last, base.odom, base.tau, max_iter=10))
    vs = 0.75
    base = map_shape(ko, vs, 24)
    huge = np.array([[-3e9 * vs, -3e9 * vs, -3e9 * vs], [-3e9 * vs, 0.1, 0.1]])
    om = ko.OracleMap(vs, FAR, 24)
    om.add_points(np.concatenate([huge, with_nonfinite(base.om.export_voxels()[2], vs, seed=34)]))
    scan = with_nonfinite(base.scan, vs, seed=35)
    out.append(Scene("nonfinite-tau1e12", om, scan, base.last, base.odom, 1e12, max_iter=1, huge=True))
    return out
