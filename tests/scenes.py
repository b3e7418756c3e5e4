"""Scenes that probe the registration kernel's nearest-neighbour choice (test infrastructure, shared by the emulator tests and the
GPU tests).

The reference picks, per query q, the map point c with the smallest (c - q).norm() = sqrt((dx dx + dy dy) + dz dz) under a strict
<: the first in the 27-voxel visiting order, the first in insertion order inside a voxel.  Its query is Sophus' quaternion
formula.  A kernel that squares with an FMA, or forms q from a rotation matrix, sees other last bits; where two candidates are at
(nearly) the same distance it may then take the other one.  Smooth synthetic scenes hold no such ties: these scenes are made of
them, and of the map shapes the workloads never use (non-power-of-two voxel sizes, full voxels of many points, maps far from the
origin).

Every builder returns a Scene: the map as an oracle map in the reference's insertion order (`voxels`: the same map as the
voxel-grouped arrays the device loads), a scan, the last pose and the odometry, tau and the solver settings.  Tie scenes count
their `traps`: the queries at which a kernel that squares with an FMA (fma(dz,dz, fma(dy,dy, dx*dx))) would pick another point
than the reference, so that a test can insist the scene keeps its teeth."""
import math
from fractions import Fraction

import numpy as np

SHIFTS = [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (1, 1, 0), (1, -1, 0), (-1, 1, 0), (-1, -1, 0),
          (1, 0, 1), (1, 0, -1), (-1, 0, 1), (-1, 0, -1), (0, 1, 1), (0, 1, -1), (0, -1, 1), (0, -1, -1), (1, 1, 1), (1, 1, -1), (1, -1, 1),
          (1, -1, -1), (-1, 1, 1), (-1, 1, -1), (-1, -1, 1), (-1, -1, -1)]  # KISS-ICP's voxel_shifts: the visiting order
SHIFT_INDEX = {s: k for k, s in enumerate(SHIFTS)}
IDENTITY = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
FAR = 1.0e7  # the maps' max_distance: nothing is ever evicted here


class Scene:
    def __init__(self, name, om, scan, last, odom, tau, traps=0, **kw):
        self.name, self.om, self.scan, self.last, self.odom, self.tau, self.traps = name, om, scan, last, odom, tau, traps
        self.kw = kw  # solver settings (max_iter, conv, adaptive, fixed_reg)
        self.voxel_size, self.cap = om.voxel_size, om.max_points_per_voxel
        self.voxels = om.export_voxels()

    def queries(self, ko):
        """The reference's queries of the first pass: prior * scan point."""
        return ko.se3_transform(ko.se3_compose(self.last, self.odom), self.scan)

    def __repr__(self):
        return self.name


# ------------------------------------------------------------------------------------------------ distances and tie rules
def ref_sq(c, q):
    """The reference's squared distance: (dx dx + dy dy) + dz dz, every operation rounded (Python floats are IEEE doubles)."""
    dx, dy, dz = float(c[0]) - float(q[0]), float(c[1]) - float(q[1]), float(c[2]) - float(q[2])
    return (dx * dx + dy * dy) + dz * dz


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))  # exact, then one rounding (int / int division rounds correctly)


def fma_sq(c, q):
    """The same square as fma(dz, dz, fma(dy, dy, dx * dx))."""
    dx, dy, dz = float(c[0]) - float(q[0]), float(c[1]) - float(q[1]), float(c[2]) - float(q[2])
    return _fma(dz, dz, _fma(dy, dy, dx * dx))


def _closer_squares(d2, best):
    """The kernel's "norm(d2) < norm(best)" on squares (closer() in kicp_register.cu)."""
    if not d2 < best:
        return False
    if d2 >= best * (1.0 - 4e-16):
        return math.sqrt(d2) != math.sqrt(best)
    return True


def voxel_of(p, vs):
    return tuple(math.floor(float(x) / vs) for x in p)


def visiting_order(q, cands, vs):
    """Indices of the candidates inside q's 27 voxels in the reference's visiting order (shift order, then insertion order)."""
    v = voxel_of(q, vs)
    keyed = []
    for i, c in enumerate(cands):
        s = tuple(a - b for a, b in zip(voxel_of(c, vs), v))
        if s in SHIFT_INDEX:
            keyed.append((SHIFT_INDEX[s], i))
    return [i for _, i in sorted(keyed)]


def pick_reference(q, cands, vs):
    best, bd = None, None
    for i in visiting_order(q, cands, vs):
        d = math.sqrt(ref_sq(cands[i], q))
        if best is None or d < bd:
            best, bd = i, d
    return best


def pick_fma(q, cands, vs):
    best, bd = None, None
    for i in visiting_order(q, cands, vs):
        d2 = fma_sq(cands[i], q)
        if best is None or _closer_squares(d2, bd):
            best, bd = i, d2
    return best


def count_traps(qs, cand_lists, vs):
    return sum(int(pick_reference(q, c, vs) != pick_fma(q, c, vs)) for q, c in zip(qs, cand_lists))


# ------------------------------------------------------------------------------------------------------------------ priors
def _norm_square_variants(q):
    """x x + y y + z z + w w evaluated plainly and with every FMA contraction a compiler may choose."""
    sq = [Fraction(float(v)) ** 2 for v in q]
    r = lambda v: float(v)
    firsts = [r(Fraction(r(sq[0])) + Fraction(r(sq[1]))), r(sq[0] + Fraction(r(sq[1]))), r(Fraction(r(sq[0])) + sq[1])]
    out = []
    for s1 in firsts:
        for s2 in (r(Fraction(s1) + Fraction(r(sq[2]))), r(Fraction(s1) + sq[2])):
            for s3 in (r(Fraction(s2) + Fraction(r(sq[3]))), r(Fraction(s2) + sq[3])):
                out.append(s3)
    return out


def rotated_prior(ko, rng):
    """(last, odometry): a general 3-D pose and the identity.  The kernel composes the two in a file compiled with FMA contraction;
    with identity odometry every product is exact, and this pose's quaternion is one whose norm rounds to exactly 1 under every
    contraction, so the device's prior is the reference's to the last bit."""
    while True:
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        if all(math.sqrt(s) == 1.0 for s in _norm_square_variants(q)):
            last = np.r_[q, rng.uniform(-2.0, 2.0, 3)]
            assert np.array_equal(ko.se3_compose(last, IDENTITY), last)
            return last, IDENTITY.copy()


def _scan_for(ko, targets, last, odom):
    """Scan points whose queries land at `targets` (exactly under the identity prior); returns (scan, the oracle's queries)."""
    prior = ko.se3_compose(last, odom)
    scan = ko.se3_transform(ko.se3_inverse(prior), targets) if not np.array_equal(prior, IDENTITY) else targets.copy()
    return scan, ko.se3_transform(prior, scan)


def _lattice(i, spacing=4, side=8):
    """Voxel index of the i-th query: 4 voxels apart, so no query's 27 voxels hold another query's points; negative ones included."""
    return np.array([i % side, (i // side) % side, i // (side * side)]) * spacing - spacing * side // 2


def _dyadic(x, step):
    return np.round(np.asarray(x) / step) * step


def _oracle_map(ko, vs, cap, pts):
    om = ko.OracleMap(vs, FAR, cap)
    om.add_points(np.asarray(pts, dtype=np.float64))
    assert om.num_points() == len(pts), "the map must keep every point in the given order"
    return om


# ------------------------------------------------------------------------------------------------------------------ ties
def permuted_ties(ko, n=400, vs=1.0, cap=20, rotated=False, seed=1):
    """Pairs q + (x, y, z) and q + (y, x, z): the reference's squares are identical (the sum x x + y y commutes), so the first
    point in visiting order wins; FMA squares of the two differ in the last bit.  q anywhere in its voxel, so a pair lies in one
    voxel (inserted in both orders) or across a face, edge or corner."""
    rng = np.random.default_rng(seed)
    last, odom = rotated_prior(ko, rng) if rotated else (IDENTITY.copy(), IDENTITY.copy())
    targets = _dyadic(np.array([(_lattice(i) + rng.uniform(0.05, 0.95, 3)) * vs for i in range(n)]), 2.0 ** -20)
    scan, qs = _scan_for(ko, targets, last, odom)
    pts, cands = [], []
    for i, q in enumerate(qs):
        for _ in range(1000):
            x, y, z = _dyadic(rng.uniform(-0.45, 0.45, 3) * vs, 2.0 ** -30)
            if abs(x - y) < 0.2 * vs:
                continue
            c1 = q + [x, y, z]
            d = c1 - q
            c2 = q + [d[1], d[0], d[2]]
            if np.array_equal(c2 - q, [d[1], d[0], d[2]]) and ref_sq(c1, q) == ref_sq(c2, q):
                break
        else:
            raise AssertionError("no exact pair")
        pair = [c1, c2] if i % 2 == 0 else [c2, c1]
        pts += pair
        cands.append(pair)
    om = _oracle_map(ko, vs, cap, pts)
    return Scene("permuted-ties-vs%g%s" % (vs, "-rotated" if rotated else ""), om, scan, last, odom, vs, traps=count_traps(qs, cands, vs),
                 max_iter=1)


# (query position in its voxel, candidate offsets in insertion order), both in units of vs / 16: every coordinate and every square
# is exact, so the ties are exact for any evaluation order and the visiting order across the three search stages decides
_STAGE_PATTERNS = [
    ((0, 8, 8), [(4, 2, 1), (-4, 2, 1)]),             # query on the -x face: own voxel and face voxel tie, own wins
    ((0, 8, 8), [(-4, 2, 1), (4, 2, 1)]),             # ... inserted the other way round
    ((8, 0, 8), [(2, -4, 1), (2, 4, 1)]),             # -y face
    ((8, 8, 0), [(1, 2, -4), (1, 2, 4)]),             # -z face
    ((0, 0, 8), [(-3, -2, 1), (3, -2, 1), (-2, 3, 1)]),  # on an edge, own voxel empty: face -x (shift 2) before -y (4), edge (10)
    ((0, 0, 0), [(sx * 3, sy * 2, sz * 1) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]),  # corner: 8-way tie, own wins
    ((0, 0, 0), [(sx * 3, sy * 2, sz * 1) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)][:-1]),  # ... own empty: face -x
    ((0, 0, 0), [(5, 5, 5), (3, -2, -1), (-3, 2, -1), (-3, -2, 1), (-3, -2, -1)]),  # farther own point; edges tie, (-1,-1,0) wins
    ((0, 0, 0), [(5, 5, 5), (-3, -2, -1)]),             # only the corner voxel beats the own point
    ((8, 8, 8), [(7, 4, 4), (9, 0, 0)]),              # centre: own 81/256 ties the +x face voxel's point at its gap + 1/16
    ((8, 8, 8), [(9, 0, 0), (0, 9, 0), (0, 0, -9), (7, 4, 5)]),  # own at 90/256; three faces tie at 81/256: +x (shift 1) wins
    ((8, 8, 8), [(0, 0, 9), (0, -9, 0), (8, 8, 1)]),  # -y (shift 4) before +z (5); an edge point beyond the bound
    ((8, 8, 8), [(8, 0, 0), (0, 0, -8)]),             # own point on its face; the +x point at exactly its voxel's bound: own wins
]


def stage_ties(ko, vs=1.0, cap=20, reps=8):
    """Exact ties across the three search stages (own voxel, faces, edges and corners): queries exactly on a voxel face, edge or
    corner and at a voxel centre, candidates spread over the voxels that touch it (KISS-ICP visits them in a fixed order: the
    first wins).  They exercise the visiting order of the staged search and its pruning bound bound (1 + 1e-6) + 1e-10."""
    assert math.frexp(vs)[0] == 0.5, "dyadic scenes need a power-of-two voxel size"
    targets, cands, pts = [], [], []
    i = 0
    for _ in range(reps):
        for u, offs in _STAGE_PATTERNS:
            q = (_lattice(i) + np.array(u) / 16.0) * vs
            cs = [q + np.array(o) / 16.0 * vs for o in offs]
            targets.append(q)
            cands.append(cs)
            pts += cs
            i += 1
    targets = np.array(targets)
    scan, qs = _scan_for(ko, targets, IDENTITY, IDENTITY)
    assert np.array_equal(qs, targets)
    om = _oracle_map(ko, vs, cap, pts)
    return Scene("stage-ties-vs%g" % vs, om, scan, IDENTITY.copy(), IDENTITY.copy(), vs, max_iter=1)


def near_ties(ko, n=200, vs=1.0, cap=20, rotated=False, seed=3):
    """Ulp-level near-ties, two points A (inserted first) and B of one voxel, found by walking B's z through consecutive doubles:
    even queries: B's square is one ulp below A's but both round to the same norm — A must win (the same_norm rule);
    odd queries: B's norm is one ulp below A's — B must win."""
    rng = np.random.default_rng(seed)
    last, odom = rotated_prior(ko, rng) if rotated else (IDENTITY.copy(), IDENTITY.copy())
    targets = _dyadic(np.array([(_lattice(i) + rng.uniform(0.47, 0.53, 3)) * vs for i in range(n)]), 2.0 ** -20)
    scan, qs = _scan_for(ko, targets, last, odom)
    pts, cands = [], []
    ks = np.arange(-600, 601, dtype=np.float64)
    for i, q in enumerate(qs):
        for _ in range(1000):
            x, y = _dyadic(rng.uniform(-0.44, 0.44, 2) * vs, 2.0 ** -30)
            z = _dyadic(rng.uniform(0.002, 0.02) * vs * rng.choice([-1, 1]), 2.0 ** -30)
            if abs(x - y) < 0.25 * vs:
                continue
            a = q + [x, y, z]
            d = a - q
            bx, by = q[0] + d[1], q[1] + d[0]
            if bx - q[0] != d[1] or by - q[1] != d[0]:
                continue
            sa = ref_sq(a, q)
            # steps of about 1/8 ulp of the square
            unit = math.ulp(a[2]) * max(1.0, round(math.ulp(sa) / (16.0 * abs(d[2]) * math.ulp(a[2]))))
            bz = a[2] + ks * unit
            dz = bz - q[2]
            sb = (d[1] * d[1] + d[0] * d[0]) + dz * dz  # (numpy float64: one rounding per operation, as the reference)
            if i % 2 == 0:
                ok = (sb == np.nextafter(sa, 0.0)) & (np.sqrt(sb) == math.sqrt(sa))
            else:
                ok = np.sqrt(sb) == np.nextafter(math.sqrt(sa), 0.0)
            if not ok.any():
                continue
            b = np.array([bx, by, bz[np.flatnonzero(ok)[0]]])
            if voxel_of(a, vs) != voxel_of(b, vs):
                continue
            break
        else:
            raise AssertionError("no near-tie")
        pts += [a, b]
        cands.append([a, b])
    om = _oracle_map(ko, vs, cap, pts)
    for k, (q, c) in enumerate(zip(qs, cands)):  # the construction holds: the reference's own choice
        assert pick_reference(q, c, vs) == k % 2
    return Scene("near-ties-vs%g%s" % (vs, "-rotated" if rotated else ""), om, scan, last, odom, vs, traps=count_traps(qs, cands, vs),
                 max_iter=1)


def tie_scenes(ko):
    """The tie scenes of the suite.  The rotated ones run one pass only: after the first solve the kernel's pose differs from the
    reference's in the last bits (its sums are added in another order), so an exact tie of a later pass is not defined."""
    return [permuted_ties(ko), permuted_ties(ko, vs=0.5, seed=2), permuted_ties(ko, rotated=True, seed=4), stage_ties(ko),
            stage_ties(ko, vs=0.5), near_ties(ko), near_ties(ko, vs=0.5, seed=5), near_ties(ko, rotated=True, seed=6)]


# ------------------------------------------------------------------------------------------------------------- map shapes
def map_shape(ko, vs, cap, origin=(0.0, 0.0, 0.0), n_surface=240, seed=7, **kw):
    """A block of 6 x 6 x 2 voxels around `origin` (negative coordinates when it is 0), every voxel filled to the cap, and a scan of
    points near the stored ones plus queries exactly on voxel faces.  The pose is the block's origin with the identity rotation,
    so a face point's query of the first pass is the face point itself."""
    assert math.frexp(vs)[0] != 0.5, "map shapes use voxel sizes that are not powers of two"
    rng = np.random.default_rng(seed)
    origin = np.asarray(origin, dtype=np.float64)
    ov = np.floor(origin / vs).astype(np.int64)
    g = int(math.ceil(cap ** (1.0 / 3.0)))
    cell = (np.stack(np.meshgrid(np.arange(g), np.arange(g), np.arange(g), indexing="ij"), -1).reshape(-1, 3) + 0.5) / g
    pts = []
    for v in [(i, j, k) for i in range(-3, 3) for j in range(-3, 3) for k in range(-1, 1)]:
        local = cell[rng.permutation(len(cell))[:cap]] + rng.uniform(-0.1, 0.1, (cap, 3)) / g
        pts.append((ov + np.array(v) + local) * vs)
    pts = np.concatenate(pts)
    om = _oracle_map(ko, vs, cap, pts)
    assert np.all(om.export_voxels()[1] == cap)
    last = np.r_[0.0, 0.0, 0.0, 1.0, origin]
    # points near the stored ones, seen from a pose slightly off the prior ...
    true_rel = ko.se3_exp([0.03 * vs, -0.02 * vs, 0.0, 0.0, 0.0, 0.01])
    world = pts[rng.integers(0, len(pts), n_surface)] + 0.05 * vs * rng.standard_normal((n_surface, 3))
    surface = ko.se3_transform(ko.se3_inverse(ko.se3_compose(last, true_rel)), world)
    # ... and points whose first query lies exactly on a voxel face (p = w - t is exact for w near t, and then so is p + t)
    faces = []
    while len(faces) < 60:
        w = (ov + rng.integers(-3, 3, 3) + rng.uniform(0.0, 1.0, 3)) * vs
        ax = rng.integers(0, 3)
        w[ax] = float(ov[ax] + rng.integers(-3, 4)) * vs
        p = w - origin
        if np.array_equal(p + origin, w):
            faces.append(p)
    scan = np.concatenate([surface, np.array(faces)])
    name = "shape-vs%g-cap%d%s" % (vs, cap, "" if not origin.any() else "-at(%g,%g,%g)" % tuple(origin))
    return Scene(name, om, scan, last, IDENTITY.copy(), 1.5 * vs, **kw)


def shape_scenes(ko):
    """Non-power-of-two voxel sizes (PointToVoxel divides), caps that shrink the kernel's tasks per batch below 32 (25 and more
    points per voxel) and fill its line buffer, and maps far from the origin, where an ulp of a coordinate is larger than the
    certificates' absolute margins."""
    return [map_shape(ko, 0.3, 1), map_shape(ko, 0.75, 24), map_shape(ko, 0.6, 25, seed=8), map_shape(ko, 0.75, 29, origin=(-3e5, 2e5, 10.0)),
            map_shape(ko, 0.3, 255, n_surface=100, max_iter=3), map_shape(ko, 0.75, 20, origin=(4.2e5, 5.8e6, 0.0), seed=9)]


# ------------------------------------------------------------------------------------------------------------------ fuzz
def fuzz_cases(ko):
    """40 small random scenes and random solver settings (0..25 iterations, adaptive / fixed regularisation, gates from 5 cm to
    3 m, empty scans), each as (oracle map, its voxel-grouped points, scan, last pose, odometry, tau, solver settings).  The
    reference's own poses for them are tests/golden/ref_fuzz.npz."""
    from oracle.workloads import unicycle
    rng = np.random.default_rng(20260923)
    for case in range(40):
        vs = float(rng.choice([0.5, 1.0, 2.0]))
        cap = int(rng.choice([1, 5, 20]))
        # a bumpy ground patch plus two walls, mapped from a few random poses
        n_map = int(rng.integers(500, 6000))
        ground = np.c_[rng.uniform(-25, 25, (n_map, 2)), 0.05 * rng.standard_normal(n_map)]
        wall = np.c_[rng.uniform(-25, 25, n_map // 2), np.full(n_map // 2, 12.0) + 0.02 * rng.standard_normal(n_map // 2),
                     rng.uniform(0, 4, n_map // 2)]
        om = ko.OracleMap(vs, 100.0, cap)
        pts = np.concatenate([ground, wall])
        om.add_points(pts)
        _, _, stored = om.export_voxels()
        last = ko.planar_pose(*rng.uniform(-3, 3, 2), rng.uniform(-3.1, 3.1))
        true_rel = unicycle(rng.uniform(0.0, 1.0), rng.uniform(-0.1, 0.1))
        odom = unicycle(rng.uniform(0.0, 1.1), rng.uniform(-0.12, 0.12))
        n_scan = int(rng.integers(0, 3000))
        world = pts[rng.integers(0, len(pts), n_scan)] + 0.01 * rng.standard_normal((n_scan, 3))
        scan = ko.se3_transform(ko.se3_inverse(ko.se3_compose(last, true_rel)), world) if n_scan else np.zeros((0, 3))
        tau = float(rng.choice([0.05, 0.3, 1.0, 3.0]))
        kw = dict(max_iter=int(rng.choice([0, 1, 3, 10, 25])), conv=float(rng.choice([1e-3, 1e-6, 1e-1])),
                  adaptive=bool(rng.integers(0, 2)), fixed_reg=float(rng.choice([0.0, 0.1, 10.0])))
        yield om, vs, cap, stored, scan, last, odom, tau, kw


# --------------------------------------------------------------------------------------------------------------- edges
# Scenes that sit on the decisions of the map and front-end kernels: points on voxel faces, norms equal to the range gate,
# candidates exactly map_resolution from a stored point, first points exactly max_distance from the origin, probe chains that
# wrap past the last slot of the table, and coordinates that are not finite or do not fit an int once divided by the voxel size.
NAN, INF = float("nan"), float("inf")


def bits(a):
    """The bit patterns of a float64 array: equal arrays compare equal, NaN included."""
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def floor_key(x, vs):
    """PointToVoxel of one coordinate as the reference's x86-64 build evaluates it: NaN, +-Inf and values outside the int range
    become INT_MIN."""
    f = math.floor(x / vs) if math.isfinite(x / vs) else None
    return f if f is not None and -2 ** 31 <= f < 2 ** 31 else -2 ** 31


def boundary_cloud(vs, origin=0.0, span=6):
    """Points at exact multiples k vs of the voxel size (k in [-span, span]) and one ulp either side of them, on every axis and
    on both signs, +0.0 and -0.0, around a scalar `origin` (UTM-like offsets: 5e5, 4e6).  Returns the cloud, how many of its
    coordinates a reciprocal multiply x * (1 / vs) puts in another voxel than x / vs, and how many have a quotient that rounds up
    onto an integer that the exact quotient does not reach."""
    xs = []
    base = math.floor(origin / vs)
    for k in range(base - span, base + span + 1):
        x = k * vs
        xs += [x, np.nextafter(x, -INF), np.nextafter(x, INF)]
        # the doubles just below k vs whose quotient still rounds onto k: exact arithmetic would floor them to k - 1
        y = np.nextafter(x, -INF)
        for _ in range(4):
            y = np.nextafter(y, -INF)
            xs.append(y)
    xs += [0.0, -0.0]
    # and, from further out, the doubles next to multiples of vs where x * (1 / vs) floors into another voxel than x / vs
    inv = 1.0 / vs
    ks = np.arange(base - 4000, base + 4001, dtype=np.float64) * vs
    for steps in range(-3, 4):
        c = ks
        for _ in range(abs(steps)):
            c = np.nextafter(c, INF if steps > 0 else -INF)
        xs += list(c[np.floor(c / vs) != np.floor(c * inv)][:6])
    xs = np.array(xs)
    flips = int(sum(math.floor(x / vs) != math.floor(x * inv) for x in xs))
    rounded = int(sum(math.floor(x / vs) != math.floor(Fraction(x) / Fraction(vs)) for x in xs))
    n = len(xs)
    rng = np.random.default_rng(int(vs * 1000) + int(origin) % 1000)
    pts = []
    for ax in range(3):  # one coordinate on the boundary, the others anywhere in a voxel near it (also on boundaries)
        p = np.empty((n, 3))
        p[:, ax] = xs
        for o in range(3):
            if o != ax:
                p[:, o] = xs[rng.permutation(n)] if o == (ax + 1) % 3 else origin + rng.uniform(-3, 3, n) * vs
        pts.append(p)
    pts.append(np.stack([xs, xs[::-1], xs[rng.permutation(n)]], 1))
    return np.concatenate(pts), flips, rounded


def boundary_clouds():
    """(cloud, voxel size, reciprocal flips, rounded-up quotients): voxel sizes that are not powers of two (0.37, 0.3, 0.1) and
    the pipeline's own 0.5 vs and 1.5 vs of a 1.0 map, near the origin and at UTM-like offsets."""
    return [(vs,) + boundary_cloud(vs, origin) for vs in (0.37, 0.3, 0.1, 0.5, 1.5) for origin in (0.0, 5e5, 4e6)]


def range_gate_cloud(min_range, max_range):
    """Points whose norm sqrt(x x + y y + z z) is exactly min_range or max_range (axis points and (3, 4, 12) 2^k, norm 13 2^k), one
    ulp inside and outside, and the zero point.  Both ranges must be 13 2^k.  Returns the cloud and the norms the reference sees."""
    pts = []
    for r in (min_range, max_range):
        m, e = math.frexp(r / 13.0)
        assert m == 0.5, "ranges of the form 13 2^k"
        for sgn in (1.0, -1.0):
            for ax in range(3):
                p = np.zeros(3)
                p[ax] = sgn * r
                pts += [p.copy()]
                for d in (-INF, INF):
                    q = p.copy()
                    q[ax] = np.nextafter(p[ax], d)
                    pts.append(q)
            t = np.array([3.0, 4.0, 12.0]) * (r / 13.0) * sgn
            pts.append(t)
            for ax in range(3):
                for d in (-INF, INF):
                    q = t.copy()
                    q[ax] = np.nextafter(t[ax], d)
                    pts.append(q)
    pts.append(np.zeros(3))
    pts.append(np.array([-0.0, 0.0, -0.0]))
    pts = np.array(pts)
    norms = np.sqrt(pts[:, 0] * pts[:, 0] + pts[:, 1] * pts[:, 1] + pts[:, 2] * pts[:, 2])
    return pts, norms


def map_rule_points(vs=1.0, cap=4, n_voxels=24, seed=11):
    """Points for AddPoints whose candidates sit exactly map_resolution = sqrt(vs^2 / cap) from a stored point (kept: the rule is
    a strict <) or one ulp closer (dropped), along each axis, in voxels on both sides of the origin.  vs and cap are chosen so
    that map_resolution is exact (vs 1: cap 4 gives 0.5, cap 16 gives 0.25).  Returns the points and (exact, one ulp closer)
    counts of candidates, measured against the first point of their voxel."""
    res = math.sqrt(vs * vs / cap)
    assert res * res == vs * vs / cap
    rng = np.random.default_rng(seed)
    pts, exact, closer = [], 0, 0
    for i in range(n_voxels):
        v = (_lattice(i, spacing=2, side=4) * vs).astype(np.float64)
        a = v + _dyadic(rng.uniform(0.05, 0.4, 3) * vs, 2.0 ** -12)
        pts.append(a)
        ax = i % 3
        b = a.copy()
        b[ax] = a[ax] + res
        if i % 2:
            b[ax] = np.nextafter(b[ax], a[ax])  # one ulp closer
        dx = b[ax] - a[ax]
        dist = math.sqrt(dx * dx)
        if i % 2 == 0:
            assert dist == res
            exact += 1
        else:
            assert dist < res
            closer += 1
        assert floor_key(b[ax], vs) == floor_key(a[ax], vs)
        pts.append(b)
        for _ in range(cap + 2):  # more than the cap: the voxel fills up and the rest is skipped
            pts.append(v + _dyadic(rng.uniform(0.0, 1.0, 3) * vs, 2.0 ** -12))
    return np.array(pts), exact, closer


def far_first_points(max_distance=12.0, vs=3.0):
    """First points of voxels exactly max_distance from the origin (dx^2 + dy^2 + dz^2 == max_distance^2 exactly: evicted by
    the >= rule), one ulp inside (kept), and voxels whose far first point is followed by near later points (the first point
    decides).  Returns the points and the squared norms of the first points."""
    md = max_distance
    firsts = [np.array([md, 0, 0]), np.array([0, -md, 0]), np.array([0, 0, md]),
              np.array([np.nextafter(md, 0.0), 0, 0]), np.array([0, np.nextafter(-md, 0.0), 0]),
              np.array([md * 0.6, md * 0.8, 0.0]) if (md * 0.6) ** 2 + (md * 0.8) ** 2 == md * md else np.array([0, 0, -md])]
    pts = []
    for f in firsts:
        pts.append(f)
        v = np.floor(f / vs) * vs
        pts.append(v + 0.25 * vs)  # a later point of the same voxel, nearer the origin
    # a far first point (outside max_distance) followed by near points of the same voxel
    f = np.array([3.9 * vs, 3.9 * vs, 0.1])
    assert float(f @ f) >= md * md
    pts += [f, np.array([3.05 * vs, 3.05 * vs, 0.1]), np.array([3.1 * vs, 3.2 * vs, 0.2])]
    pts = np.array(pts, dtype=np.float64)
    sq = np.array([x[0] * x[0] + x[1] * x[1] + x[2] * x[2] for x in firsts])
    return pts, sq


def voxel_hash_np(x, y, z):
    """voxel_hash of kicp_device.cuh (the reference's three-prime XOR, then a murmur3 finaliser) on integer arrays."""
    u = lambda a: np.asarray(a, dtype=np.int64).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = (u(x) * np.uint32(73856093)) ^ (u(y) * np.uint32(19349669)) ^ (u(z) * np.uint32(83492791))
        h ^= h >> np.uint32(16)
        h *= np.uint32(0x85EBCA6B)
        h ^= h >> np.uint32(13)
        h *= np.uint32(0xC2B2AE35)
        h ^= h >> np.uint32(16)
    return h


_COLLIDING = {}


def colliding_keys(bits=18, half=128):
    """Voxel keys of the cube [-half, half)^3 whose hash has its low `bits` bits all set: they share the LAST home slot of every
    table of up to 2^bits slots, so a chain of them wraps past slot 0 whatever the table's size."""
    if (bits, half) not in _COLLIDING:
        r = np.arange(-half, half, dtype=np.int64)
        Y, Z = np.meshgrid(r, r, indexing="ij")
        Y, Z = Y.ravel(), Z.ravel()
        want = np.uint32((1 << bits) - 1)
        found = []
        for x in r:
            h = voxel_hash_np(np.full_like(Y, x), Y, Z)
            sel = np.flatnonzero((h & want) == want)
            found += [(int(x), int(Y[i]), int(Z[i])) for i in sel]
        _COLLIDING[(bits, half)] = np.array(found, dtype=np.int64)
    return _COLLIDING[(bits, half)]


def collision_scene(ko, n_map, vs=1.0, cap=5, n_absent=6, seed=13, max_distance=FAR):
    """A map of `n_map` voxels whose keys all collide (one chain that starts at the last slot and wraps), each holding `cap`
    points; a scan of points near the stored ones, points in the 26 neighbours of the colliding voxels, and points in colliding
    voxels absent from the map (a probe walks the whole chain, then stops at an empty slot)."""
    keys = colliding_keys()
    assert len(keys) >= n_map + n_absent
    rng = np.random.default_rng(seed)
    sel = keys[rng.permutation(len(keys))[:n_map + n_absent]]
    present, absent = sel[:n_map], sel[n_map:]
    corners = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (1, 1, 0), (0, 1, 1), (1, 0, 1)])[:cap] * 0.9 + 0.03
    pts = np.concatenate([(k + _dyadic(corners + rng.uniform(0.0, 0.04, (cap, 3)), 2.0 ** -16)) * vs for k in present])
    om = ko.OracleMap(vs, max_distance, cap)
    om.add_points(pts)
    assert om.num_points() == len(pts)
    near = pts + _dyadic(0.03 * vs * rng.standard_normal(pts.shape), 2.0 ** -20)
    shifts = np.array(SHIFTS[1:])
    nbr = np.concatenate([(k + shifts[rng.permutation(26)[:8]] + rng.uniform(0.0, 1.0, (8, 3))) * vs for k in present])
    miss = np.concatenate([(k + rng.uniform(0.0, 1.0, (4, 3))) * vs for k in absent])
    scan = np.concatenate([near, nbr, miss])
    sc = Scene("collide-%d-vs%g" % (n_map, vs), om, scan, IDENTITY.copy(), IDENTITY.copy(), 1.5 * vs, max_iter=3)
    sc.present, sc.absent = present, absent
    return sc


def collision_scenes(ko):
    return [collision_scene(ko, n, vs=vs, seed=13 + n) for n, vs in ((3, 1.0), (9, 0.5), (17, 0.3), (40, 1.0))]


def nonfinite_rows(vs):
    """Rows with NaN, +-Inf and +-3e9 vs in one or all coordinates (the reference's key of such a coordinate is INT_MIN), the
    others inside voxel 0 so that a conversion that gave 0 for NaN would put the point into voxel (0, 0, 0)."""
    bad = [NAN, INF, -INF, 3e9 * vs, -3e9 * vs]
    rows = []
    for b in bad:
        for ax in range(3):
            p = np.full(3, 0.25 * vs)
            p[ax] = b
            rows.append(p)
        rows.append(np.full(3, b))
    return np.array(rows)


def with_nonfinite(pts, vs, seed=17):
    """`pts` with the rows of nonfinite_rows() spread through it, NaN rows first (so that a NaN point comes first in voxel
    (0, 0, 0) under a conversion that gives 0 for NaN), and a real point of voxel (0, 0, 0) after them."""
    rng = np.random.default_rng(seed)
    bad = nonfinite_rows(vs)
    nan_first = np.array([[NAN, 0.25 * vs, 0.25 * vs], [NAN, NAN, NAN], [0.3 * vs, 0.3 * vs, 0.3 * vs]])
    out = np.array(pts, dtype=np.float64, copy=True)
    for row in bad:
        i = int(rng.integers(0, len(out) + 1))
        out = np.insert(out, i, row, axis=0)
    return np.concatenate([nan_first, out])
