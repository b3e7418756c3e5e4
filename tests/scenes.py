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
