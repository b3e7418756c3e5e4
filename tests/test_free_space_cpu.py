"""The free-space oracle (tests/free_space_oracle.py) against the rule of include/kicp.h: the DDA's visit set against a brute-force
segment-cube test, and hand-built cases whose visits and decisions are known exactly (binary-exact coordinates)."""
import numpy as np
import pytest

import free_space_oracle as F

I7 = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def _visits(o, q, v=1.0, margin=0.0, D=100.0):
    ray, keys = F.dda_visits(np.asarray(o, float), np.asarray([q], float), v, margin, D)
    return [tuple(k) for k in keys.tolist()]


def _map(keys, v=1.0):
    """an export with one point at the centre of every voxel"""
    keys = np.asarray(keys, np.int32).reshape(-1, 3)
    return keys, np.ones(len(keys), np.int32), (keys + 0.5) * v


def test_dda_matches_brute_force_segment_cube_test():
    rng = np.random.default_rng(3)
    v = 0.5
    for _ in range(300):
        # coordinates at least 0.05 v from every voxel face, so that no crossing is a near tie
        o = (rng.integers(-6, 6, 3) + rng.uniform(0.1, 0.9, 3)) * v
        q = (rng.integers(-12, 12, 3) + rng.uniform(0.1, 0.9, 3)) * v
        margin = float(rng.choice([0.0, rng.uniform(0.0, 2.0)]))
        got = _visits(o, q, v, margin)
        assert len(set(got)) == len(got)  # each visited voxel is distinct
        assert set(got) == F.brute_visits(o, q, v, margin, 100.0), (o, q, margin)


def test_axis_aligned_ray():
    assert _visits([0.5, 0.5, 0.5], [5.5, 0.5, 0.5]) == [(k, 0, 0) for k in range(6)]
    assert _visits([0.5, 0.5, 0.5], [0.5, -3.5, 0.5]) == [(0, -k, 0) for k in range(5)]


def test_ray_through_an_edge_and_a_corner_takes_the_lowest_axis_first():
    assert _visits([0.5, 0.5, 0.5], [2.5, 2.5, 0.5]) == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (2, 1, 0), (2, 2, 0)]
    assert _visits([0.5, 0.5, 0.5], [1.5, 1.5, 1.5]) == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (1, 1, 1)]
    assert _visits([0.5, 0.5, 0.5], [-0.5, 1.5, -0.5]) == [(0, 0, 0), (-1, 0, 0), (-1, 1, 0), (-1, 1, -1)]


def test_end_margin_at_and_just_past_a_face():
    # L = 4, faces crossed at t = 0.125, 0.375, 0.625, 0.875 (all exact)
    o, q = [0.5, 0.5, 0.5], [4.5, 0.5, 0.5]
    assert _visits(o, q, margin=1.5) == [(0, 0, 0), (1, 0, 0), (2, 0, 0)]  # t_end = 0.625: the crossing at t_end is not taken
    assert _visits(o, q, margin=1.5 - 1e-9) == [(k, 0, 0) for k in range(4)]
    assert _visits(o, q, margin=0.0) == [(k, 0, 0) for k in range(5)]


def test_t_end_capped_by_max_distance():
    # t_end = min(4, 2) / 4 = 0.5: crossings 0.125 and 0.375 are taken, 0.625 is not
    assert _visits([0.5, 0.5, 0.5], [4.5, 0.5, 0.5], D=2.0) == [(0, 0, 0), (1, 0, 0), (2, 0, 0)]


def test_zero_length_ray_visits_nothing_but_hits(oracle):
    vox = _map([[0, 0, 0], [1, 0, 0]])
    out, st = F.clear_free_space(oracle, vox, 0, 1.0, 100.0, [[0.5, 0.5, 0.5]], I7, [0.5, 0.5, 0.5], 0.0, 1)
    assert st == dict(rays=1, visits=0, cleared_voxels=0, cleared_points=0, prior_contradicted=0)
    assert all(np.array_equal(a, b) for a, b in zip(out, vox))


def test_non_finite_and_int_min_keys_are_not_cast(oracle):
    vox = _map([[1, 0, 0], [2, 0, 0]])
    pts = [[np.nan, 0.5, 0.5], [np.inf, 0.5, 0.5], [1e300, 0.5, 0.5], [-3e9, 0.5, 0.5], [3.5, 0.5, 0.5]]
    out, st = F.clear_free_space(oracle, vox, 0, 1.0, 100.0, pts, I7, [0.5, 0.5, 0.5], 0.0, 1)
    assert st["rays"] == 1 and st["cleared_voxels"] == 2 and st["visits"] == 4
    assert len(out[1]) == 0
    # a non-finite origin casts nothing
    _, st = F.clear_free_space(oracle, vox, 0, 1.0, 100.0, pts, I7, [np.nan, 0.0, 0.0], 0.0, 1)
    assert st["rays"] == 0 and st["visits"] == 0


@pytest.mark.parametrize("min_misses,cleared", [(3, 1), (4, 0)])
def test_min_misses_met_exactly_versus_one_short(oracle, min_misses, cleared):
    vox = _map([[2, 0, 0], [6, 0, 0], [6, 1, 0], [6, -1, 0]])
    rays = [[6.5, 0.5, 0.5], [6.5, 1.2, 0.5], [6.5, -0.2, 0.5]]  # three rays through voxel (2, 0, 0), each ending in its own wall voxel
    out, st = F.clear_free_space(oracle, vox, 0, 1.0, 100.0, rays, I7, [0.5, 0.5, 0.5], 0.0, min_misses)
    assert st["cleared_voxels"] == cleared and st["cleared_points"] == cleared
    assert st["rays"] == 3
    assert [tuple(k) for k in out[0].tolist()] == ([(6, 0, 0), (6, 1, 0), (6, -1, 0)] if cleared else [tuple(k) for k in vox[0].tolist()])


def test_a_hit_protects_and_a_prior_voxel_is_counted_not_cleared(oracle):
    vox = _map([[2, 0, 0], [3, 0, 0], [6, 0, 0]])
    rays = [[6.5, 0.5, 0.5], [6.5, 0.5, 0.5], [3.5, 0.5, 0.5]]  # the third ray ends in (3, 0, 0)
    out, st = F.clear_free_space(oracle, vox, 0, 1.0, 100.0, rays, I7, [0.5, 0.5, 0.5], 0.0, 2)
    assert [tuple(k) for k in out[0].tolist()] == [(3, 0, 0), (6, 0, 0)]
    assert st["cleared_voxels"] == 1 and st["prior_contradicted"] == 0
    out, st = F.clear_free_space(oracle, vox, 1, 1.0, 100.0, rays, I7, [0.5, 0.5, 0.5], 0.0, 2)
    assert [tuple(k) for k in out[0].tolist()] == [(2, 0, 0), (3, 0, 0), (6, 0, 0)]
    assert st["cleared_voxels"] == 0 and st["prior_contradicted"] == 1


def test_result_does_not_depend_on_the_order_of_the_rays(oracle):
    rng = np.random.default_rng(5)
    keys = np.unique(rng.integers(-8, 8, (400, 3)), axis=0)
    vox = _map(keys, 0.5)
    pts = rng.uniform(-4, 4, (500, 3))
    pose = np.array([0.0, 0.0, np.sin(0.15), np.cos(0.15), 0.3, -0.2, 0.1])
    a = F.clear_free_space(oracle, vox, 40, 0.5, 100.0, pts, pose, [0.1, 0.0, 0.2], 0.25, 2)
    b = F.clear_free_space(oracle, vox, 40, 0.5, 100.0, pts[rng.permutation(len(pts))], pose, [0.1, 0.0, 0.2], 0.25, 2)
    assert a[1] == b[1] and a[1]["cleared_voxels"] > 0
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))
