"""Pins the CPU oracle to the golden vectors produced by the reference's own sources (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from scenes import fuzz_cases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_map(ko, z):
    m = ko.OracleMap(float(z["voxel_size"]), float(z["max_range"]), int(z["max_points_per_voxel"]))
    m.add_points(z["map_points"])  # voxel-grouped, insertion order kept
    assert m.num_points() == len(z["map_points"])
    return m


@pytest.mark.parametrize("name", ["reg_cfg1", "reg_cfg2_small"])
def test_oracle_matches_reference_golden(oracle, name):
    ko = oracle
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    m = load_map(ko, z)
    keys, counts, pts = m.export_voxels()
    assert np.array_equal(keys, z["map_keys"]) and np.array_equal(counts, z["map_counts"]) and np.array_equal(pts, z["map_points"])
    for case in z["cases"]:
        max_iter, conv, adaptive, fixed, tau = int(case[0]), case[1], bool(case[2]), case[3], case[4]
        pose, st = m.register(z["scan"], z["last_pose"], z["rel_odom"], tau, max_iter=max_iter, conv=conv, adaptive=adaptive,
                              fixed_reg=fixed)
        # same sources of rounding, same order: the restatement reproduces the reference bit for bit
        assert np.array_equal(pose, case[5:]), (name, case[:5], ko.pose_delta(pose, case[5:]))


def test_threshold_matches_reference_golden(oracle):
    ko = oracle
    z = np.load(os.path.join(GOLDEN, "threshold.npz"))
    th = ko.OracleThreshold(float(z["map_err"]), float(z["max_range"]), True, 1.0)
    for e, tau in zip(z["errs"], z["taus"]):
        th.update(e)
        assert th.compute() == tau


def test_oracle_matches_reference_build_live(oracle, workload):
    """The restatement against the poses the reference's own Registration.cpp (oracle/_ref) returned on cfg2 with 1 and 3 threads
    (tests/golden/ref_cfg2_threads.npz)."""
    ko = oracle
    z = np.load(os.path.join(GOLDEN, "ref_cfg2_threads.npz"))
    w = workload(2)
    po, _ = w.map.register(w.scan, w.last_pose, w.rel_odom, w.tau)
    for thr, pr in zip(z["threads"], z["poses"]):
        dt, ang = ko.pose_delta(pr, po)
        assert dt < 1e-12 and ang < 1e-12, (thr, dt, ang)


@pytest.mark.skipif(not os.path.exists(os.path.join(os.path.dirname(GOLDEN), "..", "oracle", "_ref", "libkicp_ref.so")),
                    reason="oracle/_ref (the reference's own sources, built where a reference checkout exists) not built")
def test_pipeline_golden_is_reproducible(oracle):
    """The committed pipeline fixture equals a fresh run of the reference's own pipeline sources (threads = 1)."""
    from oracle import sequences as S
    ko = oracle
    z = np.load(os.path.join(GOLDEN, "pipeline_seq.npz"))
    seq = S.unpack_sequence(z, True)
    pipe = ko.ref_pipeline(max_num_threads=1, deskew=True)
    poses, n_src, n_map = S.run_pipeline(pipe, seq)
    pipe.close()
    assert np.array_equal(poses, z["deskew_poses"]) and np.array_equal(n_map, z["deskew_n_map"])


def test_oracle_matches_reference_build_fuzz(oracle):
    """Randomised pin of the restatement: the oracle on the scenes of fuzz_cases against the poses the reference's own
    Registration.cpp (oracle/_ref, one thread = the same summation order) returned for them (tests/golden/ref_fuzz.npz).  Same NaN
    pattern, poses within 1e-14 (most are bit-identical; the rest differ by one rounding: the test wrapper rebuilds Sophus::SE3d
    from a pose7, whose constructor re-normalises the quaternion)."""
    ko = oracle
    ref = np.load(os.path.join(GOLDEN, "ref_fuzz.npz"))["poses"]
    exact = 0
    for case, (om, _, _, stored, scan, last, odom, tau, kw) in enumerate(fuzz_cases(ko)):
        assert om.num_points() == len(stored)
        po, _ = om.register(scan, last, odom, tau, **kw)
        pr = ref[case]
        assert np.array_equal(np.isnan(po), np.isnan(pr)), (case, kw)
        if np.isnan(po).any():
            continue
        dt, ang = ko.pose_delta(po, pr)
        assert dt < 1e-14 and ang < 1e-14, (case, kw, dt, ang)
        exact += int(np.array_equal(po, pr))
    assert case == 39 and exact >= 20
