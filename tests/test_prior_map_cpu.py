"""A frozen prior inside the voxel map, without a GPU: the rule of tests/prior_map_oracle.py on its own cases (a point in a prior voxel
is dropped, a prior voxel beyond max_distance survives, the live layer is the map the same calls build from an empty map fed the points
that were not dropped); the layer constants against the header and the ctypes mirror; every argument check of the new calls that fails
before any device work, with its text; and kicp_replay's refusal of --freeze-prior without --load-map."""
import os
import re
import subprocess

import numpy as np

from prior_map_oracle import PriorMap, voxel_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    import __graft_entry__ as g
    g.build()


def _prior(ko, pts, vs=1.0, md=30.0):
    m = ko.OracleMap(vs, md, 20)
    m.add_points(pts)
    return m.export_voxels()


def test_points_in_prior_voxels_are_dropped(oracle):
    ko = oracle
    prior = _prior(ko, np.array([[0.5, 0.5, 0.5], [3.25, 0.5, 0.5]]))
    pm = PriorMap(ko, prior, 1.0, 30.0, 20)
    new = np.array([[0.9, 0.9, 0.9], [1.5, 0.5, 0.5], [3.0, 0.99, 0.0], [-0.5, 0.5, 0.5]])
    pm.add_points(new)
    lk, lc, lp = pm.live_voxels()
    assert sorted(map(tuple, lk.tolist())) == [(-1, 0, 0), (1, 0, 0)]
    assert pm.num_points() == 4 and pm.num_voxels() == 4
    keys, counts, pts = pm.export_voxels()
    assert np.array_equal(keys[:2], prior[0]) and np.array_equal(pts[:2], prior[2])  # the prior first, as given


def test_the_live_layer_is_the_map_of_the_points_kept(oracle):
    ko = oracle
    rng = np.random.default_rng(5)
    base = rng.uniform(-10, 10, (2000, 3))
    prior = _prior(ko, base)
    pm = PriorMap(ko, prior, 1.0, 30.0, 20)
    frame = rng.uniform(-20, 20, (3000, 3))
    pose = np.array([0.0, 0.0, np.sin(0.3), np.cos(0.3), 2.0, -1.0, 0.0])
    pm.update_pose(frame, pose)
    world = ko.se3_transform(pose, frame)
    pk = {tuple(k) for k in prior[0].tolist()}
    kept = world[[tuple(k) not in pk for k in voxel_keys(world, 1.0).tolist()]]
    assert 0 < len(kept) < len(world)
    ref = ko.OracleMap(1.0, 30.0, 20)
    ref.add_points(kept)
    ref.remove_far(pose[4:])
    a, b = pm.live_voxels(), ref.export_voxels()
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_far_prior_voxels_survive_and_thaw(oracle):
    """a prior voxel beyond max_distance survives every eviction while frozen; thawed, the same map (an OracleMap of the union) loses
    it at the next eviction"""
    ko = oracle
    prior = _prior(ko, np.array([[0.5, 0.5, 0.5], [250.5, 0.5, 0.5]]), md=1000.0)
    pm = PriorMap(ko, prior, 1.0, 30.0, 20)
    pm.update_origin(np.array([[5.5, 0.5, 0.5], [80.5, 0.5, 0.5]]), [0.0, 0.0, 0.0])
    keys, counts, _ = pm.export_voxels()
    assert (250, 0, 0) in set(map(tuple, keys.tolist())) and (80, 0, 0) not in set(map(tuple, keys.tolist()))
    thawed = pm.union_map()  # thaw: the voxels stay, as ordinary ones
    assert thawed.num_voxels() == pm.num_voxels()
    thawed.remove_far([0.0, 0.0, 0.0])
    keys, _, _ = thawed.export_voxels()
    assert set(map(tuple, keys.tolist())) == {(0, 0, 0), (5, 0, 0)}


def test_layer_constants():
    from kinematic_icp_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "kicp.h")).read()
    defs = dict((k, int(v)) for k, v in re.findall(r"#define (KICP_MAP_LAYER_[A-Z]+) (\d+)", hdr))
    assert defs == {"KICP_MAP_LAYER_ALL": 0, "KICP_MAP_LAYER_PRIOR": 1, "KICP_MAP_LAYER_LIVE": 2}
    for k, v in defs.items():
        assert getattr(_capi, k) == v
    for name in ("kicp_map_freeze", "kicp_map_thaw", "kicp_map_prior_size", "kicp_map_pointcloud_layer",
                 "kicp_map_pointcloud_layer_device_async"):
        assert re.search(r"\bint %s\(" % name, hdr), name
        assert name in {s[0] for s in _capi.SYMBOLS}, name


def test_validation():
    """every check before the map is reachable with a null map (no device); the map last"""
    import ctypes as C
    _build()
    from kinematic_icp_b200 import _capi
    lib = _capi.lib()

    def err(rc, fn, text):
        assert rc == _capi.KICP_ERR_INVALID, rc
        assert lib.kicp_last_error().decode() == "%s: %s" % (fn, text)

    err(lib.kicp_map_freeze(None), "kicp_map_freeze", "null map")
    err(lib.kicp_map_thaw(None), "kicp_map_thaw", "null map")
    v, n = C.c_int64(), C.c_int64()
    err(lib.kicp_map_prior_size(None, None, C.byref(n)), "kicp_map_prior_size", "voxels: null pointer")
    err(lib.kicp_map_prior_size(None, C.byref(v), None), "kicp_map_prior_size", "points: null pointer")
    err(lib.kicp_map_prior_size(None, C.byref(v), C.byref(n)), "kicp_map_prior_size", "null map")
    buf = (C.c_double * 3)()
    for fn, f in (("kicp_map_pointcloud_layer", lib.kicp_map_pointcloud_layer),
                  ("kicp_map_pointcloud_layer_device_async", lib.kicp_map_pointcloud_layer_device_async)):
        for layer in (-1, 3):
            err(f(None, layer, 0, buf, 1, C.byref(n)), fn, "layer: not KICP_MAP_LAYER_ALL, KICP_MAP_LAYER_PRIOR or KICP_MAP_LAYER_LIVE")
        for dtype in (-1, 2):
            err(f(None, 1, dtype, buf, 1, C.byref(n)), fn, "dtype: not KICP_DTYPE_F64 or KICP_DTYPE_F32")
        err(f(None, 2, 0, buf, 1, None), fn, "n: null pointer")
        err(f(None, 0, 1, buf, 1, C.byref(n)), fn, "null map")
    err(lib.kicp_map_pointcloud_layer_device_async(None, 0, 0, None, 1, C.byref(n)), "kicp_map_pointcloud_layer_device_async",
        "out: null pointer")


def test_replay_refuses_freeze_without_a_map(tmp_path):
    _build()
    exe = os.path.join(ROOT, "kinematic-icp_b200", "bin", "kicp_replay")
    out = subprocess.run([exe, str(tmp_path / "none.kseq"), str(tmp_path / "x.tum"), "--freeze-prior"], capture_output=True, text=True,
                         timeout=60)
    assert out.returncode == 2 and "--freeze-prior" in out.stderr and "--load-map" in out.stderr
    out = subprocess.run([exe, str(tmp_path / "none.kseq"), str(tmp_path / "x.tum"), "--freeze-prior", "--map-update", "never"],
                         capture_output=True, text=True, timeout=60)
    assert out.returncode == 2 and "--load-map" in out.stderr
