"""The voxel map's launch sequences, entry point by entry point: the ctx.launch_count difference of every branch of every call is
pinned, and after every call the map equals the CPU oracle's bit for bit (export_voxels, num_points, num_voxels).

The map starts with storage for 16384 voxels (KICP_MAP_VOXELS), and a first insert of 8000 points sizes its hash table for 8192
voxels.  map_reserve makes room for one new voxel per inserted point, so an insert of n points grows the table when num_voxels + n
exceeds 8192 and the storage when it exceeds 16384; the calls below stay under both bounds except the three growth calls at the end.
Every inserted point lies within 9 * sqrt(3) < max_distance of the origin it is inserted with.  The frame path's map update is
pinned by test_gpu_frame_launches.py."""
import numpy as np
import pytest

import scenes as S

pytestmark = pytest.mark.gpu

VS, MAXD, CAP = 1.0, 20.0, 20
HERE, NEAR, AWAY = np.zeros(3), np.array([20.0, 0.0, 0.0]), np.array([1000.0, 0.0, 0.0])  # evicts nothing / some voxels / all
NONE = np.zeros((0, 3))
YAW = [0.0, 0.0, np.sin(0.05), np.cos(0.05)]

EXPECTED = {
    "AddPoints n=0": 0,
    "AddPoints": 2,  # k_add_find_or_create, k_add_commit
    "RemovePointsFarFromLocation empty map": 0,
    "RemovePointsFarFromLocation nothing evicted": 1,  # k_mark_far
    "RemovePointsFarFromLocation some evicted": 4,  # k_mark_far, k_exclusive_sum, k_compact_blocks, k_table_rebuild
    "RemovePointsFarFromLocation all evicted": 3,  # no survivor: the table is cleared, not rebuilt
    "Update(points, origin) nothing evicted": 3,
    "Update(points, origin) some evicted": 6,
    "Update(points, origin) all evicted": 5,
    "Update(points, pose) nothing evicted": 3,
    "Update(points, pose) some evicted": 6,
    "Update(points, pose) all evicted": 5,
    "Update n=0 empty map": 0,
    "Update n=0 nothing evicted": 1,
    "Update n=0 some evicted": 4,
    "Update n=0 all evicted": 3,
    "load_voxels 0 voxels": 0,
    "load_voxels": 2,  # k_load_voxels, k_table_rebuild
    "Pointcloud empty map": 0,
    "Pointcloud": 3,  # k_block_counts, k_exclusive_sum, k_pack_points
    "PointcloudF32 empty map": 0,
    "PointcloudF32": 3,
    "export_voxels empty map": 0,
    "export_voxels": 3,
    "GetClosestNeighbor": 1,  # k_nearest
    "PointcloudF32Live first call": 3,  # k_live_init, k_exclusive_sum, k_live_add
    "PointcloudF32Live unchanged map": 6,  # + k_live_match, k_exclusive_sum, k_live_holes
    "PointcloudF32Live map that shrank": 7,  # + k_live_move
    "AddPoints growing the table": 3,  # k_table_rebuild at the new size, then the insert
    "AddPoints growing the storage": 5,  # k_fill_i32, k_table_rebuild in the new slab and at the new size, then the insert
    "reserve beyond the storage": 2,  # k_fill_i32, k_table_rebuild in the new slab
    "reserve within the storage": 0,
}


def sorted_voxels(keys, counts, pts):
    """a map's voxels in key order (the device's block order is not part of the result)"""
    off = np.concatenate([[0], np.cumsum(counts)])
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return keys[order], counts[order], np.concatenate([pts[off[i]:off[i + 1]] for i in order]) if len(order) else pts


def same_rows32(a, b):
    """two float32 clouds hold the same records, bit for bit, in any order"""
    a, b = np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])])


class Drive:
    """one GPU map and its CPU oracle, driven call by call: the launches of each call are recorded under the call's name"""

    def __init__(self, ctx, gm, om):
        self.ctx, self.gm, self.om, self.launches = ctx, gm, om, {}

    def same_map(self, om=None):
        om = om or self.om
        gm = self.gm
        assert gm.num_points() == om.num_points() and gm.num_voxels() == om.num_voxels()
        k1, c1, p1 = sorted_voxels(*gm.export_voxels())
        k0, c0, p0 = sorted_voxels(*om.export_voxels())
        assert np.array_equal(k1, k0) and np.array_equal(c1, c0) and S.same_bits(p1, p0)

    def call(self, name, gpu, cpu=None, om=None):
        l0 = self.ctx.launch_count
        out = gpu()
        self.launches.setdefault(name, set()).add(self.ctx.launch_count - l0)
        if cpu:
            cpu()
        self.same_map(om)
        return out

    def add(self, pts, name="AddPoints"):
        self.call(name, lambda: self.gm.AddPoints(pts), lambda: self.om.add_points(pts))

    def remove(self, origin, what):
        self.call("RemovePointsFarFromLocation " + what, lambda: self.gm.RemovePointsFarFromLocation(origin),
                  lambda: self.om.remove_far(origin))

    def update(self, pts, origin, what):
        self.call("Update(points, origin) " + what, lambda: self.gm.Update(pts, origin), lambda: self.om.update_origin(pts, origin))

    def update_pose(self, pts, pose, what):
        self.call("Update(points, pose) " + what, lambda: self.gm.Update(pts, pose), lambda: self.om.update_pose(pts, pose))

    def update_none(self, origin, what):
        self.call("Update n=0 " + what, lambda: self.gm.Update(NONE, origin), lambda: self.om.update_origin(NONE, origin))


def test_map_launches_per_entry_point(oracle, monkeypatch):
    import kinematic_icp_b200 as kb
    rng = np.random.default_rng(5)

    def cloud(n):
        return rng.uniform(-9.0, 9.0, size=(n, 3))

    ctx = kb.Context(0)
    monkeypatch.setenv("KICP_MAP_VOXELS", "16384")
    gm = kb.VoxelHashMap(ctx, VS, MAXD, CAP)
    monkeypatch.delenv("KICP_MAP_VOXELS")
    d = Drive(ctx, gm, oracle.OracleMap(VS, MAXD, CAP))
    try:
        for name in ("Pointcloud", "PointcloudF32", "export_voxels"):
            d.call(name + " empty map", getattr(gm, name))
        d.remove(HERE, "empty map")
        d.update_none(HERE, "empty map")
        d.add(cloud(8000))  # sizes the table: the growth of an empty map's table launches nothing
        d.add(NONE, "AddPoints n=0")
        d.add(cloud(1000))
        d.remove(HERE, "nothing evicted")
        d.remove(NEAR, "some evicted")
        assert gm.num_voxels() > 0
        d.update(cloud(1000), HERE, "nothing evicted")
        d.update(cloud(1000), NEAR, "some evicted")
        d.update(cloud(1000) - AWAY, AWAY, "all evicted")
        assert gm.Empty()
        d.update_pose(cloud(1000), np.r_[YAW, HERE], "nothing evicted")
        d.update_pose(cloud(1000), np.r_[YAW, 0.6 * NEAR], "some evicted")
        d.update_pose(cloud(1000) - AWAY, np.r_[0.0, 0.0, 0.0, 1.0, AWAY], "all evicted")
        assert gm.Empty()
        d.add(cloud(1000))
        d.update_none(HERE, "nothing evicted")
        d.update_none(NEAR, "some evicted")
        assert gm.num_voxels() > 0
        d.update_none(AWAY, "all evicted")
        d.add(cloud(1000))
        d.remove(AWAY, "all evicted")
        assert gm.Empty()

        d.add(cloud(4000))
        pc = d.call("Pointcloud", gm.Pointcloud)
        pc32 = d.call("PointcloudF32", gm.PointcloudF32)
        keys, counts, pts = d.call("export_voxels", gm.export_voxels)
        assert len(pc) == gm.num_points() > 0 and S.same_bits(pc, pts)  # both pack the voxels in block order
        assert np.array_equal(pc32.view(np.uint32), pc.astype(np.float32).view(np.uint32))
        q = rng.uniform(-12.0, 12.0, size=(2000, 3))
        gp, gd = d.call("GetClosestNeighbor", lambda: gm.GetClosestNeighbor(q))
        op, od = d.om.nearest(q)
        assert S.same_bits(gp, op) and S.same_bits(gd, od)

        d.call("load_voxels 0 voxels", lambda: gm.load_voxels(np.zeros((0, 3), np.int32), np.zeros(0, np.int32), NONE),
               om=oracle.OracleMap(VS, MAXD, CAP))
        d.call("load_voxels", lambda: gm.load_voxels(keys, counts, pts))

        for name in ("first call", "unchanged map"):
            rec, _ = d.call("PointcloudF32Live " + name, gm.PointcloudF32Live)
            assert same_rows32(rec, gm.PointcloudF32())
        d.remove(NEAR, "some evicted")
        rec, st = d.call("PointcloudF32Live map that shrank", gm.PointcloudF32Live)
        assert st["removed"] > 0 and same_rows32(rec, gm.PointcloudF32())

        d.add(cloud(9000), "AddPoints growing the table")  # 8192 < num_voxels + 9000 <= 16384
        d.add(cloud(16384), "AddPoints growing the storage")
        d.call("reserve beyond the storage", lambda: gm.reserve(200000))
        d.call("reserve within the storage", lambda: gm.reserve(1000))
        d.add(cloud(1000))
        assert d.launches == {k: {v} for k, v in EXPECTED.items()}
    finally:
        gm.close()
        ctx.close()
