"""The rule of a map with a frozen prior (include/kicp.h, kicp_map_freeze), restated from the CPU oracle's pieces (test infrastructure).

The prior's voxels are kept exactly as given, never evicted and never written into.  The live layer is an OracleMap fed the points (in
the map's frame, after the pose) whose voxel key is not a prior voxel's key, then evicted by the usual rule.  The map is the prior's
voxels followed by the live ones.  Finite points only (the voxel key of a non-finite point is not restated here)."""
import numpy as np


def voxel_keys(pts, voxel_size):
    """the voxel key of every (finite) point: floor(p / voxel_size) per axis, as the reference's PointToVoxel"""
    return np.floor(np.asarray(pts, dtype=np.float64) / voxel_size).astype(np.int64)


class PriorMap:
    """a map whose voxels `prior` = (keys, counts, points) are frozen, with an empty live layer beside them"""

    def __init__(self, ko, prior, voxel_size=1.0, max_distance=100.0, max_points_per_voxel=20):
        self.ko = ko
        keys, counts, pts = prior
        self.prior = (np.asarray(keys, np.int32).reshape(-1, 3).copy(), np.asarray(counts, np.int32).copy(),
                      np.asarray(pts, np.float64).reshape(-1, 3).copy())
        self.prior_keys = {tuple(k) for k in self.prior[0].tolist()}
        self.voxel_size = voxel_size
        self.live = ko.OracleMap(voxel_size, max_distance, max_points_per_voxel)

    def not_prior(self, world):
        """the points whose voxel is not a prior voxel, in input order"""
        world = np.asarray(world, dtype=np.float64).reshape(-1, 3)
        if len(world) == 0 or not self.prior_keys:
            return world
        keep = np.fromiter((tuple(k) not in self.prior_keys for k in voxel_keys(world, self.voxel_size).tolist()), bool, len(world))
        return world[keep]

    def add_points(self, pts):
        self.live.add_points(self.not_prior(pts))

    def remove_far(self, origin):
        self.live.remove_far(origin)

    def update_origin(self, pts, origin):
        self.add_points(pts)
        self.remove_far(origin)

    def update_pose(self, pts, p7):
        self.add_points(self.ko.se3_transform(p7, np.asarray(pts, dtype=np.float64).reshape(-1, 3)))
        self.remove_far(np.asarray(p7, dtype=np.float64)[4:])

    def live_voxels(self):
        return self.live.export_voxels()

    def export_voxels(self):
        """the union: the prior's voxels, then the live layer's (each voxel's points in insertion order)"""
        lk, lc, lp = self.live.export_voxels()
        pk, pc, pp = self.prior
        return np.concatenate([pk, lk]).astype(np.int32), np.concatenate([pc, lc]).astype(np.int32), np.concatenate([pp, lp])

    def num_points(self):
        return int(self.prior[1].sum()) + self.live.num_points()

    def num_voxels(self):
        return len(self.prior[1]) + self.live.num_voxels()

    def union_map(self):
        """an OracleMap that holds the union (for the oracle's registration against it): loaded voxel by voxel, each voxel's points in
        order, which the insertion rule keeps as they are (they were accepted into that voxel in that order)"""
        m = self.ko.OracleMap(self.voxel_size, self.live.max_distance, self.live.max_points_per_voxel)
        keys, counts, pts = self.export_voxels()
        m.add_points(pts)
        return m


def prior_pack(prior):
    """the prior's points in block order (what kicp_map_pointcloud_layer returns for KICP_MAP_LAYER_PRIOR)"""
    return np.asarray(prior[2], dtype=np.float64).reshape(-1, 3)
