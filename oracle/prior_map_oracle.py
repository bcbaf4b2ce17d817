"""Host model of a kd local map that starts from a set cloud (KdTreeLocalMap.set_map_pointcloud, update and
get_last_frame, slam/odometry/local_map.py:289-362, 425-427), for the CPU tests: which rows the map holds after every
update, in order, and which of them get_last_frame returns.

The set cloud is held as no frame, so the eviction that follows local_map_size frames drops the oldest FRAME's row
count from the front of the map: prior-map rows go first.  Rows are float32, moved as the reference moves a float32 map
(float32 inverse, float32 einsum); NaN rows of a frame are dropped before its count is taken.
"""
import numpy as np


class PriorMapOracle:
    def __init__(self, local_map_size: int):
        self.local_map_size = local_map_size
        self.rows = None
        self.counts = []

    def set_map_pointcloud(self, cloud):
        cloud = np.asarray(cloud)
        assert cloud.ndim == 2 and cloud.shape[1] == 3
        assert np.isfinite(cloud.astype(np.float32)).all(), "the GPU map refuses non-finite rows"
        self.rows = cloud.astype(np.float32)
        self.counts = []

    def update(self, rel_pose, points=None):
        new = None
        if points is not None:
            new = np.asarray(points, np.float32).reshape(-1, 3)
            new = new[~np.isnan(new).any(axis=1)]
        if self.rows is None:
            self.rows = new
            self.counts.append(0 if new is None else new.shape[0])
            return
        inv = np.linalg.inv(np.asarray(rel_pose, np.float32).reshape(4, 4))
        moved = np.einsum("ij,nj->ni", inv[:3, :3], self.rows) + inv[:3, 3].reshape(1, 3)
        if new is not None:
            self.rows = np.concatenate([moved, new], axis=0)
            self.counts.append(new.shape[0])
        else:
            self.rows = moved
        if len(self.counts) > self.local_map_size:
            self.rows = self.rows[self.counts.pop(0):]

    def get_last_frame(self):
        if not self.counts:
            raise IndexError("list index out of range")
        return self.rows[-self.counts[-1]:]
