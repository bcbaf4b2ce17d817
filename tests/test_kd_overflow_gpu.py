"""Normals of the kd map when a coarser level's cell table overflows.

A level whose hashed cell table is too small for the map's cells is unusable: the search skips it and goes on at the
next coarser level.  The (k+1)-NN search of the normals carries the list and the distance bound of a finer level across
such a level, so the case needs a map that is dense enough for some searches to hold k+1 candidates at a fine level
and sparse enough elsewhere to fill a coarser level's table: clusters of points in a sparse lattice.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

K_NORMALS = 10
CELL0 = 0.2             # the default level-0 cell side (kdmap_device.cuh: KD_CELL_TARGET)


def _table_cells(m, local_map_size):
    """Per level: (occupied cells, table slots), following the index build of a map inserted as one frame."""
    n = m.shape[0]
    cap = max(n + n // 4 + 64, min(int(1.3 * n * (local_map_size + 1)), n + (8 << 20)))
    mn = m.min(0)
    ext = np.float32(max(float((m.max(0) - mn).max()), 1e-6))
    scale = min(np.float32(8 / CELL0), np.float32(8191) / ext)
    q = np.clip((m - mn) * scale, 0, 8191).astype(np.int64)
    out = []
    for level in range(5):
        want, slots = int(1.5 * cap) >> level, 64
        while slots < want:
            slots <<= 1
        out.append((len(np.unique(q >> (3 + level), axis=0)), slots))
    return out


def _map(seed):
    rng = np.random.RandomState(seed)
    g = np.arange(17) * 1.65
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    lattice = lattice + rng.uniform(-0.1, 0.1, lattice.shape)
    centres = rng.uniform(1.0, 25.0, (110, 3))
    clusters = (centres[:, None, :] + rng.normal(0.0, 0.45, (110, 30, 3))).reshape(-1, 3)
    return np.concatenate([lattice, clusters]).astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1])
def test_kd_normals_across_an_overflowed_level(seed):
    import pylidar_slam_b200 as b200
    from scipy.spatial import cKDTree
    m = _map(seed)
    levels = _table_cells(m, local_map_size=1)
    assert levels[0][0] <= levels[0][1] // 2                        # level 0 is usable ...
    assert any(cells > slots for cells, slots in levels[1:]), levels  # ... a coarser level certainly overflows

    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=1, num_neighbors_normals=K_NORMALS))
    lm.init()
    lm.update(np.eye(4, dtype=np.float32)[None], new_pc_data=m)
    res = lm.nearest_neighbor_search(m)
    assert np.array_equal(res.neighbor_points, m)                    # every query is a map point: its own match

    # independent float64 normals from the exact k nearest other points (cKDTree on the same float32 map)
    tree = cKDTree(m.astype(np.float64))
    d, idx = tree.query(m.astype(np.float64), k=K_NORMALS + 2)
    unique_set = d[:, K_NORMALS + 1] > d[:, K_NORMALS] * (1 + 1e-6)  # no tie at the k-th neighbour
    diff = (m[idx[:, 1:K_NORMALS + 1]] - m[:, None, :]).astype(np.float64)
    C = (diff[:, :, :, None] * diff[:, :, None, :]).mean(axis=1)
    w, v = np.linalg.eigh(C)
    gap = (w[:, 1] - w[:, 0]) / np.maximum(w[:, 2], 1e-300)
    sin = np.linalg.norm(np.cross(res.neighbor_normals.astype(np.float64), v[:, :, 0]), axis=1)
    ok = unique_set & (gap > 1e-3)
    assert ok.mean() > 0.95, ok.mean()
    assert (sin[ok] <= 2e-5 / gap[ok] + 2e-7).all(), (int((sin[ok] > 2e-5 / gap[ok] + 2e-7).sum()), float(sin[ok].max()))
