"""TEST INFRASTRUCTURE ONLY -- kd maps that drive the normals' (k+1)-NN search through each of its paths
(kdmap_device.cuh: warp_knn).  Every map is float32, built on the CPU from a fixed seed, and inserted as one frame.

  cfg2       synthetic 64x2048 scans grid-sampled at 0.3 m (the cfg2 workload): level-0 blocks of <= 64 candidates
  clusters   dense Gaussian blobs: level-0 blocks of 65 ... 128 and of more than 128 candidates
  overflow   clusters in a sparse lattice whose coarser cell tables overflow (tests/test_kd_overflow_gpu.py)
  ties       a dyadic lattice anchored at the origin (exact distance ties, points on level-0 and level-1 cell faces)
             with exact duplicates, one point with 40 copies
  planar     every point at z = 0
  collinear  every point on the x axis
  outlier    the cfg2 map of one scan plus one point 2 km away: level-0 cells of 2 km / 1024
"""
import numpy as np

SCENES = ["cfg2", "clusters", "overflow", "ties", "planar", "collinear", "outlier"]


def _cfg2(frames):
    from oracle import icp_oracle as orc
    from pylidar_slam_b200 import synthetic as syn
    m = None
    for k in range(frames):
        s, _ = orc.grid_sample(syn.scan(k, 64, 2048), 0.3)
        s = np.asarray(s, np.float32)
        if m is not None:
            inv = np.linalg.inv(syn.gt_relative_pose(k).astype(np.float64))
            m = (m.astype(np.float64) @ inv[:3, :3].T + inv[:3, 3]).astype(np.float32)
            m = np.concatenate([m, s])
        else:
            m = s
    return m


def _overflow(seed=0):
    rng = np.random.RandomState(seed)
    g = np.arange(17) * 1.65
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    lattice = lattice + rng.uniform(-0.1, 0.1, lattice.shape)
    centres = rng.uniform(1.0, 25.0, (110, 3))
    clusters = (centres[:, None, :] + rng.normal(0.0, 0.45, (110, 30, 3))).reshape(-1, 3)
    return np.concatenate([lattice, clusters]).astype(np.float32)


def build(name):
    """(map [M, 3] float32, extra off-map query points [P, 3] float32)."""
    rng = np.random.RandomState(SCENES.index(name) + 11)
    if name == "cfg2":
        m = _cfg2(2)
        probes = m[rng.choice(len(m), 2000, replace=False)] + rng.normal(0, 0.5, (2000, 3)).astype(np.float32)
    elif name == "clusters":
        mid = rng.uniform(0, 30, (40, 3))[:, None, :] + rng.normal(0, 0.25, (40, 250, 3))
        dense = rng.uniform(0, 30, (20, 3))[:, None, :] + rng.normal(0, 0.12, (20, 500, 3))
        sparse = rng.uniform(0, 30, (3000, 3))
        m = np.concatenate([mid.reshape(-1, 3), dense.reshape(-1, 3), sparse]).astype(np.float32)
        probes = rng.uniform(-2, 32, (2000, 3)).astype(np.float32)
    elif name == "overflow":
        m = _overflow(0)
        probes = rng.uniform(-5, 35, (2000, 3)).astype(np.float32)
    elif name == "ties":
        g = np.arange(12, dtype=np.float32) * np.float32(0.25)
        lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
        dup = lat[rng.choice(len(lat), 300, replace=False)]
        many = np.repeat(lat[len(lat) // 2][None], 40, 0)
        m = np.concatenate([lat, dup, many, dup[:100]]).astype(np.float32)
        m = m[rng.permutation(len(m))]
        probes = (rng.randint(-2, 14, (1000, 3)) * 0.125).astype(np.float32)   # on and between lattice planes
    elif name == "planar":
        xy = rng.uniform(-20, 20, (20000, 2))
        m = np.concatenate([xy, np.zeros((len(xy), 1))], 1).astype(np.float32)
        probes = np.concatenate([rng.uniform(-22, 22, (1000, 2)), rng.normal(0, 1, (1000, 1))], 1).astype(np.float32)
    elif name == "collinear":
        x = np.sort(rng.uniform(-50, 50, 5000))
        m = np.stack([x, np.zeros_like(x), np.zeros_like(x)], 1).astype(np.float32)
        probes = np.stack([rng.uniform(-55, 55, 1000), rng.normal(0, 0.3, 1000), rng.normal(0, 0.3, 1000)], 1)
        probes = probes.astype(np.float32)
    elif name == "outlier":
        m = _cfg2(1)
        m = np.concatenate([m, np.array([[2000.0, 0.0, 0.0]], np.float32)])
        probes = m[rng.choice(len(m) - 1, 1000, replace=False)] + rng.normal(0, 1.0, (1000, 3)).astype(np.float32)
    else:
        raise KeyError(name)
    return np.ascontiguousarray(m, np.float32), np.ascontiguousarray(probes, np.float32)


def tiny(M, seed=0):
    """A map of M points (M = 1, 2, k, k + 1: the (k+1)-NN finds fewer than k + 1 points or exactly k + 1)."""
    rng = np.random.RandomState(seed + M)
    return rng.uniform(-1, 1, (M, 3)).astype(np.float32)
