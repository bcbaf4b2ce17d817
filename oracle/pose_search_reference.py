"""Float64 reference of pls_kdmap_pose_search (the correlative pose search on a kd map), for the tests.

Every quantity is written as explicit element-wise numpy expressions in the order include/plslam_b200.h fixes: no
matrix product (BLAS reorders and fuses), no fused multiply-add (numpy never contracts).  np.rint rounds half to even,
as the kernels' __double2ll_rn does.
"""
import numpy as np

_BIAS = 1 << 20  # cells are packed into one int64 key: |coordinate| < 2^20 on every axis


def valid_rows(scan: np.ndarray) -> np.ndarray:
    """The rows of scan [n,3] float32 with three finite coordinates (the multiset P)."""
    scan = np.asarray(scan, np.float32).reshape(-1, 3)
    return scan[np.isfinite(scan).all(axis=1)]


def map_cells(points: np.ndarray, cell: float) -> np.ndarray:
    """pls_voxel_hash's coordinates: rint(float64(p) / cell) per axis, int64 [m,3]."""
    return np.rint(np.asarray(points, np.float32).astype(np.float64) / np.float64(cell)).astype(np.int64)


def base_cells(points: np.ndarray, base: np.ndarray, cell: float) -> np.ndarray:
    """cell_a(p) for the valid rows `points` [n,3] and one base [4,4] float64: q = ((R0 x + R1 y) + R2 z) + t."""
    p = np.asarray(points, np.float32).astype(np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    T = np.asarray(base, np.float64).reshape(4, 4)
    out = np.empty((p.shape[0], 3), np.int64)
    for r in range(3):
        q = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
        out[:, r] = np.rint(q / np.float64(cell)).astype(np.int64)
    return out


def _keys(cells: np.ndarray) -> np.ndarray:
    assert np.all(np.abs(cells) < _BIAS), "the reference packs cells with |coordinate| < 2^20"
    c = cells + _BIAS
    return (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]


def score_volume(scan, bases, cell, half_x, half_y, map_points) -> np.ndarray:
    """score[a, j + half_y, i + half_x] = #{p in P : cell_a(p) + (i, j, 0) in O}, int32 [A, 2 half_y + 1, 2 half_x + 1]."""
    P = valid_rows(scan)
    bases = np.asarray(bases, np.float64).reshape(-1, 4, 4)
    A, Wy, Wx = bases.shape[0], 2 * half_y + 1, 2 * half_x + 1
    out = np.zeros((A, Wy, Wx), np.int32)
    if P.shape[0] == 0 or len(map_points) == 0:
        return out
    m = map_cells(map_points, cell)
    occupied = np.unique(_keys(m[np.all(np.abs(m) < _BIAS, axis=1)]))
    # a shift (i, j) adds i << 42 and j << 21 to a packed key: no carry while every shifted cell stays packable
    j, i = np.meshgrid(np.arange(-half_y, half_y + 1), np.arange(-half_x, half_x + 1), indexing="ij")
    shifts = ((i.astype(np.int64) << 42) + (j.astype(np.int64) << 21)).reshape(-1)
    for a in range(A):
        cells = base_cells(P, bases[a], cell)
        assert np.all(np.abs(cells) + max(half_x, half_y) < _BIAS), "the reference packs cells with |coordinate| < 2^20"
        keys = _keys(cells)
        hits = np.isin(keys[None, :] + shifts[:, None], occupied)
        out[a] = np.count_nonzero(hits, axis=1).reshape(Wy, Wx)
    return out


def candidates(volume: np.ndarray) -> list:
    """The L of every candidate, in key order: score > 0 and (score, -L) strictly greater than each existing
    neighbour's in the 3x3x3 block (a +- 1 without wrap-around, i +- 1, j +- 1, clipped)."""
    A, Wy, Wx = volume.shape
    flat = volume.reshape(-1)
    found = []
    for a, jj, ii in zip(*np.nonzero(volume > 0)):
        L = (a * Wy + jj) * Wx + ii
        s = int(flat[L])
        peak = True
        for da in (-1, 0, 1):
            for dj in (-1, 0, 1):
                for di in (-1, 0, 1):
                    if (da, dj, di) == (0, 0, 0):
                        continue
                    b, j, i = a + da, jj + dj, ii + di
                    if not (0 <= b < A and 0 <= j < Wy and 0 <= i < Wx):
                        continue
                    Ln = (b * Wy + j) * Wx + i
                    sn = int(flat[Ln])
                    if sn > s or (sn == s and Ln < L):
                        peak = False
        if peak:
            found.append((-s, int(L)))
    found.sort()
    return [L for _, L in found]


def search(scan, bases, cell, half_x, half_y, K, map_points):
    """What pls_kdmap_pose_search returns: (volume, T [k,4,4], score [k], index [k], num)."""
    volume = score_volume(scan, bases, cell, half_x, half_y, map_points)
    bases = np.asarray(bases, np.float64).reshape(-1, 4, 4)
    Wy, Wx = 2 * half_y + 1, 2 * half_x + 1
    top = candidates(volume)[:K]
    T = np.zeros((len(top), 4, 4), np.float64)
    score = np.zeros(len(top), np.int32)
    for c, L in enumerate(top):
        a, rem = divmod(L, Wy * Wx)
        jj, ii = divmod(rem, Wx)
        T[c] = bases[a]
        T[c, 0, 3] = bases[a, 0, 3] + np.float64(ii - half_x) * np.float64(cell)
        T[c, 1, 3] = bases[a, 1, 3] + np.float64(jj - half_y) * np.float64(cell)
        score[c] = volume.reshape(-1)[L]
    return volume, T, score, np.array(top, np.int64), len(top)
