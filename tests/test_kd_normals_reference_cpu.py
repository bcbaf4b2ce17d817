"""The reference of the kd map's (k+1)-NN lists and normals (oracle/kd_icp_reference.py: kernel_sort_positions,
knn_lists, reference_covs, tight_normal_bound), pinned on the CPU: its moments are the oracle's bit for bit, its
normals the goldens', its sort positions follow the index build's quantisation, and the eigen-solver the kernels run
(eigen_device.cuh, through tests/host_harness.cu) meets its tight bound on every scene of the GPU tests."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import icp_oracle as orc
from oracle import kd_icp_reference as ref
from oracle import kd_normals_scenes as scenes
from test_host_math import hh  # noqa: F401  (the host harness fixture)


def _svd_normals(covs):
    return np.linalg.svd(covs)[2][:, 2, :]


@pytest.mark.parametrize("source", ["synthetic", "golden"])
def test_reference_covs_are_the_oracle_moments_bit_for_bit(source, golden_helpers):
    """reference_covs on cKDTree's own lists gives the oracle's moments: the oracle's SVD of them returns its normals
    bit for bit.  The kernel's sequential float32 sum in list order is the same numbers."""
    if source == "golden":
        m = golden_helpers["kd_map"]
    else:
        m, _ = scenes.build("outlier")
    k = 10
    lm = orc.KdTreeLocalMap(local_map_size=1, num_neighbors_normals=k)
    lm.update(np.eye(4, dtype=np.float32), new_points=m)
    _, nrm, idx = lm.nearest_neighbor_search(m)
    _, lists = cKDTree(lm.points).query(lm.points[idx], k=k + 1)
    covs = ref.reference_covs(lm.points, idx, lists, k)
    assert covs.dtype == np.float32
    assert np.array_equal(_svd_normals(covs).view(np.uint32), nrm.view(np.uint32))
    # warp_second_moments' order: sequential float32 sums over entries 1..k, then one division by k
    d = lm.points[lists[:, 1:]] - lm.points[idx][:, None, :]
    acc = np.zeros((len(idx), 3, 3), np.float32)
    for j in range(k):
        acc = acc + d[:, j, :, None] * d[:, j, None, :]
    assert np.array_equal(acc / np.float32(k), covs)


def test_normals_from_the_reference_lists_match_the_golden(golden_helpers):
    g = golden_helpers
    m, q = g["kd_map"], g["kd_queries"]
    tree = cKDTree(m.astype(np.float64))
    _, match = tree.query(q.astype(np.float64))
    assert np.abs(m[match] - g["kd_nb"]).max() <= 2e-5
    pos = ref.kernel_sort_positions(m)
    lists, _, _, amb = ref.knn_lists(m, m[match], 10, pos, tree)
    v = np.linalg.eigh(ref.reference_covs(m, match, lists, 10).astype(np.float64))[1][:, :, 0]
    dots = np.abs((v * g["kd_normals"].astype(np.float64)).sum(1))
    assert np.mean(dots > 1 - 1e-4) > 0.99 and amb.mean() < 0.05


def test_kernel_sort_positions_on_a_hand_built_map():
    """scale = 40 (ext 100 m < 8191 / 40): a level-0 cell is 8 units = 0.2 m.  0.125 m -> 5 units (cell 0);
    float32(0.2) -> 8 units exactly, on the face of cell 1; 0.25 m -> 10 units (cell 1)."""
    p = np.array([[100, 0, 0],      # x cell 500: Morton spread(500)
                  [0.25, 0, 0],     # cell (1, 0, 0): id 1
                  [0, 0, 0.25],     # cell (0, 0, 1): id 4
                  [0.125, 0, 0],    # cell 0
                  [0.2, 0, 0],      # on the face: cell (1, 0, 0)
                  [0, 0.25, 0],     # cell (0, 1, 0): id 2
                  [0, 0, 0],        # cell 0
                  [0.2, 0.2, 0.2]], np.float32)  # cell (1, 1, 1): id 7
    mn, scale = ref.kernel_grid(p)
    assert scale == np.float32(40) and (mn == 0).all()
    assert ref.kernel_quantise(p, mn, scale)[4, 0] == 8
    # ids 0: rows 3, 6; id 1: rows 1, 4; id 2: row 5; id 4: row 2; id 7: row 7; spread(500): row 0
    assert ref.kernel_sort_positions(p).tolist() == [7, 2, 5, 0, 3, 4, 1, 6]
    # the clamp: scale = 8191 / 1000 and the far corner lands on (or, rounded down, next to) 8191: cell 1023
    c = np.array([[1000, 1000, 1000], [0, 0, 0], [1000, 0, 0], [0, 0, 999.9]], np.float32)
    mn, scale = ref.kernel_grid(c)
    assert scale == np.float32(8191) / np.float32(1000)
    q = ref.kernel_quantise(c, mn, scale)
    assert q.max() <= 8191 and (q[0] >> 3 == 1023).all()
    assert ref.kernel_sort_positions(c).tolist() == [3, 0, 1, 2]


def _sym(c6):
    M = np.zeros((len(c6), 3, 3))
    M[:, 0, 0], M[:, 0, 1], M[:, 0, 2], M[:, 1, 1], M[:, 1, 2], M[:, 2, 2] = np.asarray(c6, np.float64).T
    M[:, 1, 0], M[:, 2, 0], M[:, 2, 1] = M[:, 0, 1], M[:, 0, 2], M[:, 1, 2]
    return M


@pytest.mark.parametrize("name", scenes.SCENES)
def test_tight_bound_holds_for_the_device_eigen_solver(hh, name):  # noqa: F811
    """smallest_eigenvector (closed form, Jacobi fall-back) on the reference moments of every map point: within
    tight_normal_bound of float64 eigh wherever the gap exceeds 1e-9, in both solver ranges."""
    m, _ = scenes.build(name)
    pos = ref.kernel_sort_positions(m)
    tree = cKDTree(m.astype(np.float64))
    closed = jacobi = 0
    for k in (3, 10, 31):
        lists, _, _, _ = ref.knn_lists(m, m, k, pos, tree)
        covs = ref.reference_covs(m, np.arange(len(m)), lists, k)
        c6 = np.ascontiguousarray(covs.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]])
        out = np.empty((len(m), 3), np.float32)
        used = np.zeros(len(m), np.int32)
        hh.hh_smallest_eigenvectors(c6.ctypes.data_as(C.c_void_p), C.c_int64(len(m)), 0,
                                    out.ctypes.data_as(C.c_void_p), None)
        probe = np.empty_like(out)
        hh.hh_smallest_eigenvectors(c6.ctypes.data_as(C.c_void_p), C.c_int64(len(m)), 2,
                                    probe.ctypes.data_as(C.c_void_p), used.ctypes.data_as(C.c_void_p))
        C64 = _sym(c6)
        v = np.linalg.eigh(C64)[1][:, :, 0]
        bound, gap = ref.tight_normal_bound(C64)
        sin = np.linalg.norm(np.cross(out.astype(np.float64), v), axis=1)
        ok = gap > 1e-9
        assert np.isfinite(out).all() and np.abs(np.linalg.norm(out, axis=1) - 1).max() <= 1e-6
        assert (sin[ok] <= bound[ok]).all(), (name, k, float((sin[ok] / bound[ok]).max()))
        closed += int((ok & (used == 1)).sum())
        jacobi += int((ok & (used == 0)).sum())
    if name in ("cfg2", "clusters", "outlier"):
        assert closed >= 1000, closed
    if name in ("cfg2", "outlier"):  # scan-line rows and pillar edges: nearly degenerate planes
        assert jacobi >= 10, jacobi
