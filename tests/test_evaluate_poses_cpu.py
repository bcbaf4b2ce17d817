"""pls_kdmap_evaluate_poses without a GPU: the float64 reference (oracle/evaluate_poses_reference.py) against a
brute-force nearest neighbour and against kd_icp_reference's first-iteration sums, RegistrationQuality's assembly of a
row, and ICPFrameToModel.evaluate_registrations over the host-logic stand-in (tests/dryrun_next_rows.FakeContext)
answering pls_kdmap_evaluate_poses as include/plslam_b200.h declares it."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import evaluate_poses_reference as er  # noqa: E402
from oracle import kd_icp_reference as kref  # noqa: E402
from oracle import projection_reference as pr  # noqa: E402

SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


def _pose(yaw, t):
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4, dtype=np.float32)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    return T


def _scene(seed=0, m=4000, n=600):
    rng = np.random.RandomState(seed)
    cloud = rng.uniform([-20, -20, -2], [20, 20, 3], (m, 3)).astype(np.float32)
    scan = cloud[rng.choice(m, n, replace=False)] + rng.normal(0, 0.05, (n, 3)).astype(np.float32)
    return cloud, scan.astype(np.float32)


@pytest.mark.parametrize("max_distance", [0.0, 0.05, 0.2, 1.0, np.inf])
def test_reference_against_brute_force_nn(max_distance):
    cloud, scan = _scene()
    p = pr.transform32(_pose(0.03, [0.1, -0.05, 0.0]), scan)
    idx = cKDTree(cloud.astype(np.float64)).query(p.astype(np.float64))[1]
    d2_all = ((p.astype(np.float64)[:, None, :] - cloud.astype(np.float64)[None]) ** 2).sum(-1)
    brute = d2_all.argmin(1)
    np.testing.assert_array_equal(idx, brute)
    nrm = np.tile(np.float32([0, 0, 1]), (len(p), 1))
    row, keep = er.evaluate_row(p, cloud[idx], nrm, np.ones(len(p), bool), max_distance, "default", 1.0)
    exact = np.sqrt(d2_all.min(1)) <= max_distance
    # the reference's d^2 is the element-wise float64 expression; the brute force sums in another order
    near = np.abs(np.sqrt(d2_all.min(1)) - max_distance) < 1e-12
    assert np.array_equal(keep[~near], exact[~near])
    assert row[29] == keep.sum() and row[31] == len(p)
    np.testing.assert_allclose(row[30], er.match_d2(p[keep], cloud[idx][keep]).sum(), rtol=0, atol=0)


def test_unmatched_rows_are_never_inliers():
    p = np.zeros((3, 3), np.float32)
    q = np.full((3, 3), np.nan, np.float32)
    row, keep = er.evaluate_row(p, q, q, np.array([False, True, False]), np.inf, "default", 1.0)
    assert keep.tolist() == [False, False, False] and row[29] == 0 and row[31] == 3


def test_exact_gate_boundary_is_inclusive():
    """Dyadic offsets: d is exactly max_distance, so the row is an inlier."""
    p = np.float32([[0.5, 0.0, 0.0], [0.0, 0.75, 0.0], [0.0, 0.0, 0.625]])
    q = np.zeros_like(p)
    for md, want in ((0.5, [True, False, False]), (0.75, [True, True, True]), (0.625, [True, False, True])):
        _, keep = er.evaluate_row(p, q, np.tile(np.float32([1, 0, 0]), (3, 1)), np.ones(3, bool), md, "default", 1.0)
        assert keep.tolist() == want


@pytest.mark.parametrize("scheme", SCHEMES)
def test_reference_at_inf_is_the_first_icp_iteration(scheme):
    cloud, scan = _scene(1, 3000, 400)
    it = kref.kd_icp_iteration(cloud, scan, _pose(0.02, [0.2, 0.1, 0.0]), scheme, 0.3)
    m64 = cloud.astype(np.float64)
    row, keep = er.evaluate_row(it["p"], m64[it["match"]], it["normals"], np.ones(len(scan), bool), np.inf, scheme, 0.3)
    assert keep.all()
    np.testing.assert_array_equal(row[:30], it["sums"])
    assert row[31] == len(scan)


# ---------------------------------------------------------------------------------- RegistrationQuality assembly
def _row_from_terms(terms, d2, valid):
    row = np.zeros(32)
    row[:30] = terms.sum(0)
    row[30] = d2
    row[31] = valid
    return row


def test_quality_ratios_and_covariance():
    from pylidar_slam_b200.odometry import RegistrationQuality
    cloud, scan = _scene(2, 3000, 500)
    it = kref.kd_icp_iteration(cloud, scan, np.eye(4, dtype=np.float32), "default", 1.0)
    terms = kref.terms(it["p"], cloud.astype(np.float64)[it["match"]], it["normals"], "default", 1.0)
    d2 = er.match_d2(it["p"], cloud[it["match"]]).sum()
    q = RegistrationQuality.from_stats(_row_from_terms(terms, d2, 520))
    assert q.valid == 520 and q.inliers == 500
    assert q.fitness == pytest.approx(500 / 520)
    assert q.rmse == pytest.approx(np.sqrt(d2 / 500))
    assert q.plane_rmse == pytest.approx(np.sqrt(terms[:, 28].sum() / 500))
    H = q.information
    np.testing.assert_array_equal(H, H.T)
    J = np.concatenate([it["normals"], np.cross(it["p"], it["normals"])], 1)
    np.testing.assert_allclose(H, J.T @ J, rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(q.covariance, terms[:, 27].sum() / 494 * np.linalg.inv(H), rtol=1e-8)
    w, v = np.linalg.eigh(H)
    np.testing.assert_array_equal(q.eigenvalues, w)
    np.testing.assert_array_equal(q.eigenvectors, v)
    assert np.all(np.diff(q.eigenvalues) >= 0)


def test_quality_zero_denominators_and_few_inliers():
    from pylidar_slam_b200.odometry import RegistrationQuality
    q = RegistrationQuality.from_stats(np.zeros(32))
    assert q.valid == 0 and q.inliers == 0 and np.isnan(q.fitness) and np.isnan(q.rmse) and np.isnan(q.plane_rmse)
    assert q.covariance is None
    row = np.zeros(32)
    row[[0, 6, 11, 15, 18, 20]] = 1.0     # the identity information
    row[29], row[31], row[27] = 6, 10, 2.0
    q = RegistrationQuality.from_stats(row)
    assert q.fitness == 0.6 and q.covariance is None   # inliers <= 6
    row[29] = 7
    np.testing.assert_allclose(RegistrationQuality.from_stats(row).covariance, 2.0 * np.eye(6))


def test_quality_of_a_single_plane_is_rank_three():
    """Points on z = 0 with normal +z: J = [0, 0, 1, y, -x, 0] leaves tx, ty and rz free."""
    from pylidar_slam_b200.odometry import RegistrationQuality
    rng = np.random.RandomState(4)
    p = np.c_[rng.uniform(-10, 10, (200, 2)), np.zeros(200)].astype(np.float32)
    n = np.tile(np.float32([0, 0, 1]), (200, 1))
    terms = kref.terms(p, p, n, "default", 1.0)
    q = RegistrationQuality.from_stats(_row_from_terms(terms, 0.0, 200))
    assert np.linalg.matrix_rank(q.information) == 3
    assert q.covariance is None
    free = q.eigenvectors[:, :3]
    np.testing.assert_allclose(q.eigenvalues[:3], 0, atol=1e-9)
    for axis in (0, 1, 5):   # tx, ty, rz lie in the span of the three smallest
        e = np.zeros(6)
        e[axis] = 1.0
        np.testing.assert_allclose(np.linalg.norm(free.T @ e), 1.0, atol=1e-9)


# ---------------------------------------------------------------------------------- the Python entry point
PLANE = np.c_[np.mgrid[-5:5.5:0.5, -5:5.5:0.5].reshape(2, -1).T, np.zeros(441)].astype(np.float32)


@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext plus pls_kdmap_evaluate_poses over a fixed map (a 0.5 m grid on z = 0, normals +z), computed with
    the reference and a brute-force nearest neighbour.  The refusals are the library's."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class EvalFakeContext(dry.FakeContext):
        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def pls_kdmap_evaluate_poses(self, scans, n, S, scan_of, T, B, max_distance, out):
            if S <= 0 or B <= 0 or not T or not out or (not scan_of and B != S) or not (max_distance >= 0):
                return _lib.check(None, _lib.PLS_E_INVALID)
            rows = dry.arr(n, (S,), np.int64)
            addr = dry.arr(scans, (S,), np.uint64)
            of = dry.arr(scan_of, (B,), np.int32) if scan_of else np.arange(B)
            if np.any(rows <= 0) or np.any(addr == 0) or np.any((of < 0) | (of >= S)):
                return _lib.check(None, _lib.PLS_E_INVALID)
            poses = dry.arr(T, (B, 4, 4), np.float32)
            stats = dry.arr(out, (B, 32), np.float64)
            for b in range(B):
                s = dry.arr(int(addr[of[b]]), (int(rows[of[b]]), 3), np.float32)
                s = s[~np.isnan(s).any(1)]
                p = pr.transform32(poses[b], s)
                idx = ((p[:, None, :].astype(np.float64) - PLANE[None]) ** 2).sum(-1).argmin(1)
                nrm = np.tile(np.float32([0, 0, 1]), (len(p), 1))
                stats[b] = er.evaluate_row(p, PLANE[idx], nrm, np.ones(len(p), bool), max_distance, "default", 1.0)[0]

    monkeypatch.setattr(_lib, "Context", EvalFakeContext)
    monkeypatch.setattr(common, "_default_ctx", EvalFakeContext())
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = EvalFakeContext()
    odo.config = ICPFrameToModelConfig()
    return odo, calls


@pytest.mark.parametrize("form", ["numpy", "torch", "float64"])
def test_evaluate_registrations_conversions_and_outliers(stand_in, form):
    odo, calls = stand_in
    rng = np.random.RandomState(5)
    on = PLANE[rng.choice(len(PLANE), 40, replace=False)] + np.float32([0.01, -0.02, 0.0])
    off = on[:10] + np.float32([0, 0, 3.0])          # 10 outliers 3 m above the plane
    scan = np.concatenate([on, off, np.full((2, 3), np.nan, np.float32)])
    conv = {"numpy": lambda a: a, "torch": torch.from_numpy, "float64": lambda a: a.astype(np.float64)}[form]
    poses = np.tile(np.eye(4, dtype=np.float32), (3, 1, 1))
    poses[2, 2, 3] = 10.0                             # every row 10 m off the plane
    qs = odo.evaluate_registrations([conv(scan)], conv(poses), 1.0, conv(np.zeros(3, np.int64)))
    assert len(qs) == 3
    assert qs[0].valid == 50 and qs[0].inliers == 40 and qs[0].fitness == pytest.approx(0.8)
    d2 = np.float64(0.01) ** 2 + np.float64(0.02) ** 2
    assert qs[0].rmse == pytest.approx(np.sqrt(d2), rel=1e-5)
    assert qs[2].inliers == 0 and np.isnan(qs[2].rmse) and qs[2].covariance is None
    name, a = calls[-1]
    assert name == "pls_kdmap_evaluate_poses" and a[2] == 1 and a[5] == 3 and a[6] == 1.0
    every = odo.evaluate_registrations([scan], poses[:1])[0]
    assert every.inliers == 50 and calls[-1][1][3] is None and calls[-1][1][6] == np.inf


@pytest.mark.parametrize("bad", [dict(max_distance=-1.0), dict(max_distance=float("nan")),
                                 dict(scan_indices=[0, 1]), dict(poses=np.zeros((0, 4, 4), np.float32))])
def test_evaluate_registrations_refusals(stand_in, bad):
    odo, _ = stand_in
    args = dict(scans=[PLANE[:5]], poses=np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)), max_distance=1.0,
                scan_indices=[0, 0])
    args.update(bad)
    with pytest.raises((AssertionError, ValueError, RuntimeError)):
        odo.evaluate_registrations(**args)
