"""The eigenvalue-thresholded solve without a GPU: the kernels' 6x6 eigen-solver and projected step (eigen6_jacobi,
solve6_projected in eigen_device.cuh, built for the host by tests/degeneracy_harness.cu) against numpy.linalg.eigh and
the float64 oracle (oracle/degeneracy_reference.py) on random, rank-deficient, repeated-eigenvalue and J^T W J-scaled
matrices; the oracle on hand cases; the flat-field and tunnel scenes' eigenvalue gaps; and the Python routing of
min_eigenvalue over a stand-in backend."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import degeneracy_reference as dr  # noqa: E402
from oracle import kd_icp_reference as kref  # noqa: E402

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
EPS = 2.0 ** -52
# The eigen-solver's error bound, |lambda - lambda_ref| <= EIG_C eps ||H||_F, and the residual bound of its
# eigenvectors, ||H v - lambda v|| <= EIG_C eps ||H||_F: cyclic Jacobi on a 6x6 matrix makes a few dozen rotations, each
# with an error of a few eps ||H||_F; numpy's eigh has its own of the same order.  The largest ratio measured over the
# matrices below is 5.3 (test_eigen_bound_is_not_loose keeps the constant honest).
EIG_C = 16


@pytest.fixture(scope="module")
def dh(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    so = str(tmp_path_factory.mktemp("dh") / "degeneracy_harness.so")
    subprocess.check_call([NVCC, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
                           "-o", so, os.path.join(ROOT, "tests", "degeneracy_harness.cu")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def eigen6(dh, H):
    H = np.ascontiguousarray(H, np.float64).reshape(-1, 36)
    w, V = np.zeros((len(H), 6)), np.zeros((len(H), 36))
    dh.dh_eigen6(_p(H), C.c_int64(len(H)), _p(w), _p(V))
    return w, V.reshape(-1, 6, 6)


def projected(dh, sums, min_eigenvalue):
    sums = np.ascontiguousarray(sums, np.float64).reshape(-1, 30)
    dx, lam, kept = np.zeros((len(sums), 6)), np.zeros((len(sums), 6)), np.zeros(len(sums), np.int32)
    dh.dh_solve6_projected(_p(sums), C.c_int64(len(sums)), C.c_double(min_eigenvalue), _p(dx), _p(lam), _p(kept))
    return dx, lam, kept


def _random_rotations(rng, n):
    Q, R = np.linalg.qr(rng.normal(size=(n, 6, 6)))
    return Q * np.sign(np.diagonal(R, axis1=1, axis2=2))[:, None, :]


def _jtwj_sums(rng, n_points, radius):
    """The 30 accumulators of n_points point-to-plane rows at `radius` metres (unit normals, default scheme):
    translation entries about N, rotation entries about N radius^2."""
    p = rng.normal(size=(n_points, 3))
    p *= radius * rng.uniform(0.2, 1.0, (n_points, 1)) / np.linalg.norm(p, axis=1, keepdims=True)
    n = rng.normal(size=(n_points, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    q = p - n * rng.normal(0, 0.05, (n_points, 1))
    return kref.accumulate(p, q, n, "default", 0.3)


def _sums_of(H, g, N):
    s = np.zeros(30)
    s[:21] = [H[a, b] for a, b in kref._UPPER]
    s[21:27] = g
    s[28] = 1.0
    s[29] = N
    return s


def _matrices(kind, rng, count=200):
    if kind == "spd":
        A = rng.normal(size=(count, 6, 6))
        return A @ A.transpose(0, 2, 1)
    if kind.startswith("rank"):
        r = int(kind[4:])
        B = rng.normal(size=(count, 6, r))
        return B @ B.transpose(0, 2, 1)
    if kind == "repeated":
        Q = _random_rotations(rng, count)
        d = np.array([1.0, 1.0, 1.0, 2.0, 2.0, 5.0])
        return (Q * d[None, None, :]) @ Q.transpose(0, 2, 1)
    if kind == "jtwj":
        return np.array([dr.hessian(_jtwj_sums(rng, 500, 50.0)) for _ in range(count // 4)])
    raise ValueError(kind)


KINDS = ["spd", "rank1", "rank2", "rank3", "rank4", "rank5", "repeated", "jtwj"]


@pytest.mark.parametrize("kind", KINDS)
def test_eigen6_against_eigh(dh, kind):
    rng = np.random.RandomState(KINDS.index(kind) + 1)
    H = _matrices(kind, rng)
    w, V = eigen6(dh, H)
    w_ref = np.linalg.eigvalsh(H)
    fro = np.linalg.norm(H, axis=(1, 2))
    assert np.all(np.diff(w, axis=1) >= 0)                                   # ascending
    assert np.all(np.abs(w - w_ref) <= EIG_C * EPS * fro[:, None])
    res = np.linalg.norm(H @ V - V * w[:, None, :], axis=1)                  # per eigen-pair
    assert np.all(res <= EIG_C * EPS * fro[:, None])
    assert np.abs(V.transpose(0, 2, 1) @ V - np.eye(6)).max() <= EIG_C * EPS
    if kind.startswith("rank"):
        r = int(kind[4:])
        assert np.all(np.abs(w[:, :6 - r]) <= EIG_C * EPS * fro[:, None])


def test_eigen6_exact_zero_rows_stay_exact(dh):
    """H with exactly zero rows and columns (the flat field's tx, ty, rz): their eigenvalues are exactly 0 and the
    other eigenvectors exactly 0 there -- no rotation touches a zero row."""
    rng = np.random.RandomState(9)
    for _ in range(50):
        H = _matrices("spd", rng, 1)[0]
        for i in (0, 1, 5):
            H[i, :] = 0.0
            H[:, i] = 0.0
        w, V = eigen6(dh, H[None])
        assert list(w[0, :3]) == [0.0, 0.0, 0.0]
        assert np.all(V[0][[0, 1, 5]][:, 3:] == 0.0)


def test_eigen6_is_deterministic(dh):
    H = _matrices("jtwj", np.random.RandomState(4), 40)
    a, b = eigen6(dh, H), eigen6(dh, H[::-1].copy())
    assert a[0].tobytes() == b[0][::-1].tobytes() and a[1].tobytes() == b[1][::-1].tobytes()


def test_eigen_bound_is_not_loose(dh):
    """The bound is used with a margin a few times the worst measured error, not orders of magnitude."""
    worst = 0.0
    for kind in KINDS:
        H = _matrices(kind, np.random.RandomState(KINDS.index(kind) + 1))
        w, _ = eigen6(dh, H)
        worst = max(worst, (np.abs(w - np.linalg.eigvalsh(H)) / (EPS * np.linalg.norm(H, axis=(1, 2)))[:, None]).max())
    assert 0.0 < worst <= EIG_C / 2, worst


def _separated(lam_n, N, fro, thr):
    """No eigenvalue of H within the eigen-solver's bound of the threshold: the kept set is decided."""
    return np.all(np.abs(lam_n * N - thr * N) > 2 * EIG_C * EPS * fro)


@pytest.mark.parametrize("kind", ["spd", "rank2", "rank4", "jtwj"])
def test_projected_step_against_the_oracle(dh, kind):
    rng = np.random.RandomState(20 + KINDS.index(kind))
    H = _matrices(kind, rng, 100)
    checked = 0
    for i, h in enumerate(H):
        N = float(rng.randint(1, 5000))
        s = _sums_of(h, rng.normal(size=6) * np.sqrt(np.diag(h) + 1e-3), N)
        w_ref = np.linalg.eigvalsh(h) / N
        for thr in (w_ref[0] * 0.5 + 1e-300, (w_ref[1] + w_ref[2]) / 2, (w_ref[3] + w_ref[4]) / 2, w_ref[5] * 2):
            if thr <= 0 or not _separated(w_ref, N, np.linalg.norm(h), thr):
                continue
            step, kept, lam = dr.projected_step(s, thr)
            dx, lam_n, k = projected(dh, s, thr)
            assert k[0] == kept.sum(), (i, thr)
            np.testing.assert_allclose(lam_n[0], lam, rtol=0, atol=EIG_C * EPS * np.linalg.norm(h) / N)
            # the step's error, to first order: a backward error E of the decomposition (||E|| <= EIG_C eps ||H||_F)
            # moves the kept subspace by ||E|| / sep (sep: the distance of the kept eigenvalues to the others) and its
            # inverse by ||E|| / lambda_min_kept^2
            if kept.any():
                w_all = np.linalg.eigvalsh(h)
                wk, wd = w_all[kept], w_all[~kept]
                sep = np.abs(np.subtract.outer(wk, wd)).min() if wd.size else np.inf
                tol = 8 * EIG_C * EPS * np.linalg.norm(h) * np.linalg.norm(s[21:27]) / (wk.min() * min(wk.min(), sep))
                assert np.linalg.norm(dx[0] - step) <= tol, (i, thr, np.linalg.norm(dx[0] - step), tol)
            else:
                assert np.all(dx[0] == 0)
            checked += 1
    assert checked >= 100


def test_projected_step_full_rank_is_the_newton_step(dh):
    """With a threshold below every eigenvalue the projected step is -H^-1 g (kd_icp_reference.gauss_newton_step)."""
    rng = np.random.RandomState(31)
    for _ in range(50):
        s = _jtwj_sums(rng, 400, 30.0)
        step, kept, lam = dr.projected_step(s, 1e-12)
        assert kept.all()
        want = kref.gauss_newton_step(s)
        np.testing.assert_allclose(step, want, rtol=1e-8, atol=1e-12 * np.abs(want).max())
        dx, _, k = projected(dh, s, 1e-12)
        assert k[0] == 6
        np.testing.assert_allclose(dx[0], want, rtol=1e-8, atol=1e-12 * np.abs(want).max())


# ------------------------------------------------------------------------------------------------ oracle by hand
def test_oracle_by_hand():
    """H = diag(4, 0, 9, 1e-6, 2, 0) N, g = (1, 5, 3, 7, 2, 9), N = 10, threshold 0.5: kept tx, tz, ry."""
    N = 10.0
    H = np.diag([4.0, 0.0, 9.0, 1e-6, 2.0, 0.0]) * N
    g = np.array([1.0, 5.0, 3.0, 7.0, 2.0, 9.0])
    step, kept, lam = dr.projected_step(_sums_of(H, g, N), 0.5)
    assert list(kept) == [False, False, False, True, True, True]   # ascending: 0, 0, 1e-6, 2, 4, 9
    np.testing.assert_allclose(step, [-1 / 40, 0, -3 / 90, 0, -2 / 20, 0], rtol=1e-15)
    np.testing.assert_allclose(lam, [0, 0, 1e-6, 2, 4, 9], rtol=1e-15)
    # N = 0: nothing is kept, the eigenvalues are reported as zeros
    step, kept, lam = dr.projected_step(np.zeros(30), 0.5)
    assert not kept.any() and not step.any() and not lam.any()
    # a rotated H: the step along the kept eigenvector only
    c, s_ = np.cos(0.3), np.sin(0.3)
    R = np.eye(6)
    R[:2, :2] = [[c, -s_], [s_, c]]
    Hr = R @ np.diag([1e-9, 1.0, 1, 1, 1, 1]) @ R.T
    step, kept, _ = dr.projected_step(_sums_of(Hr, R[:, 0] * 3 + R[:, 1] * 2, 1.0), 1e-3)
    assert kept.sum() == 5
    np.testing.assert_allclose(step, -R[:, 1] * 2, atol=1e-15)


def test_device_code_on_the_hand_cases(dh):
    N = 10.0
    H = np.diag([4.0, 0.0, 9.0, 1e-6, 2.0, 0.0]) * N
    s = _sums_of(H, np.array([1.0, 5.0, 3.0, 7.0, 2.0, 9.0]), N)
    dx, lam, k = projected(dh, s, 0.5)
    assert k[0] == 3 and list(lam[0]) == [0, 0, 1e-6 * N / N, 2, 4, 9]
    assert list(dx[0]) == [-1 / 40, 0, -3 / 90, 0, -2 / 20, 0]
    dx, lam, k = projected(dh, np.zeros(30), 0.5)
    assert k[0] == 0 and not dx.any() and not lam.any()


# ------------------------------------------------------------------------------------------------ scenes
def test_flat_field_is_exactly_degenerate_in_x_y_yaw():
    m, s, truth, start = dr.flat_field_scene(0, 40000, 4000)
    assert not m[:, 2].any() and not s[:, 2].any()
    sums = dr.sums_at(m, s, start)
    H = dr.hessian(sums)
    assert np.all(np.abs(H[[0, 1, 5]]) <= 1e-12 * np.abs(H).max())
    step, kept, lam = dr.projected_step(sums, dr.FLAT_MIN_EIGENVALUE)
    assert kept.sum() == 3 and np.all(lam[3:] > 100 * dr.FLAT_MIN_EIGENVALUE)
    assert np.all(np.abs(step[[0, 1, 5]]) <= 1e-12)


def test_tunnel_eigenvalue_gap():
    """At the truth and at the start, exactly one eigenvalue of H / N (the translation along the axis) lies below
    TUNNEL_MIN_EIGENVALUE, with a factor of 4 of margin on either side."""
    m, s, truth, start = dr.tunnel_scene(0, 60000, 8000)
    for T in (truth, start):
        sums = dr.sums_at(m, s, T)
        step, kept, lam = dr.projected_step(sums, dr.TUNNEL_MIN_EIGENVALUE)
        assert kept.sum() == 5
        assert lam[0] < dr.TUNNEL_MIN_EIGENVALUE / 4 and lam[1] > dr.TUNNEL_MIN_EIGENVALUE * 4, lam
        v = np.linalg.eigh(dr.hessian(sums))[1][:, 0]
        assert abs(v[0]) > 0.99, v   # the degenerate direction is x


# ------------------------------------------------------------------------------------------------ Python routing
@pytest.fixture
def stand_in(monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class DegenFakeContext(dry.FakeContext):
        M = 4

        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def _answer(self, B, out_T, out_iters, out_status):
            dry.arr(out_T, (B, 4, 4), np.float32)[:] = np.eye(4, dtype=np.float32)
            dry.arr(out_iters, (B,), np.int32)[:] = 1
            dry.arr(out_status, (B,), np.int32)[:] = _lib.PLS_OK

        def pls_register_scans(self, scans, n, S, scan_of, T0s, B, out_T, out_params, out_losses, out_iters,
                               out_status):
            self._answer(B, out_T, out_iters, out_status)

        def pls_register_scans_gated(self, scans, n, S, scan_of, T0s, B, max_distance, out_T, out_params, out_losses,
                                     out_iters, out_status, out_inliers):
            self._answer(B, out_T, out_iters, out_status)
            dry.arr(out_inliers, (B,), np.int32)[:] = np.arange(B) + 100

        def pls_register_scans_degeneracy(self, scans, n, S, scan_of, T0s, B, max_distance, min_eigenvalue, out_T,
                                          out_params, out_losses, out_iters, out_status, out_inliers, out_degenerate,
                                          out_eigenvalues):
            self._answer(B, out_T, out_iters, out_status)
            if out_inliers:
                dry.arr(out_inliers, (B,), np.int32)[:] = np.arange(B) + 100
            dry.arr(out_degenerate, (B,), np.int32)[:] = np.arange(B) % 7
            dry.arr(out_eigenvalues, (B, 6), np.float64)[:] = np.arange(6) + 0.5

        def pls_register_hypotheses(self, points, n, T0s, B, out_T, out_params, out_losses, out_iters, out_status):
            self._answer(B, out_T, out_iters, out_status)

    monkeypatch.setattr(_lib, "Context", DegenFakeContext)
    monkeypatch.setattr(common, "_default_ctx", DegenFakeContext())
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = DegenFakeContext()
    odo.ctx.cfg.local_map_type = _lib.MAP_KDTREE
    odo.config = ICPFrameToModelConfig(max_num_alignments=DegenFakeContext.M)
    return odo, calls, _lib


def _inputs(B=3):
    rng = np.random.RandomState(0)
    return [rng.randn(50, 3).astype(np.float32), rng.randn(40, 3).astype(np.float32)], \
        np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))


def test_zero_makes_the_calls_made_without_it(stand_in):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    odo.register_new_frames(scans, T0, [0, 1, 0], min_eigenvalue=0.0)
    odo.register_new_frames(scans, T0, [0, 1, 0], max_distance=0.5, min_eigenvalue=0.0)
    odo.register_new_frame_hypotheses(scans[0], T0, min_eigenvalue=0.0)
    odo.register_new_frame_hypotheses(scans[0], T0, max_distance=0.5)
    assert [c[0] for c in calls] == ["pls_register_scans", "pls_register_scans_gated", "pls_register_hypotheses",
                                     "pls_register_scans_gated"]
    assert odo.last_registrations_degenerate is None and odo.last_registrations_eigenvalues is None
    assert odo.last_hypotheses_degenerate is None and odo.last_hypotheses_eigenvalues is None


@pytest.mark.parametrize("max_distance", [np.inf, 0.75])
def test_positive_calls_the_degeneracy_entry_point(stand_in, max_distance):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    odo.register_new_frames(scans, T0, [0, 1, 0], max_distance=max_distance, min_eigenvalue=2e-3)
    name, a = calls[-1]
    assert name == "pls_register_scans_degeneracy" and a[2] == 2 and a[5] == 3
    assert a[6] == max_distance and a[7] == 2e-3
    assert list(odo.last_registrations_degenerate) == [0, 1, 2]
    assert odo.last_registrations_eigenvalues.shape == (3, 6) and odo.last_registrations_eigenvalues[2, 5] == 5.5
    if np.isinf(max_distance):
        assert a[13] is None and odo.last_registrations_inliers is None   # ungated: no inlier output
    else:
        assert list(odo.last_registrations_inliers) == [100, 101, 102]
    calls.clear()
    odo.register_new_frame_hypotheses(scans[1], T0, max_distance=max_distance, min_eigenvalue=0.1)
    name, a = calls[-1]
    assert name == "pls_register_scans_degeneracy" and a[2] == 1 and a[7] == 0.1
    import dryrun_next_rows as dry
    assert list(dry.arr(a[3], (3,), np.int32)) == [0, 0, 0]
    assert list(odo.last_hypotheses_degenerate) == [0, 1, 2]
    assert odo.last_registrations_status is not odo.last_hypotheses_status


@pytest.mark.parametrize("bad", [-1e-3, float("nan"), -np.inf, np.inf])
def test_refusals_raise_before_any_call(stand_in, bad):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    with pytest.raises(Exception):
        odo.register_new_frames(scans, T0, [0, 1, 0], min_eigenvalue=bad)
    with pytest.raises(Exception):
        odo.register_new_frame_hypotheses(scans[0], T0, min_eigenvalue=bad)
    assert calls == []


def test_positive_on_a_projective_map_raises_before_any_call(stand_in):
    odo, calls, lib = stand_in
    odo.ctx.cfg.local_map_type = lib.MAP_PROJECTIVE
    scans, T0 = _inputs()
    with pytest.raises(Exception):
        odo.register_new_frame_hypotheses(scans[0], T0, min_eigenvalue=1e-3)
    odo.register_new_frame_hypotheses(scans[0], T0)
    assert [c[0] for c in calls] == ["pls_register_hypotheses"]


def test_localize_passes_the_threshold_to_its_refinement_only(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry as od
    odo, calls, _ = stand_in
    seen = []
    T0 = np.tile(np.eye(4), (2, 1, 1))
    monkeypatch.setattr(od, "_pose_search", lambda *a, **k: (seen.append(("search", a[1:], k)), (T0, np.zeros(2), None))[1])
    monkeypatch.setattr(od, "_score_poses", lambda *a, **k: (seen.append(("score", a[1:], k)), np.zeros(2, np.int32))[1])
    monkeypatch.setattr(od, "_pose_candidates", lambda *a: list(a))
    scan = _inputs()[0][0]
    odo.localize(scan, np.eye(4), 2.0, 0.5)
    odo.localize(scan, np.eye(4), 2.0, 0.5, min_eigenvalue=1e-3)
    assert [s[0] for s in seen] == ["search", "score", "search", "score"]
    assert repr(seen[0]) == repr(seen[2]) and repr(seen[1][2]) == repr(seen[3][2])   # the search: the same call
    assert [c[0] for c in calls] == ["pls_register_hypotheses", "pls_register_scans_degeneracy"]
    assert calls[1][1][7] == 1e-3
    with pytest.raises(Exception):
        odo.localize(scan, np.eye(4), 2.0, 0.5, min_eigenvalue=-1.0)
    assert len(seen) == 4   # refused before the search


def test_localize_scans_passes_the_threshold_to_its_refinement_only(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry as od
    odo, calls, _ = stand_in
    T0 = np.tile(np.eye(4), (2, 1, 1))
    searched = []
    monkeypatch.setattr(od, "_pose_search_scans",
                        lambda ctx, scans, bases, cell, halves, num, out_scores=None:
                        searched.append(num) or [(T0, np.zeros(2), None) for _ in scans])
    monkeypatch.setattr(od, "_pose_candidates", lambda *a: list(a))
    scans = _inputs()[0]
    odo.localize_scans(scans, np.tile(np.eye(4), (2, 1, 1)), 2.0, 0.5, min_eigenvalue=5e-4)
    assert [c[0] for c in calls] == ["pls_register_scans_degeneracy"] and calls[0][1][7] == 5e-4
    with pytest.raises(Exception):
        odo.localize_scans(scans, np.tile(np.eye(4), (2, 1, 1)), 2.0, 0.5, min_eigenvalue=float("nan"))
    assert len(searched) == 2   # the search and the rescoring of the first call; the refused one made none
