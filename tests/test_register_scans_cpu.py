"""ICPFrameToModel.register_new_frames without a GPU: the mirror's conversions, scan_indices, status and logging over the
host-logic stand-in (tests/dryrun_next_rows.FakeContext) answering pls_register_scans as include/plslam_b200.h
declares it, and the refusals of the map's given normals."""
import logging
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext plus pls_register_scans.  Registration b answers with values that name its scan and estimate: T is
    T0s[b] moved by the mean of its scan's valid rows, params[:, 0] its scan index, iters the scan's valid row count
    (at most max_num_alignments), status PLS_E_SINGULAR for a one-row scan.  The refusals are the library's."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class ScansFakeContext(dry.FakeContext):
        M = 5

        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def pls_register_scans(self, scans, n, S, scan_of, T0s, B, out_T, out_params, out_losses, out_iters,
                               out_status):
            if S <= 0 or B <= 0 or not T0s or (not scan_of and B != S):
                return _lib.check(None, _lib.PLS_E_INVALID)
            rows = dry.arr(n, (S,), np.int64)
            addr = dry.arr(scans, (S,), np.uint64)
            of = dry.arr(scan_of, (B,), np.int32) if scan_of else np.arange(B)
            if np.any(rows <= 0) or np.any(addr == 0) or np.any((of < 0) | (of >= S)):
                return _lib.check(None, _lib.PLS_E_INVALID)
            pts = [dry.arr(int(addr[s]), (int(rows[s]), 3), np.float32) for s in range(S)]
            T = dry.arr(T0s, (B, 4, 4), np.float32).copy()
            for b in range(B):
                p = pts[of[b]]
                valid = p[~np.isnan(p).any(1)]
                T[b, :3, 3] += valid.mean(0) if len(valid) else 0.0
                dry.arr(out_params, (B, 6), np.float32)[b] = [of[b], b, 0, 0, 0, 0]
                it = min(len(valid), self.M)
                dry.arr(out_iters, (B,), np.int32)[b] = it
                dry.arr(out_losses, (B, self.M), np.float32)[b] = np.arange(self.M) + 10 * b
                dry.arr(out_status, (B,), np.int32)[b] = _lib.PLS_E_SINGULAR if p.shape[0] == 1 else _lib.PLS_OK
            dry.arr(out_T, (B, 4, 4), np.float32)[:] = T

    monkeypatch.setattr(_lib, "Context", ScansFakeContext)
    monkeypatch.setattr(common, "_default_ctx", ScansFakeContext())
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = ScansFakeContext()
    odo.config = ICPFrameToModelConfig(max_num_alignments=ScansFakeContext.M)
    return odo, calls


def _scans(sizes, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randn(n, 3).astype(np.float32) for n in sizes]


def _T0s(B):
    T0 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    T0[:, 0, 3] = np.arange(B)
    return T0


def _expected_T(scans, T0s, of):
    T = T0s.copy()
    for b, s in enumerate(of):
        p = scans[s].astype(np.float32)
        T[b, :3, 3] += p[~np.isnan(p).any(1)].mean(0)
    return T


@pytest.mark.parametrize("form", ["numpy", "torch", "float64"])
def test_conversions_and_scan_indices(stand_in, form):
    odo, calls = stand_in
    scans = _scans([4, 7, 3])
    scans[1][2] = np.nan
    of = np.array([2, 0, 1, 1, 2], np.int64)
    T0s = _T0s(5)
    conv = {"numpy": lambda a: a, "torch": torch.from_numpy, "float64": lambda a: a.astype(np.float64)}[form]
    params, T, losses, iters = odo.register_new_frames([conv(s) for s in scans], conv(T0s), conv(of))
    assert params.shape == (5, 6) and T.shape == (5, 4, 4) and iters.shape == (5,)
    assert params.dtype == np.float32 and T.dtype == np.float32
    np.testing.assert_array_equal(params[:, 0], of)
    np.testing.assert_allclose(T, _expected_T(scans, T0s, of), rtol=1e-6)
    assert list(iters) == [3, 4, 5, 5, 3]
    assert [len(l) for l in losses] == list(iters) and losses[1] == list(np.arange(4, dtype=np.float32) + 10)
    assert odo.last_registrations_status.tolist() == [0] * 5
    name, a = calls[-1]
    assert name == "pls_register_scans" and a[2] == 3 and a[5] == 5


def test_no_scan_indices_is_one_registration_per_scan(stand_in):
    odo, calls = stand_in
    scans = _scans([3, 8])
    params, T, losses, iters = odo.register_new_frames(scans, _T0s(2))
    np.testing.assert_array_equal(params[:, 0], [0, 1])
    assert calls[-1][1][3] is None   # scan_of = NULL
    with pytest.raises(AssertionError):   # the library's refusal: B != S without scan_indices
        odo.register_new_frames(scans, _T0s(3))


def test_status_and_logging(stand_in, caplog):
    odo, _ = stand_in
    scans = _scans([6, 1, 9])
    with caplog.at_level(logging.ERROR):
        odo.register_new_frames(scans, _T0s(4), [0, 1, 2, 1])
    from pylidar_slam_b200 import _lib
    assert odo.last_registrations_status.tolist() == [_lib.PLS_OK, _lib.PLS_E_SINGULAR, _lib.PLS_OK, _lib.PLS_E_SINGULAR]
    msgs = [r.getMessage() for r in caplog.records if r.levelno == logging.ERROR]
    assert len(msgs) == 1 and "registrations [1, 3]" in msgs[0] and "not invertible" in msgs[0]


def test_argument_checks(stand_in):
    odo, calls = stand_in
    scans = _scans([4, 5])
    n = len(calls)
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        odo.register_new_frames([scans[0], scans[1][:, :2]], _T0s(2))
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        odo.register_new_frames(scans, _T0s(2)[:, :3])
    with pytest.raises(AssertionError, match="one scan index per initial estimate"):
        odo.register_new_frames(scans, _T0s(2), [0, 1, 1])
    assert len(calls) == n   # refused before the library is called
    for bad in ([0, 2], [-1, 0]):
        with pytest.raises(AssertionError):
            odo.register_new_frames(scans, _T0s(2), bad)
    with pytest.raises(AssertionError):
        odo.register_new_frames([], _T0s(1))


def test_given_normals_raise_the_reference_index_error(stand_in):
    odo, calls = stand_in
    from pylidar_slam_b200.odometry import _NORMALS_INDEX_ERROR, _set_given_normals
    _set_given_normals(odo.ctx, True)
    n = len(calls)
    with pytest.raises(IndexError, match=_NORMALS_INDEX_ERROR):
        odo.register_new_frames(_scans([4]), _T0s(1))
    assert len(calls) == n
    _set_given_normals(odo.ctx, False)
    odo.register_new_frames(_scans([4]), _T0s(1))
    assert calls[-1][0] == "pls_register_scans"
