"""The pose search without a GPU: the float64 reference (oracle/pose_search_reference.py) against a naive triple loop on
tiny hand-made volumes, and KdTreeLocalMap.search_poses / score_poses and ICPFrameToModel.localize over the host-logic
stand-in (tests/dryrun_next_rows.FakeContext) answering pls_kdmap_pose_search as include/plslam_b200.h declares it."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pose_search_reference as ref  # noqa: E402


def _naive_volume(scan, bases, cell, hx, hy, map_points):
    occ = {tuple(int(v) for v in np.rint(np.float64(p) / cell)) for p in np.asarray(map_points, np.float32)}
    out = np.zeros((len(bases), 2 * hy + 1, 2 * hx + 1), np.int32)
    for a, T in enumerate(bases):
        for p in np.asarray(scan, np.float32):
            if not np.isfinite(p).all():
                continue
            x, y, z = (float(v) for v in p)
            c = [int(np.rint((((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]) / cell)) for r in range(3)]
            for j in range(-hy, hy + 1):
                for i in range(-hx, hx + 1):
                    out[a, j + hy, i + hx] += (c[0] + i, c[1] + j, c[2]) in occ
    return out


def _naive_candidates(vol):
    A, Wy, Wx = vol.shape
    L = np.arange(vol.size).reshape(vol.shape)
    keep = []
    for a in range(A):
        for j in range(Wy):
            for i in range(Wx):
                s = vol[a, j, i]
                if s <= 0:
                    continue
                nb = [(vol[b, jj, ii], L[b, jj, ii]) for b in range(max(a - 1, 0), min(a + 2, A))
                      for jj in range(max(j - 1, 0), min(j + 2, Wy)) for ii in range(max(i - 1, 0), min(i + 2, Wx))
                      if (b, jj, ii) != (a, j, i)]
                if all(s > sn or (s == sn and L[a, j, i] < ln) for sn, ln in nb):
                    keep.append((-int(s), int(L[a, j, i])))
    return [l for _, l in sorted(keep)]


def test_reference_scores_equal_the_naive_loop():
    rng = np.random.RandomState(0)
    m = rng.uniform(-3, 3, (300, 3)).astype(np.float32)
    scan = rng.uniform(-2, 2, (40, 3)).astype(np.float32)
    scan[3, 1], scan[7] = np.nan, [np.inf, 0, 0]
    scan[9] = [0.25, -0.75, 0.25]             # half cells at c = 0.5: round half to even both ways
    th = rng.uniform(-3, 3, 3)
    bases = np.tile(np.eye(4), (3, 1, 1))
    bases[:, 0, 0], bases[:, 0, 1], bases[:, 1, 0], bases[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    bases[:, :3, 3] = rng.uniform(-1, 1, (3, 3))
    for cell, hx, hy in ((0.5, 2, 1), (1.0, 0, 0), (0.3, 1, 3)):
        assert np.array_equal(ref.score_volume(scan, bases, cell, hx, hy, m), _naive_volume(scan, bases, cell, hx, hy, m))


@pytest.mark.parametrize("vol", [
    np.array([[[1, 1, 0], [0, 0, 2]]]),                              # plateau of two: the lower L wins
    np.array([[[3, 3], [3, 3]], [[3, 3], [3, 3]]]),                  # one plateau over a: only L = 0
    np.array([[[0, 0, 0]], [[0, 0, 0]]]),                            # all zero: no candidate
    np.array([[[5, 0, 0, 0, 5]], [[0, 0, 0, 0, 0]], [[5, 0, 0, 0, 6]]]),  # edges, a = 0 and a = A - 1, no wrap
    np.array([[[2, 1, 2], [1, 2, 1]], [[2, 2, 2], [2, 2, 2]]]),
])
def test_reference_candidates_equal_the_naive_loop(vol):
    assert ref.candidates(vol.astype(np.int32)) == _naive_candidates(vol)


def test_reference_search_outputs():
    m = np.array([[1, 0, 0], [0, -1, 0], [3, 3, 0]], np.float32)
    scan = np.array([[0, 0, 0]], np.float32)
    bases = np.tile(np.eye(4), (2, 1, 1))
    bases[1, 2, 3] = 10.0
    vol, T, sc, ix, num = ref.search(scan, bases, 1.0, 1, 1, 8, m)
    # (a 0, j -1, i 0) and (a 0, j 0, i 1) are diagonal neighbours with equal scores: the lower L is the candidate
    assert num == 1 and sc.tolist() == [1] and ix.tolist() == [1]
    assert T[0, 1, 3] == -1.0 and T[0, 0, 3] == 0.0 and np.array_equal(T[0, :3, :3], np.eye(3))


@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext plus pls_kdmap_pose_search answered by the reference on a host map, and register_hypotheses that
    moves each T0 by a fixed offset (and marks one singular)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class SearchFakeContext(dry.FakeContext):
        M = 4
        map_points = np.zeros((0, 3), np.float32)
        singular = ()

        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def pls_kdmap_pose_search(self, scan, n, bases, A, cell, hx, hy, K, out_scores, out_T, out_score, out_index,
                                  out_num):
            if not scan or not bases or n <= 0 or A <= 0 or hx < 0 or hy < 0 or not 0 <= K <= 1024 or \
                    not np.isfinite(cell) or cell <= 0:
                return _lib.check(None, _lib.PLS_E_INVALID)
            s = dry.arr(scan, (n, 3), np.float32)
            b = dry.arr(bases, (A, 4, 4), np.float64)
            vol, T, sc, ix, num = ref.search(s, b, cell, hx, hy, K, self.map_points)
            if out_scores:
                dry.arr(out_scores, vol.shape, np.int32)[:] = vol
            if num:
                dry.arr(out_T, (num, 4, 4), np.float64)[:] = T
                dry.arr(out_score, (num,), np.int32)[:] = sc
                dry.arr(out_index, (num,), np.int64)[:] = ix
            out_num._obj.value = num

        def pls_register_hypotheses(self, pts, n, T0s, B, out_T, out_params, out_losses, out_iters, out_status):
            T = dry.arr(T0s, (B, 4, 4), np.float32).copy()
            T[:, 0, 3] += np.float32(0.5)
            dry.arr(out_T, (B, 4, 4), np.float32)[:] = T
            dry.arr(out_iters, (B,), np.int32)[:] = 3
            st = dry.arr(out_status, (B,), np.int32)
            st[:] = _lib.PLS_OK
            for b in self.singular:
                if b < B:
                    st[b] = _lib.PLS_E_SINGULAR

    monkeypatch.setattr(_lib, "Context", SearchFakeContext)
    monkeypatch.setattr(common, "_default_ctx", SearchFakeContext())
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig, KdTreeLocalMap, KdTreeLocalMapConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = SearchFakeContext()
    odo.config = ICPFrameToModelConfig(max_num_alignments=SearchFakeContext.M)
    km = KdTreeLocalMap(KdTreeLocalMapConfig(), ctx=odo.ctx)
    return odo, km, calls


def _grid_map():
    g = np.stack(np.meshgrid(np.arange(-6, 7), np.arange(-6, 7), [0], indexing="ij"), -1).reshape(-1, 3)
    keep = (np.abs(g[:, 0]) + 2 * np.abs(g[:, 1])) % 5 != 0
    return g[keep].astype(np.float32)


def test_search_and_score_poses_convert_their_inputs(stand_in):
    odo, km, calls = stand_in
    odo.ctx.map_points = _grid_map()
    scan = np.random.RandomState(2).uniform(-2, 2, (30, 3)).astype(np.float32)
    bases = np.tile(np.eye(4), (3, 1, 1))
    bases[1, 0, 3], bases[2, 1, 3] = 0.4, -0.6
    T, sc, ix = km.search_poses(scan, bases, 1.0, (2, 1), num_candidates=5)
    vol, wT, wsc, wix, wnum = ref.search(scan, bases, 1.0, 2, 1, 5, odo.ctx.map_points)
    assert T.dtype == np.float64 and sc.dtype == np.int32 and ix.dtype == np.int64
    assert np.array_equal(T, wT) and np.array_equal(sc, wsc) and np.array_equal(ix, wix) and T.shape == (wnum, 4, 4)
    # torch inputs, float32 bases: the same call
    T2, sc2, ix2 = km.search_poses(torch.from_numpy(scan), torch.from_numpy(bases.astype(np.float32)), 1.0, (2, 1), 5)
    assert np.array_equal(sc2, sc) and np.array_equal(ix2, ix)
    s = km.score_poses(scan, bases, 1.0)
    assert s.dtype == np.int32 and s.tolist() == ref.score_volume(scan, bases, 1.0, 0, 0, odo.ctx.map_points)[:, 0, 0].tolist()
    name, args = calls[-1]
    assert name == "pls_kdmap_pose_search" and args[5:8] == (0, 0, 0)
    with pytest.raises(AssertionError):
        km.search_poses(scan[:, :2], bases, 1.0, (1, 1))
    with pytest.raises(AssertionError):
        km.score_poses(scan, bases[:, :3], 1.0)
    with pytest.raises(AssertionError):
        km.search_poses(scan, bases, 0.0, (1, 1))


def test_yaw_sweep_rules():
    from pylidar_slam_b200.odometry import yaw_sweep
    prior = np.eye(4)
    prior[:3, :3] = [[1, 0, 0], [0, np.cos(0.1), -np.sin(0.1)], [0, np.sin(0.1), np.cos(0.1)]]  # a roll
    prior[:3, 3] = [5.0, -3.0, 1.5]
    full = yaw_sweep(prior, np.pi, np.deg2rad(7))
    A = int(np.ceil(2 * np.pi / np.deg2rad(7)))
    assert full.shape == (A, 4, 4)
    th = 2 * np.pi * np.arange(A) / A
    part = yaw_sweep(prior, np.deg2rad(20), np.deg2rad(6))
    assert part.shape == (7, 4, 4)
    for bases, theta in ((full, th), (part, (np.arange(7) - 3) * np.deg2rad(6))):
        for T, t in zip(bases, theta):
            Rz = np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1]])
            assert np.allclose(T[:3, :3], Rz @ prior[:3, :3], atol=1e-15, rtol=0)
            assert np.array_equal(T[:3, 3], prior[:3, 3]) and np.array_equal(T[3], [0, 0, 0, 1])
    assert yaw_sweep(prior, 0.0, 0.1).shape == (1, 4, 4)


def test_localize_ranks_by_status_then_score_then_rank(stand_in):
    odo, km, calls = stand_in
    odo.ctx.map_points = _grid_map()
    scan = np.random.RandomState(4).uniform(-3, 3, (40, 3)).astype(np.float32)
    odo.ctx.singular = (0,)
    res = odo.localize(scan, np.eye(4), radius=2.0, cell_size=1.0, yaw_range=np.deg2rad(10), yaw_step=np.deg2rad(5),
                       num_candidates=6)
    names = [c[0] for c in calls]
    assert names == ["pls_kdmap_pose_search", "pls_register_hypotheses", "pls_kdmap_pose_search"]
    assert calls[0][1][3] == 5 and calls[0][1][5:8] == (2, 2, 6)     # A = 2m + 1 = 5, half = ceil(2 / 1), K
    bases = __import__("pylidar_slam_b200.odometry", fromlist=["yaw_sweep"]).yaw_sweep(np.eye(4), np.deg2rad(10),
                                                                                         np.deg2rad(5))
    _, T0, coarse, _, num = ref.search(scan, bases, 1.0, 2, 2, 6, odo.ctx.map_points)
    assert len(res) == num > 1
    refined = T0.astype(np.float32)
    refined[:, 0, 3] += np.float32(0.5)
    rescored = ref.score_volume(scan, refined.astype(np.float64), 1.0, 0, 0, odo.ctx.map_points)[:, 0, 0]
    status = np.where(np.arange(num) == 0, 3, 0)
    want = sorted(range(num), key=lambda r: (status[r] == 3, -rescored[r], r))
    assert [c.coarse_rank for c in res] == want
    assert res[-1].coarse_rank == 0 and res[-1].status == 3
    for c in res:
        assert np.array_equal(c.T0, T0[c.coarse_rank]) and c.coarse_score == coarse[c.coarse_rank]
        assert np.array_equal(c.T, refined[c.coarse_rank].astype(np.float64)) and c.score == rescored[c.coarse_rank]
        assert c.iterations == 3


def test_localize_checks(stand_in):
    odo, km, calls = stand_in
    odo.ctx.map_points = np.array([[100, 100, 100]], np.float32)
    scan = np.zeros((5, 3), np.float32)
    assert odo.localize(scan, np.eye(4), 1.0, 1.0) == []          # no candidate: nothing to refine
    with pytest.raises(AssertionError):
        odo.localize(scan, np.eye(4), -1.0, 1.0)
    with pytest.raises(AssertionError):
        odo.localize(scan, np.eye(4), 1.0, 0.0)
    with pytest.raises(AssertionError):
        odo.localize(scan, np.eye(4), 1.0, 1.0, yaw_step=0.0)
    odo.ctx.kd_given_normals = True
    with pytest.raises(IndexError):
        odo.localize(scan, np.eye(4), 1.0, 1.0)
