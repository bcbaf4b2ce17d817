"""The pruned pose search without a GPU: a numpy restatement of pls_kdmap_pose_search_pyramid (pooled grids, bounds,
threshold passes and the E_tau peak rule, include/plslam_b200.h) against the exhaustive reference
(oracle/pose_search_reference.py) on many small volumes, the pooled bounds against every covered score, and
_pose_search's choice between the two calls over a host stand-in."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pose_search_reference as ref  # noqa: E402

ROOT_SIDE = 16


def _next_tau(tau):
    return max(1, min(tau - 1, (3 * tau) // 4))


class Pyramid:
    """B_0 over the reachable box clipped to the map's cell box, B_k pooled from B_(k-1), and the bound of a node."""

    def __init__(self, scan, bases, cell, hx, hy, map_points, root_side=ROOT_SIDE):
        P = ref.valid_rows(scan)
        bases = np.asarray(bases, np.float64).reshape(-1, 4, 4)
        self.A, self.Wx, self.Wy, self.hx, self.hy = bases.shape[0], 2 * hx + 1, 2 * hy + 1, hx, hy
        self.kmax = 0
        while -(-max(self.Wx, self.Wy) // (1 << self.kmax)) > root_side:
            self.kmax += 1
        self.empty = P.shape[0] == 0 or len(map_points) == 0
        if self.empty:
            return
        self.cells = [ref.base_cells(P, bases[a], cell) for a in range(self.A)]
        m = ref.map_cells(map_points, cell)
        allc = np.concatenate(self.cells)
        half = np.array([hx, hy, 0])
        self.o = np.maximum(allc.min(0) - half, m.min(0))
        self.e = np.minimum(allc.max(0) + half, m.max(0)) - self.o + 1
        if np.any(self.e <= 0):
            self.empty = True
            return
        B = np.zeros(self.e[::-1], bool)  # [Z, Y, X]
        r = m - self.o
        keep = np.all((r >= 0) & (r < self.e), axis=1)
        B[r[keep, 2], r[keep, 1], r[keep, 0]] = True
        self.levels = [B]
        for k in range(1, self.kmax + 1):
            s, prev = 1 << (k - 1), self.levels[-1]
            nxt = prev.copy()
            nxt[:, :, :-s] |= prev[:, :, s:]
            nxt[:, :-s, :] |= prev[:, s:, :]
            nxt[:, :-s, :-s] |= prev[:, s:, s:]
            self.levels.append(nxt)

    def bound(self, a, I, J, k):
        """#{p : B_k(cell_a(p) - (hx, hy, 0) + (I 2^k, J 2^k)) set}; a block reaching into the grid from its low edge
        reads B_k at the edge (a superset), as the kernel does."""
        if self.empty:
            return 0
        c, span = self.cells[a], 1 << k
        X = c[:, 0] - self.hx - self.o[0] + (I << k)
        Y = c[:, 1] - self.hy - self.o[1] + (J << k)
        Z = c[:, 2] - self.o[2]
        X = np.where((X < 0) & (X + span > 0), 0, X)
        Y = np.where((Y < 0) & (Y + span > 0), 0, Y)
        inside = (X >= 0) & (X < self.e[0]) & (Y >= 0) & (Y < self.e[1]) & (Z >= 0) & (Z < self.e[2])
        return int(np.count_nonzero(self.levels[k][Z[inside], Y[inside], X[inside]]))

    def children(self, a, I, J, k):
        return [(a, 2 * I + dx, 2 * J + dy) for dy in (0, 1) for dx in (0, 1)
                if ((2 * I + dx) << (k - 1)) < self.Wx and ((2 * J + dy) << (k - 1)) < self.Wy]

    def roots(self):
        s = 1 << self.kmax
        return [(a, I, J) for a in range(self.A) for J in range(-(-self.Wy // s)) for I in range(-(-self.Wx // s))]

    def top_bound(self):
        """The first threshold: the largest root bound, which no score exceeds."""
        return max([1] + [self.bound(*n, self.kmax) for n in self.roots()])

    def exact_set(self, tau):
        """E_tau: {L: score} of the poses with score >= tau, found by expanding nodes with bound >= tau."""
        nodes = [n for n in self.roots() if self.bound(*n, self.kmax) >= tau]
        for k in range(self.kmax, 0, -1):
            nodes = [c for n in nodes for c in self.children(*n, k) if self.bound(*c, k - 1) >= tau]
        E = {}
        for a, i, j in nodes:
            s = self.bound(a, i, j, 0)
            if s >= tau:
                E[(a * self.Wy + j) * self.Wx + i] = s
        return E

    def peaks(self, E):
        out = []
        for L, s in E.items():
            i, t = L % self.Wx, L // self.Wx
            j, a = t % self.Wy, t // self.Wy
            peak = True
            for da in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    for di in (-1, 0, 1):
                        if (da, dj, di) == (0, 0, 0) or not (0 <= a + da < self.A and 0 <= j + dj < self.Wy
                                                             and 0 <= i + di < self.Wx):
                            continue
                        Ln = L + (da * self.Wy + dj) * self.Wx + di
                        if Ln in E and (E[Ln] > s or (E[Ln] == s and Ln < L)):
                            peak = False
            if peak:
                out.append((-s, L))
        return sorted(out)


def pruned_search(scan, bases, cell, hx, hy, K, map_points, taus=None):
    """What pls_kdmap_pose_search_pyramid returns: (score [k], index [k]).  taus: the thresholds to try, in order
    (default: the largest root bound, then _next_tau); the last must be 1 or be met by K candidates."""
    pyr = Pyramid(scan, bases, cell, hx, hy, map_points)
    if pyr.empty:
        return np.zeros(0, np.int32), np.zeros(0, np.int64)
    if taus is None:
        taus = [pyr.top_bound()]
        while taus[-1] > 1:
            taus.append(_next_tau(taus[-1]))
    for tau in taus:
        top = pyr.peaks(pyr.exact_set(tau))
        if len(top) >= K or tau == 1:
            top = top[:K]
            return np.array([-s for s, _ in top], np.int32), np.array([L for _, L in top], np.int64)
    raise AssertionError("the schedule ended above 1 with fewer than K candidates")


def _rot_bases(A, rng, spread=1.0):
    th = rng.uniform(-np.pi, np.pi, A)
    B = np.tile(np.eye(4), (A, 1, 1))
    B[:, 0, 0], B[:, 0, 1], B[:, 1, 0], B[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    B[:, :3, 3] = rng.uniform(-spread, spread, (A, 3)) * [1, 1, 0.2]
    return B


def _check(scan, bases, cell, hx, hy, K, m, taus=None):
    _, _, want_sc, want_ix, num = ref.search(scan, bases, cell, hx, hy, K, m)
    sc, ix = pruned_search(scan, bases, cell, hx, hy, K, m, taus)
    assert ix.tolist() == want_ix.tolist() and sc.tolist() == want_sc.tolist(), (ix, want_ix, sc, want_sc)
    return num


@pytest.mark.parametrize("seed", range(12))
def test_pruned_search_equals_the_exhaustive_reference(seed):
    rng = np.random.RandomState(seed)
    A = int(rng.choice([1, 2, 3]))
    hx, hy = (int(v) for v in rng.choice([0, 1, 3, 7, 8, 9, 15, 16, 17], 2))  # windows of 2^k - 1, 2^k, 2^k + 1
    cell = float(rng.choice([0.5, 1.0]))
    m = rng.uniform([-6, -6, -1], [6, 6, 1], (int(rng.choice([20, 150, 600])), 3)).astype(np.float32)
    scan = rng.uniform([-2, -2, -0.8], [2, 2, 0.8], (int(rng.choice([1, 5, 30])), 3)).astype(np.float32)
    if scan.shape[0] > 3:
        scan[1, 0], scan[2] = np.nan, [np.inf, 0, 0]
    for K in (1, 3, 40):
        _check(scan, _rot_bases(A, rng), cell, hx, hy, K, m)


def test_plateaus_edges_and_empty_volumes():
    # a map row along x: every pose of the plateau ties, and the lowest L wins
    m = np.stack([np.arange(-10, 11), np.zeros(21), np.zeros(21)], 1).astype(np.float32)
    scan = np.zeros((1, 3), np.float32)
    bases = np.tile(np.eye(4), (3, 1, 1))
    assert _check(scan, bases, 1.0, 4, 2, 5, m) >= 1
    # peaks on window edges and at a = 0 and A - 1: a map point at each corner of the reachable box
    m = np.array([[-5, -3, 0], [5, 3, 0], [5, -3, 0], [-5, 3, 0]], np.float32)
    bases = np.tile(np.eye(4), (4, 1, 1))
    bases[1:3, 2, 3] = 7.0  # the middle bases see no map at all
    assert _check(scan, bases, 1.0, 5, 3, 16, m) == 8
    # all-zero volumes: a map out of reach, and a scan without a valid row
    assert _check(scan, bases, 1.0, 2, 2, 4, m + np.float32(50)) == 0
    bad = np.full((4, 3), np.nan, np.float32)
    bad[::2, 0] = np.inf
    assert _check(bad, bases, 1.0, 2, 2, 4, m) == 0


def test_threshold_schedules_agree():
    rng = np.random.RandomState(7)
    m = rng.uniform([-6, -6, -1], [6, 6, 1], (300, 3)).astype(np.float32)
    scan = rng.uniform([-2, -2, -0.8], [2, 2, 0.8], (25, 3)).astype(np.float32)
    bases = _rot_bases(2, rng)
    n_valid = ref.valid_rows(scan).shape[0]
    for taus in ([1], [n_valid, 1], list(range(n_valid, 0, -1)), [n_valid, n_valid // 2, 2, 1], None):
        for K in (1, 6, 200):
            _check(scan, bases, 0.5, 9, 8, K, m, taus)


def test_every_pooled_bound_covers_its_poses():
    rng = np.random.RandomState(3)
    m = rng.uniform([-6, -6, -1], [6, 6, 1], (200, 3)).astype(np.float32)
    scan = rng.uniform([-2, -2, -0.8], [2, 2, 0.8], (20, 3)).astype(np.float32)
    bases = _rot_bases(2, rng)
    hx, hy = 17, 11
    vol = ref.score_volume(scan, bases, 0.5, hx, hy, m)
    pyr = Pyramid(scan, bases, 0.5, hx, hy, m, root_side=2)
    assert pyr.kmax >= 4
    for k in range(pyr.kmax + 1):
        s = 1 << k
        for a in range(2):
            for J in range(-(-pyr.Wy // s)):
                for I in range(-(-pyr.Wx // s)):
                    covered = vol[a, J * s:(J + 1) * s, I * s:(I + 1) * s]
                    assert pyr.bound(a, I, J, k) >= covered.max(), (k, a, I, J)


@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext answering both search calls: the exhaustive one by the reference, the pyramid one by the
    restatement above (and nothing at all for volumes too large to restate)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class SearchFakeContext(dry.FakeContext):
        map_points = np.zeros((0, 3), np.float32)
        refuse = False

        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def pls_kdmap_pose_search(self, scan, n, bases, A, cell, hx, hy, K, out_scores, out_T, out_score, out_index,
                                  out_num):
            s, b = dry.arr(scan, (n, 3), np.float32), dry.arr(bases, (A, 4, 4), np.float64)
            vol, T, sc, ix, num = ref.search(s, b, cell, hx, hy, K, self.map_points)
            if out_scores:
                dry.arr(out_scores, vol.shape, np.int32)[:] = vol
            if num:
                dry.arr(out_T, (num, 4, 4), np.float64)[:] = T
                dry.arr(out_score, (num,), np.int32)[:] = sc
                dry.arr(out_index, (num,), np.int64)[:] = ix
            out_num._obj.value = num

        def pls_kdmap_pose_search_pyramid(self, scan, n, bases, A, cell, hx, hy, K, out_T, out_score, out_index,
                                          out_num):
            assert K >= 1
            if self.refuse:
                return _lib.check(None, _lib.PLS_E_INVALID)
            if A * (2 * hx + 1) * (2 * hy + 1) > 10_000:
                out_num._obj.value = 0
                return
            s, b = dry.arr(scan, (n, 3), np.float32), dry.arr(bases, (A, 4, 4), np.float64)
            sc, ix = pruned_search(s, b, cell, hx, hy, K, self.map_points)
            num = len(ix)
            Wx, Wy = 2 * hx + 1, 2 * hy + 1
            for c, L in enumerate(ix.tolist()):
                a, rem = divmod(L, Wy * Wx)
                jj, ii = divmod(rem, Wx)
                T = b[a].copy()
                T[0, 3] += np.float64(ii - hx) * np.float64(cell)
                T[1, 3] += np.float64(jj - hy) * np.float64(cell)
                dry.arr(out_T, (num, 4, 4), np.float64)[c] = T
            if num:
                dry.arr(out_score, (num,), np.int32)[:] = sc
                dry.arr(out_index, (num,), np.int64)[:] = ix
            out_num._obj.value = num

    monkeypatch.setattr(_lib, "Context", SearchFakeContext)
    monkeypatch.setattr(common, "_default_ctx", SearchFakeContext())
    from pylidar_slam_b200.odometry import KdTreeLocalMap, KdTreeLocalMapConfig
    ctx = SearchFakeContext()
    return KdTreeLocalMap(KdTreeLocalMapConfig(), ctx=ctx), ctx, calls


def test_pose_search_routes_by_the_pose_count(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry
    km, ctx, calls = stand_in
    assert odometry.POSE_SEARCH_PYRAMID_MIN_POSES > 125  # localize's 125-pose window in the exhaustive tests
    monkeypatch.setattr(odometry, "POSE_SEARCH_PYRAMID_MIN_POSES", 100)  # small volumes on both sides of it
    rng = np.random.RandomState(5)
    ctx.map_points = rng.uniform([-5, -5, -0.5], [5, 5, 0.5], (200, 3)).astype(np.float32)
    scan = rng.uniform([-2, -2, -0.3], [2, 2, 0.3], (15, 3)).astype(np.float32)
    bases = _rot_bases(3, rng)
    km.search_poses(scan, bases[:1], 0.5, (4, 4), 2)                   # 81 poses
    assert calls[-1][0] == "pls_kdmap_pose_search"
    km.search_poses(scan, bases[:2], 0.5, (4, 4), 2)                   # 162 poses
    assert calls[-1][0] == "pls_kdmap_pose_search_pyramid"
    assert calls[-1][1][3] == 2 and calls[-1][1][5:8] == (4, 4, 2) and len(calls[-1][1]) == 12
    # score_poses and K = 0 always take the exhaustive call
    km.score_poses(scan, np.tile(np.eye(4), (150, 1, 1)), 0.5)
    assert calls[-1][0] == "pls_kdmap_pose_search" and calls[-1][1][5:8] == (0, 0, 0)
    km.search_poses(scan, bases, 0.5, (4, 4), 0)
    assert calls[-1][0] == "pls_kdmap_pose_search"
    # the pyramid call converts its inputs as the exhaustive one does
    import torch
    T, sc, ix = km.search_poses(scan, bases, 0.5, (4, 3), 7)
    assert calls[-1][0] == "pls_kdmap_pose_search_pyramid"
    _, wT, wsc, wix, wnum = ref.search(scan, bases, 0.5, 4, 3, 7, ctx.map_points)
    assert T.dtype == np.float64 and sc.dtype == np.int32 and ix.dtype == np.int64 and T.shape == (wnum, 4, 4)
    assert np.array_equal(T, wT) and np.array_equal(sc, wsc) and np.array_equal(ix, wix)
    T2, sc2, ix2 = km.search_poses(torch.from_numpy(scan), torch.from_numpy(bases.astype(np.float32)), 0.5, (4, 3), 7)
    assert calls[-1][0] == "pls_kdmap_pose_search_pyramid"
    _, _, wsc2, wix2, _ = ref.search(scan, bases.astype(np.float32).astype(np.float64), 0.5, 4, 3, 7, ctx.map_points)
    assert np.array_equal(sc2, wsc2) and np.array_equal(ix2, wix2)


def test_a_refused_pyramid_falls_back_below_2_31_poses(stand_in, monkeypatch):
    """A pyramid refusal (node or cell limits) is answered by the exhaustive call while it accepts the volume, with the
    results it always gave; beyond 2^31 poses the refusal reaches the caller."""
    from pylidar_slam_b200 import odometry
    km, ctx, calls = stand_in
    monkeypatch.setattr(odometry, "POSE_SEARCH_PYRAMID_MIN_POSES", 100)
    rng = np.random.RandomState(6)
    ctx.map_points = rng.uniform([-5, -5, -0.5], [5, 5, 0.5], (200, 3)).astype(np.float32)
    scan = rng.uniform([-2, -2, -0.3], [2, 2, 0.3], (15, 3)).astype(np.float32)
    bases = _rot_bases(3, rng)
    ctx.refuse = True
    del calls[:]
    T, sc, ix = km.search_poses(scan, bases, 0.5, (4, 3), 7)
    assert [c[0] for c in calls] == ["pls_kdmap_pose_search_pyramid", "pls_kdmap_pose_search"]
    assert calls[1][1][:8] == calls[0][1][:8] and calls[1][1][8] is None
    _, wT, wsc, wix, _ = ref.search(scan, bases, 0.5, 4, 3, 7, ctx.map_points)
    assert np.array_equal(T, wT) and np.array_equal(sc, wsc) and np.array_equal(ix, wix)
    del calls[:]
    h = 23170  # (2 h + 1)^2 >= 2^31: no exhaustive call can take this volume
    assert (2 * h + 1) ** 2 >= 1 << 31
    with pytest.raises(AssertionError):
        km.search_poses(scan, bases[:1], 0.5, (h, h), 7)
    assert [c[0] for c in calls] == ["pls_kdmap_pose_search_pyramid"]
