"""pls_kdmap_pose_search_scans without a GPU: a numpy restatement of the batched search (one shared grid, concatenated
volumes, a peak test that stops at scan boundaries, a key sort then a stable sort by scan) against the float64
reference run per scan, and the Python layer over a host stand-in -- routing to the pyramid, chunks of fewer than 2^31
poses, halving after a shared-grid refusal, one-scan chunks, input conversion, and localize_scans' assembly against
localize's."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pose_search_reference as ref  # noqa: E402

GRID_REFUSAL = "pls_kdmap_pose_search_scans: the shared occupancy box of {} cells exceeds PLS_POSE_SEARCH_MAX_BITS"


def _rot_bases(A, rng, spread=1.0, at=(0.0, 0.0)):
    th = rng.uniform(-np.pi, np.pi, A)
    B = np.tile(np.eye(4), (A, 1, 1))
    B[:, 0, 0], B[:, 0, 1], B[:, 1, 0], B[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    B[:, :2, 3] = rng.uniform(-spread, spread, (A, 2)) + np.asarray(at)
    return B


def shared_grid(scans, bases_list, cell, halves):
    """(origin, extent) of the union of every scan's reachable box, or None when no scan has a valid row."""
    lo, hi = [], []
    for scan, bases, (hx, hy) in zip(scans, bases_list, halves):
        P = ref.valid_rows(scan)
        if P.shape[0] == 0:
            continue
        cells = np.concatenate([ref.base_cells(P, b, cell) for b in np.asarray(bases).reshape(-1, 4, 4)])
        lo.append(cells.min(0) - [hx, hy, 0])
        hi.append(cells.max(0) + [hx, hy, 0])
    if not lo:
        return None
    o = np.min(lo, 0)
    return o, np.max(hi, 0) - o + 1


def batched_search(scans, bases_list, cell, halves, K, map_points):
    """The batched call restated: (volumes concatenated, [(T, score, index)] per scan)."""
    S = len(scans)
    grid = shared_grid(scans, bases_list, cell, halves)
    shapes = [(np.asarray(b).reshape(-1, 4, 4).shape[0], 2 * hy + 1, 2 * hx + 1) for b, (hx, hy) in zip(bases_list, halves)]
    first = np.concatenate([[0], np.cumsum([a * wy * wx for a, wy, wx in shapes])])
    vol = np.zeros(first[-1], np.int32)
    if grid is not None:
        o, e = grid
        m = ref.map_cells(map_points, cell) if len(map_points) else np.zeros((0, 3), np.int64)
        inside = np.all((m >= o) & (m < o + e), axis=1)
        occupied = {tuple(c) for c in (m[inside] - o)}
        for s in range(S):
            P = ref.valid_rows(scans[s])
            A, Wy, Wx = shapes[s]
            hx, hy = halves[s]
            v = vol[first[s]:first[s + 1]].reshape(A, Wy, Wx)
            for a, b in enumerate(np.asarray(bases_list[s]).reshape(-1, 4, 4)):
                rel = ref.base_cells(P, b, cell) - o - [hx, hy, 0]   # relative to the grid at shift (-hx, -hy)
                for jj in range(Wy):
                    for ii in range(Wx):
                        c = rel + [ii, jj, 0]
                        assert np.all((c >= 0) & (c < e)), "every lookup lies inside the shared grid"
                        v[a, jj, ii] = sum(tuple(x) in occupied for x in c)
    # peaks within each scan's volume, keys (~score << 32) | L_local, a key sort, then a stable sort by scan
    keys, scan_of = [], []
    for s in range(S):
        A, Wy, Wx = shapes[s]
        for L in ref.candidates(vol[first[s]:first[s + 1]].reshape(A, Wy, Wx)):
            keys.append(((~int(vol[first[s] + L]) & 0xffffffff) << 32) | L)
            scan_of.append(s)
    keys, scan_of = np.array(keys, np.uint64), np.array(scan_of, np.int64)
    by_key = np.argsort(keys, kind="stable")
    order = by_key[np.argsort(scan_of[by_key], kind="stable")]
    out = []
    for s in range(S):
        A, Wy, Wx = shapes[s]
        hx, hy = halves[s]
        mine = [int(keys[e]) for e in order if scan_of[e] == s][:K]
        B = np.asarray(bases_list[s], np.float64).reshape(-1, 4, 4)
        T = np.zeros((len(mine), 4, 4))
        for c, k in enumerate(mine):
            a, rem = divmod(k & 0xffffffff, Wy * Wx)
            jj, ii = divmod(rem, Wx)
            T[c] = B[a]
            T[c, 0, 3] = B[a, 0, 3] + np.float64(ii - hx) * np.float64(cell)
            T[c, 1, 3] = B[a, 1, 3] + np.float64(jj - hy) * np.float64(cell)
        out.append((T, np.array([~(k >> 32) & 0xffffffff for k in mine], np.uint32).astype(np.int32),
                    np.array([k & 0xffffffff for k in mine], np.int64)))
    return vol, out


def test_batched_restatement_equals_the_reference_per_scan():
    rng = np.random.RandomState(11)
    m = rng.uniform([-8, -8, -1], [8, 8, 1], (500, 3)).astype(np.float32)
    for trial in range(4):
        S = rng.randint(1, 5)
        scans, bases, halves = [], [], []
        for s in range(S):
            n = rng.randint(1, 25)
            scan = rng.uniform([-2, -2, -0.8], [2, 2, 0.8], (n, 3)).astype(np.float32)
            if n > 2:
                scan[rng.randint(n), rng.randint(3)] = rng.choice([np.nan, np.inf])
            if trial == 3 and s == 0:
                scan[:] = np.nan                                   # a scan with no valid row
            scans.append(scan)
            bases.append(_rot_bases(rng.randint(1, 4), rng, at=rng.uniform(-3, 3, 2)))
            halves.append((int(rng.randint(0, 4)), int(rng.randint(0, 4))))
        for K in (0, 1, 5, 1024):
            vol, got = batched_search(scans, bases, 0.5, halves, K, m)
            at = 0
            for s in range(S):
                wv, wT, wsc, wix, wnum = ref.search(scans[s], bases[s], 0.5, *halves[s], K, m)
                assert np.array_equal(vol[at:at + wv.size], wv.reshape(-1))
                at += wv.size
                T, sc, ix = got[s]
                assert len(ix) == wnum and np.array_equal(T, wT) and np.array_equal(sc, wsc)
                assert np.array_equal(ix, wix)


def test_peaks_never_cross_a_scan_boundary():
    """Two scans whose volumes meet: the last pose of scan 0 and the first of scan 1 are both candidates, although a
    single volume over both would let the better one suppress the other."""
    cell = 1.0
    m = np.array([[0, 0, 0], [1, 0, 0]], np.float32)
    scan = np.array([[0, 0, 0]], np.float32)
    b0 = np.tile(np.eye(4), (2, 1, 1))
    b0[1, 0, 3] = 1.0
    b1 = np.eye(4)[None].copy()
    vol, got = batched_search([scan, scan], [b0, b1], cell, [(0, 0), (0, 0)], 4, m)
    assert vol.tolist() == [1, 1, 1]
    assert got[0][2].tolist() == [0] and got[1][2].tolist() == [0]


@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext answering the three search calls by the reference and the restatement above, and both
    registration calls by one deterministic rule, so that localize and localize_scans can be compared."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    def refine(scan, T0):
        """A stand-in refinement of T0 [4,4] float32: moves it by a scan-dependent step; singular when the scan's
        first row is negative in x."""
        step = np.float32(np.nansum(scan[:, :2]) % 1.0 * 0.1)
        T = T0.copy()
        T[0, 3] += step
        T[1, 3] -= step
        return T, 1 + int(step * 30) % 3, _lib.PLS_E_SINGULAR if scan[0, 0] < -1.5 else _lib.PLS_OK

    class SearchFakeContext(dry.FakeContext):
        map_points = np.zeros((0, 3), np.float32)
        max_grid_cells = None  # refuse a batch whose shared grid holds more cells than this

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
            return self.pls_kdmap_pose_search(scan, n, bases, A, cell, hx, hy, K, None, out_T, out_score, out_index,
                                              out_num)

        def pls_kdmap_pose_search_scans(self, scans, n, S, bases, num_bases, cell, hx, hy, K, out_scores, out_T,
                                        out_score, out_index, out_num):
            rows = dry.arr(n, (S,), np.int64)
            A = dry.arr(num_bases, (S,), np.int32)
            addr = dry.arr(scans, (S,), np.uint64)
            B = dry.arr(bases, (int(A.sum()), 4, 4), np.float64)
            first = np.concatenate([[0], np.cumsum(A)])
            sc_list = [dry.arr(int(addr[s]), (int(rows[s]), 3), np.float32) for s in range(S)]
            b_list = [B[first[s]:first[s + 1]] for s in range(S)]
            halves = list(zip(dry.arr(hx, (S,), np.int32).tolist(), dry.arr(hy, (S,), np.int32).tolist()))
            grid = shared_grid(sc_list, b_list, cell, halves)
            if grid is not None and self.max_grid_cells is not None and np.prod(grid[1]) > self.max_grid_cells:
                raise AssertionError(GRID_REFUSAL.format(" x ".join(str(int(x)) for x in grid[1])))
            vol, got = batched_search(sc_list, b_list, cell, halves, K, self.map_points)
            if out_scores:
                dry.arr(out_scores, vol.shape, np.int32)[:] = vol
            Kc = max(K, 1)
            for s, (T, sc, ix) in enumerate(got):
                k = len(ix)
                if k:
                    dry.arr(out_T, (S, Kc, 4, 4), np.float64)[s, :k] = T
                    dry.arr(out_score, (S, Kc), np.int32)[s, :k] = sc
                    dry.arr(out_index, (S, Kc), np.int64)[s, :k] = ix
            dry.arr(out_num, (S,), np.int32)[:] = [len(g[2]) for g in got]

        def pls_register_hypotheses(self, pts, n, T0s, B, out_T, out_params, out_losses, out_iters, out_status):
            scan = dry.arr(pts, (n, 3), np.float32)
            for b, T0 in enumerate(dry.arr(T0s, (B, 4, 4), np.float32)):
                T, it, st = refine(scan, T0)
                dry.arr(out_T, (B, 4, 4), np.float32)[b] = T
                dry.arr(out_iters, (B,), np.int32)[b] = it
                dry.arr(out_status, (B,), np.int32)[b] = st

        def pls_register_scans(self, scans, n, S, scan_of, T0s, B, out_T, out_params, out_losses, out_iters,
                               out_status):
            rows, addr = dry.arr(n, (S,), np.int64), dry.arr(scans, (S,), np.uint64)
            idx = dry.arr(scan_of, (B,), np.int32)
            for b, T0 in enumerate(dry.arr(T0s, (B, 4, 4), np.float32)):
                s = int(idx[b])
                T, it, st = refine(dry.arr(int(addr[s]), (int(rows[s]), 3), np.float32), T0)
                dry.arr(out_T, (B, 4, 4), np.float32)[b] = T
                dry.arr(out_iters, (B,), np.int32)[b] = it
                dry.arr(out_status, (B,), np.int32)[b] = st

    monkeypatch.setattr(_lib, "Context", SearchFakeContext)
    monkeypatch.setattr(common, "_default_ctx", SearchFakeContext())
    from pylidar_slam_b200.odometry import KdTreeLocalMap, KdTreeLocalMapConfig
    ctx = SearchFakeContext()
    return KdTreeLocalMap(KdTreeLocalMapConfig(), ctx=ctx), ctx, calls


def _batch(rng, S, spread=3.0, n=(5, 20)):
    scans = [rng.uniform([-2, -2, -0.3], [2, 2, 0.3], (rng.randint(*n), 3)).astype(np.float32) for _ in range(S)]
    bases = [_rot_bases(rng.randint(1, 3), rng, at=rng.uniform(-spread, spread, 2)) for _ in range(S)]
    return scans, bases


def _assert_same(got, want):
    assert len(got) == len(want)
    for (T, sc, ix), (wT, wsc, wix) in zip(got, want):
        assert T.dtype == np.float64 and sc.dtype == np.int32 and ix.dtype == np.int64
        assert np.array_equal(T, wT) and np.array_equal(sc, wsc) and np.array_equal(ix, wix)


def test_routing_pyramid_sized_scans_go_single(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry
    km, ctx, calls = stand_in
    monkeypatch.setattr(odometry, "POSE_SEARCH_PYRAMID_MIN_POSES", 100)
    rng = np.random.RandomState(1)
    ctx.map_points = rng.uniform([-6, -6, -0.5], [6, 6, 0.5], (300, 3)).astype(np.float32)
    scans, bases = _batch(rng, 4)
    bases[2] = _rot_bases(2, rng)                                 # 2 x 9 x 9 = 162 poses: the pyramid
    halves = [(1, 1), (2, 1), (4, 4), (0, 3)]
    got = km.search_poses_scans(scans, bases, 0.5, halves, 3)
    names = [c[0] for c in calls]
    assert names == ["pls_kdmap_pose_search_pyramid", "pls_kdmap_pose_search_scans"]
    assert calls[1][1][2] == 3                                    # the three other scans in one call
    _assert_same(got, [km.search_poses(scans[s], bases[s], 0.5, halves[s], 3) for s in range(4)])
    # K = 0 never routes to the pyramid: every scan is batched
    del calls[:]
    km.search_poses_scans(scans, bases, 0.5, halves, 0)
    assert [c[0] for c in calls] == ["pls_kdmap_pose_search_scans"] and calls[0][1][2] == 4


def test_chunks_hold_fewer_than_the_pose_limit(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry
    km, ctx, calls = stand_in
    monkeypatch.setattr(odometry, "_POSE_SEARCH_SCANS_MAX_POSES", 40)
    rng = np.random.RandomState(2)
    ctx.map_points = rng.uniform([-6, -6, -0.5], [6, 6, 0.5], (300, 3)).astype(np.float32)
    scans, bases = _batch(rng, 6)
    bases = [b[:1] for b in bases]
    halves = [(1, 1), (1, 1), (1, 1), (1, 1), (3, 3), (1, 0)]    # 9, 9, 9, 9, 49, 3 poses
    got = km.search_poses_scans(scans, bases, 0.5, halves, 2)
    # 9+9+9+9 = 36 < 40; the 49-pose scan alone (a one-scan chunk: the single call); then the last one alone
    assert [(c[0], c[1][2] if c[0].endswith("scans") else None) for c in calls] == [
        ("pls_kdmap_pose_search_scans", 4), ("pls_kdmap_pose_search", None), ("pls_kdmap_pose_search", None)]
    _assert_same(got, [km.search_poses(scans[s], bases[s], 0.5, halves[s], 2) for s in range(6)])


def test_a_refused_shared_grid_is_halved_by_x(stand_in):
    km, ctx, calls = stand_in
    rng = np.random.RandomState(3)
    ctx.map_points = rng.uniform([-40, -6, -0.5], [40, 6, 0.5], (600, 3)).astype(np.float32)
    scans, bases = _batch(rng, 5, spread=0.5)
    xs = [30.0, -30.0, 0.0, 29.0, -29.0]
    for b, x in zip(bases, xs):
        b[:, 0, 3] += x
    ctx.max_grid_cells = 2000                                     # one cluster fits; two clusters 60 m apart do not
    got = km.search_poses_scans(scans, bases, 0.5, (1, 1), 2)
    sizes = [c[1][2] if c[0].endswith("scans") else 1 for c in calls]
    names = [c[0] for c in calls]
    # 5 refused -> sorted by x: [-30, -29, 0, 29, 30] -> [-30, -29] accepted, [0, 29, 30] refused -> [0] single,
    # [29, 30] accepted
    assert sizes == [5, 2, 3, 1, 2]
    assert names == ["pls_kdmap_pose_search_scans"] * 3 + ["pls_kdmap_pose_search", "pls_kdmap_pose_search_scans"]
    ctx.max_grid_cells = None
    _assert_same(got, [km.search_poses(scans[s], bases[s], 0.5, (1, 1), 2) for s in range(5)])


def test_other_refusals_reach_the_caller(stand_in):
    km, ctx, calls = stand_in

    def refuse(*a):
        raise AssertionError("pls_kdmap_pose_search_scans: scan 1: every base must be finite")

    ctx.pls_kdmap_pose_search_scans = refuse
    rng = np.random.RandomState(4)
    scans, bases = _batch(rng, 3)
    with pytest.raises(AssertionError, match="scan 1"):
        km.search_poses_scans(scans, bases, 0.5, (1, 1), 2)
    assert len(calls) == 1


def test_inputs_numpy_torch_and_shared_or_per_scan_windows(stand_in):
    km, ctx, calls = stand_in
    rng = np.random.RandomState(5)
    ctx.map_points = rng.uniform([-6, -6, -0.5], [6, 6, 0.5], (300, 3)).astype(np.float32)
    scans, bases = _batch(rng, 3)
    want = [km.search_poses(scans[s], bases[s], 0.5, (2, 1), 4) for s in range(3)]
    _assert_same(km.search_poses_scans(scans, bases, 0.5, (2, 1), 4), want)
    _assert_same(km.search_poses_scans(scans, bases, 0.5, [(2, 1)] * 3, 4), want)
    _assert_same(km.search_poses_scans(scans, bases, 0.5, np.array([[2, 1]] * 3), 4), want)
    t_scans = [torch.from_numpy(s) for s in scans]
    t_bases = [torch.from_numpy(b) for b in bases]
    _assert_same(km.search_poses_scans(t_scans, t_bases, 0.5, (2, 1), 4), want)
    f64 = [s.astype(np.float64) for s in scans]                   # rounded to float32 as search_poses rounds them
    _assert_same(km.search_poses_scans(f64, bases, 0.5, (2, 1), 4), want)
    # per-scan windows, a scan of two scans with a shape (2, 2) pair list
    per = [(1, 0), (0, 2)]
    _assert_same(km.search_poses_scans(scans[:2], bases[:2], 0.5, per, 4),
                 [km.search_poses(scans[s], bases[s], 0.5, per[s], 4) for s in range(2)])
    with pytest.raises(AssertionError):
        km.search_poses_scans(scans, bases, 0.5, [(1, 1)] * 2, 4)
    with pytest.raises(AssertionError):
        km.search_poses_scans(scans, bases[:2], 0.5, (1, 1), 4)


def _odometry(ctx):
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200.odometry import ICPFrameToModel
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=4),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(max_iters=1)), max_num_alignments=4)
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx, odo.config = ctx, cfg
    return odo


def _same_candidates(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.score == w.score and g.coarse_score == w.coarse_score and g.coarse_rank == w.coarse_rank
        assert g.iterations == w.iterations and g.status == w.status
        assert np.array_equal(g.T, w.T) and g.T.dtype == w.T.dtype and np.array_equal(g.T0, w.T0)


@pytest.mark.parametrize("per_scan_radius", [False, True])
def test_localize_scans_assembles_as_localize(stand_in, per_scan_radius):
    from pylidar_slam_b200 import _lib
    km, ctx, calls = stand_in
    rng = np.random.RandomState(6)
    ctx.map_points = rng.uniform([-6, -6, -0.5], [6, 6, 0.5], (400, 3)).astype(np.float32)
    S = 4
    scans = [rng.uniform([-2, -2, -0.3], [2, 2, 0.3], (rng.randint(8, 20), 3)).astype(np.float32) for _ in range(S)]
    scans[1][0, 0] = -1.9                                         # singular refinements for scan 1
    scans[3][:] = np.nan                                          # no valid row: no candidate
    priors = np.tile(np.eye(4), (S, 1, 1))
    priors[:, :2, 3] = rng.uniform(-1, 1, (S, 2))
    radius = np.array([0.5, 1.0, 0.0, 0.5]) if per_scan_radius else 0.5
    odo = _odometry(ctx)
    kw = dict(cell_size=0.5, yaw_range=0.3, yaw_step=0.1, num_candidates=3)
    del calls[:]
    got = odo.localize_scans(scans, torch.from_numpy(priors) if per_scan_radius else priors, radius, **kw)
    assert [c[0] for c in calls] == ["pls_kdmap_pose_search_scans", "pls_register_scans",
                                     "pls_kdmap_pose_search_scans"]
    r = np.broadcast_to(radius, (S,))
    want = [odo.localize(scans[s], priors[s], float(r[s]), **kw) for s in range(S)]
    assert want[3] == [] and any(c.status == _lib.PLS_E_SINGULAR for c in want[1]) and sum(len(w) for w in want) >= 6
    for g, w in zip(got, want):
        _same_candidates(g, w)
