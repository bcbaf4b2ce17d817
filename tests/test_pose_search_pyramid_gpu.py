"""pls_kdmap_pose_search_pyramid on the GPU against pls_kdmap_pose_search on the same context, bit for bit: out_T,
out_score, out_index and out_num over the exhaustive call's matrix, windows at the level strides, plateaus, edge peaks,
map points out of reach and a km-scale window.  Beyond the exhaustive call's limits, the candidates are checked against
score_poses and against exhaustive calls over base groups stitched together.  Host and device inputs, the context left
unchanged, every refusal, and ICPFrameToModel.localize over a whole 2 km map."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import pylidar_slam_b200 as b200  # noqa: E402
from pylidar_slam_b200 import _lib as lib  # noqa: E402
from pylidar_slam_b200 import synthetic as syn  # noqa: E402

pytestmark = pytest.mark.gpu


def _map_ctx(points):
    ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    pts = np.ascontiguousarray(points, np.float32)
    ctx.call("pls_kdmap_set_points", lib.ptr(pts), 0, pts.shape[0])
    return ctx


def _exhaustive(ctx, scan, bases, cell, hx, hy, K):
    T, sc = np.zeros((K, 4, 4)), np.zeros(K, np.int32)
    ix, num = np.zeros(K, np.int64), C.c_int(-1)
    b = np.ascontiguousarray(bases, np.float64)
    st = lib.load().pls_kdmap_pose_search(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(b), b.shape[0], float(cell),
                                          hx, hy, K, None, lib.ptr(T), lib.ptr(sc), lib.ptr(ix), C.byref(num))
    assert st == lib.PLS_OK, lib.load().pls_last_error(ctx.handle)
    return T[:num.value], sc[:num.value], ix[:num.value]


def _pyramid(ctx, scan, bases, cell, hx, hy, K, expect=lib.PLS_OK):
    T, sc = np.zeros((K, 4, 4)), np.zeros(K, np.int32)
    ix, num = np.zeros(K, np.int64), C.c_int(-1)
    b = np.ascontiguousarray(bases, np.float64)
    st = lib.load().pls_kdmap_pose_search_pyramid(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(b), b.shape[0],
                                                  float(cell), hx, hy, K, lib.ptr(T), lib.ptr(sc), lib.ptr(ix),
                                                  C.byref(num))
    assert st == expect, lib.load().pls_last_error(ctx.handle)
    return T[:num.value], sc[:num.value], ix[:num.value]


def _same(ctx, scan, bases, cell, hx, hy, K):
    want = _exhaustive(ctx, scan, bases, cell, hx, hy, K)
    got = _pyramid(ctx, scan, bases, cell, hx, hy, K)
    for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(g, w)
    return len(want[1])


def _bases(A, rng, spread=2.0):
    th = rng.uniform(-np.pi, np.pi, A)
    B = np.tile(np.eye(4), (A, 1, 1))
    B[:, 0, 0], B[:, 0, 1], B[:, 1, 0], B[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    B[:, :3, 3] = rng.uniform(-spread, spread, (A, 3)) * [1, 1, 0.2]
    return B


def _scene(n, cell, rng, extent=12.0):
    """A map of ~40 % occupied cells around the origin and a scan of n rows with NaN and +-inf rows mixed in."""
    m = rng.uniform([-extent, -extent, -1.5], [extent, extent, 1.5], (int(3 * (2 * extent / cell) ** 2), 3))
    scan = rng.uniform([-extent / 2, -extent / 2, -1.2], [extent / 2, extent / 2, 1.2], (n, 3)).astype(np.float32)
    if n > 3:
        k = rng.choice(n, max(1, n // 50), replace=False)
        scan[k, rng.randint(0, 3, k.size)] = rng.choice([np.nan, np.inf, -np.inf], k.size)
    return m.astype(np.float32), scan


# (A, n, half_x, half_y, cell, K): base counts, scan sizes, cells and K of the exhaustive call's matrix
CASES = [
    (1, 1, 0, 0, 1.0, 1), (2, 255, 1, 1, 0.3, 8), (72, 256, 31, 33, 1.0, 1024), (360, 257, 1, 1, 2.5, 8),
    (2, 4096, 32, 32, 0.3, 1024), (1, 255, 65, 65, 1.0, 8), (2, 131072, 1, 1, 0.3, 1), (72, 4096, 0, 0, 0.1, 8),
    (1, 1000, 33, 31, 2.5, 1024), (360, 64, 4, 4, 1.0, 1024), (72, 4096, 40, 40, 0.5, 8), (4, 131072, 20, 20, 0.5, 8),
]


@pytest.mark.parametrize("A,n,hx,hy,cell,K", CASES)
def test_equals_the_exhaustive_call(A, n, hx, hy, cell, K):
    rng = np.random.RandomState(A * 7 + n + hx)
    m, scan = _scene(n, cell, rng, extent=max(6.0, 30 * cell))
    ctx = _map_ctx(m)
    num = _same(ctx, scan, _bases(A, rng, spread=3 * cell), cell, hx, hy, K)
    assert num > 0 or n == 1


@pytest.mark.parametrize("extent", [31, 32, 33, 63, 64, 65])
def test_box_word_edges_and_half_cells(extent):
    cell = 0.5
    rng = np.random.RandomState(extent)
    xs = -20 + np.arange(extent)
    scan = np.stack([xs * cell, rng.randint(-3, 3, extent) * cell, rng.randint(-2, 2, extent) * cell], 1)
    scan[1::3, 1] += 0.5 * cell
    scan = scan.astype(np.float32)
    m = scan[rng.rand(extent) < 0.6].copy()
    m[::2, 0] += np.float32(0.5 * cell)
    m = np.concatenate([m, rng.uniform(-15, 15, (4000, 3)).astype(np.float32) * [1, 0.2, 0.1]]).astype(np.float32)
    ctx = _map_ctx(m)
    for hx, hy, A in ((0, 0, 1), (1, 2, 2), (extent, 3, 3)):
        bases = np.tile(np.eye(4), (A, 1, 1))
        bases[A - 1, 0, 3] += 3 * cell * (A - 1)
        for K in (1, 8, 1024):
            _same(ctx, scan, bases, cell, hx, hy, K)


@pytest.mark.parametrize("W", [15, 17, 31, 33, 255, 257, 511, 513, 1023, 1025])
def test_windows_at_the_level_strides(W):
    """Window widths of 2^k - 1 and 2^k + 1 around the level strides (16 roots of 2^kmax shifts per side), where roots
    and children stick out past the window edge."""
    rng = np.random.RandomState(W)
    cell = 0.5
    m = rng.uniform([-W * cell / 2 - 5, -40, -1], [W * cell / 2 + 5, 40, 1], (60000, 3)).astype(np.float32)
    scan = rng.uniform([-4, -4, -0.8], [4, 4, 0.8], (700, 3)).astype(np.float32)
    ctx = _map_ctx(m)
    h = W // 2
    for hx, hy in ((h, 3), (3, h), (h, h)):
        for K in (1, 8, 1024):
            _same(ctx, scan, _bases(3, rng, 1.0), cell, hx, hy, K)


def _peak_scene():
    cell = 1.0
    scan = np.array([[0.0, 0.0, 0.0]], np.float32)
    occ = [(-4, -4), (-3, -4), (4, 4), (4, 3), (0, 0), (1, 0), (0, 1), (1, 1), (-4, 2), (2, -3)]
    m = np.array([[x, y, 0.0] for x, y in occ], np.float32)
    bases = np.tile(np.eye(4), (5, 1, 1))
    bases[:, 0, 3] = [0, 0.2, -0.3, 0.4, 0.1]
    return m, scan, bases, cell


def test_plateaus_edge_peaks_and_out_of_reach_points():
    m, scan, bases, cell = _peak_scene()
    ctx = _map_ctx(m)
    for K in (1, 3, 1024):
        assert _same(ctx, scan, bases, cell, 4, 4, K) > 0
    bases2 = bases.copy()
    bases2[:-1, 2, 3] = 50.0                          # only the last base scores: no wrap-around in a
    _same(ctx, scan, bases2, cell, 4, 4, 1024)
    # map points far outside the reachable box on every side: clipping drops them, the result is the same
    far = np.array([[x, y, z] for x in (-3000, 0, 3000) for y in (-3000, 0, 3000) for z in (-400, 0, 400)], np.float32)
    ctx2 = _map_ctx(np.concatenate([m, far[np.any(far != 0, axis=1)]]))
    for K in (1, 1024):
        assert np.array_equal(_pyramid(ctx2, scan, bases, cell, 4, 4, K)[2], _exhaustive(ctx, scan, bases, cell, 4, 4, K)[2])
        _same(ctx2, scan, bases, cell, 4, 4, K)
    # a window far larger than the map
    _same(ctx, scan, bases, cell, 3000, 2000, 1024)
    # a map wholly out of reach, and a scan without a valid row
    ctx3 = _map_ctx(m + np.float32(5000))
    assert len(_pyramid(ctx3, scan, bases, cell, 4, 4, 8)[2]) == 0
    assert len(_pyramid(ctx, np.full((4, 3), np.nan, np.float32), bases, cell, 4, 4, 8)[2]) == 0


def _wide_map_and_scan(offset):
    """The 2 km map of tools/prior_map_bench.py with the synthetic hall moved by `offset`, and frame 7 on it."""
    from prior_map_bench import make_maps
    maps, _ = make_maps()
    wide = maps["wide2km"].copy()
    wide[:200_000, :2] += np.float32(offset)
    gt = syn.gt_pose(7).astype(np.float64)
    gt[:2, 3] += offset
    return wide, gt


def test_km_scale_window_equals_the_exhaustive_call():
    """+-1000 m at 1 m with 72 yaws (288 M poses) on the 2 km map, hall off centre."""
    wide, gt = _wide_map_and_scan(np.array([430.0, -270.0]))
    scan = np.ascontiguousarray(b200.grid_sample(syn.scan(7, 64, 2048).astype(np.float32), 1.0)[0])
    ctx = _map_ctx(wide)
    prior = gt.copy()
    prior[:2, 3] = 0.0
    bases = b200.odometry.yaw_sweep(prior, np.pi, np.deg2rad(5))
    for K in (1, 8):
        assert _same(ctx, scan, bases, 1.0, 1000, 1000, K) == K


def _key_beats_neighbours(km, scan, bases, cell, hx, hy, T, sc, ix):
    """Each candidate's score is score_poses at its T, and its key beats each of its 26 neighbours' score_poses key."""
    A, Wx, Wy = bases.shape[0], 2 * hx + 1, 2 * hy + 1
    assert np.array_equal(km.score_poses(scan, T, cell), sc)
    for L, s in zip(ix.tolist(), sc.tolist()):
        i, t = L % Wx, L // Wx
        j, a = t % Wy, t // Wy
        nb, nL = [], []
        for da in (-1, 0, 1):
            for dj in (-1, 0, 1):
                for di in (-1, 0, 1):
                    b, jj, ii = a + da, j + dj, i + di
                    if (da, dj, di) == (0, 0, 0) or not (0 <= b < A and 0 <= jj < Wy and 0 <= ii < Wx):
                        continue
                    Tn = bases[b].copy()
                    Tn[0, 3] += np.float64(ii - hx) * np.float64(cell)
                    Tn[1, 3] += np.float64(jj - hy) * np.float64(cell)
                    nb.append(Tn)
                    nL.append((b * Wy + jj) * Wx + ii)
        for sn, Ln in zip(km.score_poses(scan, np.array(nb), cell).tolist(), nL):
            assert s > sn or (s == sn and L < Ln)


def _stitched(ctx, scan, bases, cell, hx, hy, K):
    """The volume's candidates from exhaustive calls over base groups (a - 1, a, a + 1): a group's middle base has every
    neighbour it has in the whole volume, so its candidates there are its candidates in the whole volume."""
    A, V1 = bases.shape[0], (2 * hx + 1) * (2 * hy + 1)
    found = []
    for a in range(A):
        lo = max(a - 1, 0)
        _, sc, ix = _exhaustive(ctx, scan, bases[lo:a + 2], cell, hx, hy, K)
        assert len(ix) < K  # the group's list is complete
        found += [(-int(s), int(L) + lo * V1) for s, L in zip(sc, ix) if int(L) // V1 + lo == a]
    return sorted(found)


def test_beyond_the_volume_limit():
    """A (2 hx + 1)(2 hy + 1) >= 2^31 with a small scan on a sparse map: no candidate missed."""
    rng = np.random.RandomState(21)
    cell, h = 1.0, 11586
    m = rng.uniform([-300, -300, -1], [300, 300, 1], (40, 3)).astype(np.float32)
    scan = rng.uniform([-3, -3, -0.5], [3, 3, 0.5], (4, 3)).astype(np.float32)
    bases = _bases(4, rng, 2.0)
    assert bases.shape[0] * (2 * h + 1) ** 2 >= 2 ** 31
    ctx = _map_ctx(m)
    T, sc, ix = _pyramid(ctx, scan, bases, cell, h, h, 1024)
    assert 0 < len(ix) < 1024
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    _key_beats_neighbours(km, scan, bases, cell, h, h, T, sc, ix)
    assert [(-int(s), int(L)) for s, L in zip(sc, ix)] == _stitched(ctx, scan, bases, cell, h, h, 1024)


def test_beyond_the_bit_limit():
    """Two bases 200 km apart: the exhaustive call's box exceeds 2^31 bits on a small map, the clipped grid does not."""
    rng = np.random.RandomState(22)
    cell, hx, hy = 0.5, 600, 1000
    m = rng.uniform([-40, -40, -1], [40, 40, 1], (3000, 3)).astype(np.float32)
    scan = rng.uniform([-4, -4, -0.8], [4, 4, 0.8], (300, 3)).astype(np.float32)
    bases = _bases(2, rng, 1.0)
    bases[1, 0, 3] += 200_000.0
    ctx = _map_ctx(m)
    st = lib.load().pls_kdmap_pose_search(ctx.handle, lib.ptr(scan), 300, lib.ptr(bases), 2, cell, hx, hy, 8, None,
                                          lib.ptr(np.zeros(128)), lib.ptr(np.zeros(8, np.int32)),
                                          lib.ptr(np.zeros(8, np.int64)), C.byref(C.c_int()))
    assert st == lib.PLS_E_INVALID and "PLS_POSE_SEARCH_MAX_BITS" in lib.load().pls_last_error(ctx.handle).decode()
    T, sc, ix = _pyramid(ctx, scan, bases, cell, hx, hy, 64)
    assert len(ix) == 64
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    _key_beats_neighbours(km, scan, bases, cell, hx, hy, T, sc, ix)
    # base 1 sees no map cell, so base 0 alone has every candidate
    assert len(_exhaustive(ctx, scan, bases[1:], cell, hx, hy, 8)[2]) == 0
    _, wsc, wix = _exhaustive(ctx, scan, bases[:1], cell, hx, hy, 64)
    assert np.array_equal(sc, wsc) and np.array_equal(ix, wix)


def test_host_and_device_inputs_give_the_same_bits():
    rng = np.random.RandomState(11)
    m, scan = _scene(3000, 0.5, rng, extent=8.0)
    bases = _bases(6, rng, 1.0)
    ctx = _map_ctx(m)
    T, sc, ix = _pyramid(ctx, scan, bases, 0.5, 40, 40, 32)
    d = [torch.from_numpy(scan).cuda(), torch.from_numpy(bases).cuda()]
    dT, dsc = torch.zeros((32, 4, 4), dtype=torch.float64, device="cuda"), torch.zeros(32, dtype=torch.int32, device="cuda")
    dix, num = torch.zeros(32, dtype=torch.int64, device="cuda"), C.c_int(-1)
    torch.cuda.synchronize()
    assert lib.load().pls_kdmap_pose_search_pyramid(ctx.handle, lib.ptr(d[0]), 3000, lib.ptr(d[1]), 6, 0.5, 40, 40, 32,
                                                    lib.ptr(dT), lib.ptr(dsc), lib.ptr(dix), C.byref(num)) == lib.PLS_OK
    assert num.value == len(ix) == 32
    assert np.array_equal(dT.cpu().numpy(), T) and np.array_equal(dsc.cpu().numpy(), sc)
    assert np.array_equal(dix.cpu().numpy(), ix)


def _odometry(max_align=8):
    proj = b200.SphericalProjector(height=32, width=512, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=4),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                              max_iters=1)),
        max_num_alignments=max_align, data_key="numpy_pc")
    o = b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0")
    o.init()
    return o


def _state(o):
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=4), ctx=o.ctx)
    nq = int(o.last_info[2])
    out = dict(points=km.points(), frames=np.array(km.frame_counts()), idx=np.empty(nq, np.int64),
               nb=np.empty((nq, 3), np.float32), state=np.empty((nq, 4), np.float32), sums=np.empty(30))
    assert lib.load().pls_kdmap_last_correspondences(o.ctx.handle, nq, lib.ptr(out["idx"]), lib.ptr(out["nb"]), None,
                                                     lib.ptr(out["state"]), lib.ptr(out["sums"])) == lib.PLS_OK
    icp, it = np.empty(30), C.c_int(0)
    assert lib.load().pls_last_icp_sums(o.ctx.handle, lib.ptr(icp), C.byref(it)) == lib.PLS_OK
    out["icp"], out["iters"] = icp, np.array([it.value])
    return out


def _equal(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_context_is_unchanged_and_refusals_change_nothing():
    a, b = _odometry(), _odometry()
    for k in range(4):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
    before = _state(a)
    scan = syn.scan(4, 32, 512).astype(np.float32)
    rng = np.random.RandomState(0)
    B = _bases(8, rng, 1.0)
    assert len(_pyramid(a.ctx, scan, B, 0.5, 30, 30, 8)[2]) > 0
    L = lib.load()
    out = [np.zeros(64 * 16), np.zeros(64, np.int32), np.zeros(64, np.int64)]

    def call(s=scan, ns=None, bb=B, A=None, cell=0.5, hx=1, hy=1, K=4, outs=None):
        num = C.c_int(-5)
        o = out if outs is None else outs
        return L.pls_kdmap_pose_search_pyramid(a.ctx.handle, lib.ptr(s), s.shape[0] if ns is None else ns,
                                               lib.ptr(bb), (bb.shape[0] if A is None else A) if bb is not None else 1,
                                               cell, hx, hy, K, lib.ptr(o[0]), lib.ptr(o[1]), lib.ptr(o[2]),
                                               C.byref(num))

    bad_base, inf_base = B.copy(), B.copy()
    bad_base[1, 2, 1], inf_base[0, 0, 3] = np.nan, np.inf
    far = B.copy()
    far[0, 0, 3] = 1e12
    refusals = [dict(s=None), dict(bb=None), dict(ns=0), dict(ns=-3), dict(A=0), dict(A=-1), dict(hx=-1), dict(hy=-1),
                dict(K=0), dict(K=-1), dict(K=1025), dict(cell=0.0), dict(cell=-0.5), dict(cell=float("nan")),
                dict(cell=float("inf")), dict(bb=bad_base), dict(bb=inf_base), dict(hx=1 << 30), dict(hy=1 << 30),
                dict(A=1 << 30, hx=(1 << 30) - 1, hy=(1 << 30) - 1),
                dict(outs=[None, out[1], out[2]]), dict(outs=[out[0], None, out[2]]), dict(outs=[out[0], out[1], None]),
                dict(bb=far), dict(s=np.zeros((131072, 3), np.float32), bb=np.tile(B, (342, 1, 1))),
                dict(cell=1e-4, hx=0, hy=0)]
    for kw in refusals:
        if kw.get("s", 0) is None:
            st = L.pls_kdmap_pose_search_pyramid(a.ctx.handle, None, 10, lib.ptr(B), 8, 0.5, 1, 1, 4, lib.ptr(out[0]),
                                                 lib.ptr(out[1]), lib.ptr(out[2]), C.byref(C.c_int()))
        else:
            st = call(**kw)
        assert st == lib.PLS_E_INVALID, kw
    assert "PLS_POSE_SEARCH_PYRAMID_MAX_BITS" in L.pls_last_error(a.ctx.handle).decode()
    assert call(s=np.zeros((131072, 3), np.float32), bb=np.tile(B, (342, 1, 1))) == lib.PLS_E_INVALID  # 2 736 bases
    assert "PLS_POSE_SEARCH_PYRAMID_MAX_CELL_BYTES" in L.pls_last_error(a.ctx.handle).decode()
    # more roots than the work lists hold: refused after work was enqueued, the context still unchanged
    many = np.tile(np.eye(4), ((1 << 26) // 225 + 1, 1, 1))
    one = np.ascontiguousarray(scan[np.isfinite(scan).all(axis=1)][:1])  # a row inside the map's box
    assert call(s=one, bb=many, hx=7, hy=7, K=8) == lib.PLS_E_INVALID
    msg = L.pls_last_error(a.ctx.handle).decode()
    assert "PLS_POSE_SEARCH_PYRAMID_MAX_NODES" in msg and "level 0" in msg and str(many.shape[0] * 225) in msg, msg
    fresh = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    assert L.pls_kdmap_pose_search_pyramid(fresh.handle, lib.ptr(scan), scan.shape[0], lib.ptr(B), 8, 0.5, 1, 1, 4,
                                           lib.ptr(out[0]), lib.ptr(out[1]), lib.ptr(out[2]),
                                           C.byref(C.c_int())) == lib.PLS_E_INVALID
    proj = lib.Context(local_map_type=lib.MAP_PROJECTIVE, height=16, width=64)
    assert L.pls_kdmap_pose_search_pyramid(proj.handle, lib.ptr(scan), scan.shape[0], lib.ptr(B), 8, 0.5, 1, 1, 4,
                                           lib.ptr(out[0]), lib.ptr(out[1]), lib.ptr(out[2]),
                                           C.byref(C.c_int())) == lib.PLS_E_INVALID
    _equal(before, _state(a))
    _equal(before, _state(b))
    for k in range(4, 7):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
        assert np.array_equal(a._pose_out, b._pose_out)
        _equal(_state(a), _state(b))


def test_localize_over_the_whole_2km_map():
    """The prior has the true z, roll and pitch, lies >= 500 m from the truth and has no yaw information."""
    wide, gt = _wide_map_and_scan(np.array([430.0, -270.0]))
    o = _odometry(max_align=30)
    b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=o.ctx).set_map_pointcloud(wide)
    scan = syn.scan(7, 64, 2048).astype(np.float32)
    prior = gt.copy()
    th = np.deg2rad(137.0)
    prior[:3, :3] = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]) @ gt[:3, :3]
    prior[:2, 3] = [-40.0, 60.0]
    assert np.linalg.norm(prior[:2, 3] - gt[:2, 3]) >= 500
    res = o.localize(scan, prior, radius=1000.0, cell_size=1.0, yaw_step=np.deg2rad(5), num_candidates=8)
    assert len(res) == 8
    d = np.linalg.inv(gt) @ res[0].T
    e_t, e_r = np.linalg.norm(d[:3, 3]), np.rad2deg(abs(np.arctan2(d[1, 0], d[0, 0])))
    assert e_t <= 0.1 and e_r <= 0.5, (e_t, e_r)


def test_search_poses_answers_a_refused_pyramid_volume(monkeypatch):
    """search_poses over a volume below 2^31 poses whose roots outnumber the pyramid's work lists: the exhaustive call
    answers it, bit for bit what it answers directly.  Beyond 2^31 poses the refusal reaches the caller."""
    rng = np.random.RandomState(31)
    m = rng.uniform([-20, -20, -1], [20, 20, 1], (3000, 3)).astype(np.float32)
    scan = rng.uniform([-3, -3, -0.5], [3, 3, 0.5], (2, 3)).astype(np.float32)
    ctx = _map_ctx(m)
    bases = np.tile(np.eye(4), ((1 << 26) // 225 + 1, 1, 1))
    bases[:, 0, 3] = rng.uniform(-5, 5, bases.shape[0])
    _pyramid(ctx, scan, bases, 0.5, 7, 7, 8, expect=lib.PLS_E_INVALID)
    assert "PLS_POSE_SEARCH_PYRAMID_MAX_NODES" in lib.load().pls_last_error(ctx.handle).decode()
    monkeypatch.setattr(b200.odometry, "POSE_SEARCH_PYRAMID_MIN_POSES", 1)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    T, sc, ix = km.search_poses(scan, bases, 0.5, (7, 7), 8)
    wT, wsc, wix = _exhaustive(ctx, scan, bases, 0.5, 7, 7, 8)
    assert len(ix) == 8 and np.array_equal(T, wT) and np.array_equal(sc, wsc) and np.array_equal(ix, wix)
    wide = np.tile(np.eye(4), ((1 << 18) + 1, 1, 1))  # 256 roots per base at +-120 cells: over 2^26 roots, 1.5e10 poses
    with pytest.raises(AssertionError, match="PLS_POSE_SEARCH_PYRAMID_MAX_NODES"):
        km.search_poses(scan, wide, 0.5, (120, 120), 8)
