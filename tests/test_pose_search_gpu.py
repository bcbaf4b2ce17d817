"""pls_kdmap_pose_search on the GPU against the float64 reference (oracle/pose_search_reference.py), bit for bit: every
score of the volume, the candidates and their order, the map occupancy, host and device inputs, the context left
unchanged, every refusal, and localisation on the synthetic hall through ICPFrameToModel.localize."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pylidar_slam_b200 as b200  # noqa: E402
from pylidar_slam_b200 import _lib as lib  # noqa: E402
from pylidar_slam_b200 import synthetic as syn  # noqa: E402
from oracle import pose_search_reference as ref  # noqa: E402

pytestmark = pytest.mark.gpu


def _map_ctx(points):
    ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    pts = np.ascontiguousarray(points, np.float32)
    ctx.call("pls_kdmap_set_points", lib.ptr(pts), 0, pts.shape[0])
    return ctx


def _search(ctx, scan, bases, cell, hx, hy, K, scores=True):
    """The raw call: (status, volume or None, T, score, index, num)."""
    A = bases.shape[0]
    vol = np.full((A, 2 * hy + 1, 2 * hx + 1), -7, np.int32) if scores else None
    T, sc = np.zeros((max(K, 1), 4, 4)), np.zeros(max(K, 1), np.int32)
    ix, num = np.zeros(max(K, 1), np.int64), C.c_int(-1)
    b = np.ascontiguousarray(bases, np.float64)
    st = lib.load().pls_kdmap_pose_search(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(b), A, float(cell), hx, hy,
                                          K, lib.ptr(vol), lib.ptr(T), lib.ptr(sc), lib.ptr(ix), C.byref(num))
    return st, vol, T[:num.value], sc[:num.value], ix[:num.value], num.value


def _bases(A, rng, spread=2.0):
    th = rng.uniform(-np.pi, np.pi, A)
    B = np.tile(np.eye(4), (A, 1, 1))
    B[:, 0, 0], B[:, 0, 1], B[:, 1, 0], B[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    B[:, :3, 3] = rng.uniform(-spread, spread, (A, 3)) * [1, 1, 0.2]
    return B


def _scene(n, cell, rng, extent=12.0, bad=True):
    """A map of ~40 % occupied cells around the origin (negative coordinates included) and a scan of n rows, with NaN
    and +-inf rows mixed in."""
    m = rng.uniform([-extent, -extent, -1.5], [extent, extent, 1.5], (int(3 * (2 * extent / cell) ** 2), 3))
    scan = rng.uniform([-extent / 2, -extent / 2, -1.2], [extent / 2, extent / 2, 1.2], (n, 3)).astype(np.float32)
    if bad and n > 3:
        k = rng.choice(n, max(1, n // 50), replace=False)
        scan[k, rng.randint(0, 3, k.size)] = rng.choice([np.nan, np.inf, -np.inf], k.size)
    return m.astype(np.float32), scan


# (A, n, half_x, half_y, cell): windows, base counts, scan sizes and cell sizes of the issue's matrix, each at least once
SCORE_CASES = [
    (1, 1, 0, 0, 1.0), (2, 255, 1, 1, 0.3), (72, 256, 31, 33, 1.0), (360, 257, 1, 1, 2.5), (2, 4096, 32, 32, 0.3),
    (1, 255, 65, 65, 1.0), (2, 131072, 1, 1, 0.3), (72, 4096, 0, 0, 0.1), (1, 1000, 33, 31, 2.5), (360, 64, 0, 0, 1.0),
]


@pytest.mark.parametrize("A,n,hx,hy,cell", SCORE_CASES)
def test_every_score_equals_the_reference(A, n, hx, hy, cell):
    rng = np.random.RandomState(A * 7 + n + hx)
    m, scan = _scene(n, cell, rng, extent=max(6.0, 30 * cell))
    bases = _bases(A, rng, spread=3 * cell)
    ctx = _map_ctx(m)
    st, vol, *_ = _search(ctx, scan, bases, cell, hx, hy, 0)
    assert st == lib.PLS_OK, lib.load().pls_last_error(ctx.handle)
    want = ref.score_volume(scan, bases, cell, hx, hy, m)
    assert np.array_equal(vol, want)
    assert want.max() > 0 or n == 1


@pytest.mark.parametrize("extent", [31, 32, 33, 63, 64, 65])
def test_box_word_edges(extent):
    """Box x extents of 31..65 bits around the 32-bit word edges, half cells rounding both ways, negative cells."""
    cell = 0.5
    rng = np.random.RandomState(extent)
    xs = -20 + np.arange(extent)                      # x cells -20 .. -20 + extent - 1
    scan = np.stack([xs * cell, rng.randint(-3, 3, extent) * cell, rng.randint(-2, 2, extent) * cell], 1)
    scan[1::3, 1] += 0.5 * cell                       # exactly half a cell: -1.5 -> -2, -0.5 -> 0, 0.5 -> 0, 1.5 -> 2
    scan = scan.astype(np.float32)
    m = scan[rng.rand(extent) < 0.6].copy()
    m[::2, 0] += np.float32(0.5 * cell)               # map points on half cells too
    m = np.concatenate([m, rng.uniform(-15, 15, (4000, 3)).astype(np.float32) * [1, 0.2, 0.1]]).astype(np.float32)
    ctx = _map_ctx(m)
    for hx, hy, A in ((0, 0, 1), (1, 2, 2)):      # one base and no shift: the box is exactly `extent` cells wide
        bases = np.tile(np.eye(4), (A, 1, 1))
        bases[A - 1, 0, 3] += 3 * cell * (A - 1)
        st, vol, *_ = _search(ctx, scan, bases, cell, hx, hy, 0)
        assert st == lib.PLS_OK
        assert np.array_equal(vol, ref.score_volume(scan, bases, cell, hx, hy, m))
    # the half cells really are ties: rint sends both to the even neighbour
    q = scan[1::3, 1].astype(np.float64) / cell
    assert np.any(q % 1 == 0.5)


def test_map_occupancy_is_voxel_hash_of_map_points():
    """Cells of the map are pls_voxel_hash's coordinates of pls_kdmap_points: with the identity base every scan point's
    base cell is its voxel-hash cell, so a window-0 score counts the scan points whose voxel cell holds a map point."""
    rng = np.random.RandomState(3)
    m = (rng.randint(-40, 40, (3000, 3)) * 0.25 + 0.125 * rng.randint(0, 2, (3000, 3))).astype(np.float32)
    ctx = _map_ctx(m)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    pts = km.points()
    scan = (rng.randint(-40, 40, (5000, 3)) * 0.25 + 0.125 * rng.randint(0, 2, (5000, 3))).astype(np.float32)
    for cell in (0.25, 0.5, 1.0):
        mc, sc = np.zeros((pts.shape[0], 3), np.int64), np.zeros((scan.shape[0], 3), np.int64)
        h = np.zeros(max(pts.shape[0], scan.shape[0]), np.int64)
        ctx.call("pls_voxel_hash", lib.ptr(pts), 0, pts.shape[0], cell, lib.ptr(mc), lib.ptr(h))
        ctx.call("pls_voxel_hash", lib.ptr(scan), 0, scan.shape[0], cell, lib.ptr(sc), lib.ptr(h))
        occ = {tuple(c) for c in mc}
        want = sum(tuple(c) in occ for c in sc)
        got = km.score_poses(scan, np.eye(4)[None], cell)
        assert got.tolist() == [want]


def _peak_scene():
    """Scores with constructed plateaus, peaks at the window edges and at a = 0 and a = A - 1."""
    cell = 1.0
    scan = np.array([[0.0, 0.0, 0.0]], np.float32)
    occ = [(-4, -4), (-3, -4), (4, 4), (4, 3), (0, 0), (1, 0), (0, 1), (1, 1), (-4, 2), (2, -3)]
    m = np.array([[x, y, 0.0] for x, y in occ], np.float32)
    A = 5
    bases = np.tile(np.eye(4), (A, 1, 1))
    bases[:, 0, 3] = [0, 0.2, -0.3, 0.4, 0.1]          # the same cell for every base: plateaus across a
    return m, scan, bases, cell


@pytest.mark.parametrize("K", [0, 1, 7, 64, 1024])
def test_top_k_equals_the_reference(K):
    rng = np.random.RandomState(K)
    m, scan = _scene(2000, 0.5, rng, extent=8.0)
    bases = _bases(9, rng, spread=1.0)
    ctx = _map_ctx(m)
    for hx, hy in ((6, 5), (0, 0), (1, 1)):
        st, vol, T, sc, ix, num = _search(ctx, scan, bases, 0.5, hx, hy, K)
        assert st == lib.PLS_OK
        w_vol, w_T, w_sc, w_ix, w_num = ref.search(scan, bases, 0.5, hx, hy, K, m)
        assert np.array_equal(vol, w_vol)
        assert num == w_num and np.array_equal(sc, w_sc) and np.array_equal(ix, w_ix)
        assert np.array_equal(T, w_T)
    # plateaus (the lowest L wins), edge peaks, no wrap in a
    m, scan, bases, cell = _peak_scene()
    ctx = _map_ctx(m)
    st, vol, T, sc, ix, num = _search(ctx, scan, bases, cell, 4, 4, K)
    w_vol, w_T, w_sc, w_ix, w_num = ref.search(scan, bases, cell, 4, 4, K, m)
    assert st == lib.PLS_OK and np.array_equal(vol, w_vol)
    assert num == w_num and np.array_equal(ix, w_ix) and np.array_equal(sc, w_sc) and np.array_equal(T, w_T)
    if K >= 7:
        assert num == len(ref.candidates(w_vol)) == min(K, num)


def test_candidate_rule_edges():
    m, scan, bases, cell = _peak_scene()
    ctx = _map_ctx(m)
    st, vol, T, sc, ix, num = _search(ctx, scan, bases, cell, 4, 4, 1024)
    Wx = Wy = 9
    picked = {(int(L) // (Wx * Wy), (int(L) // Wx) % Wy - 4, int(L) % Wx - 4) for L in ix}
    # every base sees the same cells, so each plateau's winner is its lowest L: at a = 0, the smallest j, then i
    assert {(0, -4, -4), (0, 3, 4), (0, 0, 0), (0, 2, -4), (0, -3, 2)} == picked
    assert all(a == 0 for a, _, _ in picked)
    # no wrap-around: the last base's peaks survive when it is the only one scoring
    bases2 = bases.copy()
    bases2[:-1, 2, 3] = 50.0
    st, vol, T, sc, ix, num = _search(ctx, scan, bases2, cell, 4, 4, 1024)
    assert num > 0 and all(int(L) // (Wx * Wy) == 4 for L in ix)
    assert np.array_equal(ix, ref.search(scan, bases2, cell, 4, 4, 1024, m)[3])


def test_all_zero_volume_and_no_valid_row():
    rng = np.random.RandomState(5)
    m, scan = _scene(500, 0.5, rng, extent=5.0)
    ctx = _map_ctx(m + np.float32(500.0))
    st, vol, T, sc, ix, num = _search(ctx, scan, _bases(3, rng), 0.5, 4, 4, 16)
    assert st == lib.PLS_OK and num == 0 and not vol.any()
    bad = np.full((10, 3), np.nan, np.float32)
    bad[::2, 1] = np.inf
    st, vol, T, sc, ix, num = _search(ctx, bad, _bases(3, rng), 0.5, 4, 4, 16)
    assert st == lib.PLS_OK and num == 0 and vol.shape == (3, 9, 9) and not vol.any()


def test_host_and_device_inputs_give_the_same_bits():
    rng = np.random.RandomState(11)
    m, scan = _scene(3000, 0.5, rng, extent=8.0)
    bases = _bases(6, rng, 1.0)
    ctx = _map_ctx(m)
    st, vol, T, sc, ix, num = _search(ctx, scan, bases, 0.5, 5, 5, 32)
    d_scan = torch.from_numpy(scan).cuda()
    d_bases = torch.from_numpy(bases).cuda()
    d_vol = torch.zeros(vol.shape, dtype=torch.int32, device="cuda")
    d_T, d_sc = torch.zeros((32, 4, 4), dtype=torch.float64, device="cuda"), torch.zeros(32, dtype=torch.int32, device="cuda")
    d_ix, n2 = torch.zeros(32, dtype=torch.int64, device="cuda"), C.c_int(-1)
    torch.cuda.synchronize()
    assert lib.load().pls_kdmap_pose_search(ctx.handle, lib.ptr(d_scan), 3000, lib.ptr(d_bases), 6, 0.5, 5, 5, 32,
                                            lib.ptr(d_vol), lib.ptr(d_T), lib.ptr(d_sc), lib.ptr(d_ix),
                                            C.byref(n2)) == lib.PLS_OK
    assert n2.value == num
    assert np.array_equal(d_vol.cpu().numpy(), vol)
    assert np.array_equal(d_T.cpu().numpy()[:num], T) and np.array_equal(d_sc.cpu().numpy()[:num], sc)
    assert np.array_equal(d_ix.cpu().numpy()[:num], ix)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    T2, sc2, ix2 = km.search_poses(d_scan, d_bases, 0.5, (5, 5), 32)
    assert np.array_equal(T2, T) and np.array_equal(sc2, sc) and np.array_equal(ix2, ix)
    assert np.array_equal(km.score_poses(scan, T2, 0.5), sc)


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


def _same(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_context_is_unchanged():
    a, b = _odometry(), _odometry()
    for k in range(4):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
    before = _state(a)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=4), ctx=a.ctx)
    rng = np.random.RandomState(0)
    T, sc, ix = km.search_poses(syn.scan(4, 32, 512), _bases(8, rng, 1.0), 0.5, (6, 6), 8)
    assert len(sc) > 0
    km.score_poses(syn.scan(4, 32, 512), T, 0.5)
    assert _search(a.ctx, syn.scan(4, 32, 512).astype(np.float32), _bases(2, rng), -1.0, 1, 1, 4)[0] == lib.PLS_E_INVALID
    _same(before, _state(a))
    _same(before, _state(b))
    for k in range(4, 7):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
        assert np.array_equal(a._pose_out, b._pose_out)
        _same(_state(a), _state(b))
    pa, Ta, la = a.register_new_frame(syn.scan(7, 32, 512), np.eye(4, dtype=np.float32))
    pb, Tb, lb = b.register_new_frame(syn.scan(7, 32, 512), np.eye(4, dtype=np.float32))
    assert np.array_equal(Ta, Tb) and np.array_equal(pa, pb) and la == lb


def test_every_refusal_leaves_the_context_unchanged():
    rng = np.random.RandomState(1)
    m, scan = _scene(300, 0.5, rng, extent=5.0)
    ctx = _map_ctx(m)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    pts0 = km.points()
    B = _bases(2, rng)
    L = lib.load()
    out = [np.zeros(64 * 16), np.zeros(64, np.int32), np.zeros(64, np.int64)]

    def call(c, s=scan, ns=None, b=B, A=None, cell=0.5, hx=1, hy=1, K=4):
        num = C.c_int(-5)
        st = L.pls_kdmap_pose_search(c.handle, lib.ptr(s), s.shape[0] if ns is None else ns, lib.ptr(b),
                                     (b.shape[0] if A is None else A) if b is not None else 1, cell, hx, hy, K, None,
                                     lib.ptr(out[0]), lib.ptr(out[1]), lib.ptr(out[2]), C.byref(num))
        return st, num.value

    assert call(ctx)[0] == lib.PLS_OK
    bad_base = B.copy()
    bad_base[1, 2, 1] = np.nan
    inf_base = B.copy()
    inf_base[0, 0, 3] = np.inf
    refusals = [dict(s=None), dict(b=None), dict(ns=0), dict(ns=-3), dict(A=0), dict(A=-1), dict(hx=-1), dict(hy=-1),
                dict(K=-1), dict(K=1025), dict(cell=0.0), dict(cell=-0.5), dict(cell=float("nan")),
                dict(cell=float("inf")), dict(b=bad_base), dict(b=inf_base),
                dict(A=2, hx=20000, hy=20000), dict(cell=1e-4, hx=0, hy=0)]
    for kw in refusals:
        if kw.get("s", 0) is None:
            num = C.c_int(-5)
            st = L.pls_kdmap_pose_search(ctx.handle, None, 10, lib.ptr(B), 2, 0.5, 1, 1, 4, None, lib.ptr(out[0]),
                                         lib.ptr(out[1]), lib.ptr(out[2]), C.byref(num))
        else:
            st, _ = call(ctx, **kw)
        assert st == lib.PLS_E_INVALID, kw
    assert "PLS_POSE_SEARCH_MAX_BITS" in L.pls_last_error(ctx.handle).decode()
    assert " x " in L.pls_last_error(ctx.handle).decode()
    assert np.array_equal(km.points(), pts0)
    fresh = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    assert call(fresh)[0] == lib.PLS_E_INVALID
    assert "before any update" in L.pls_last_error(fresh.handle).decode()
    proj = lib.Context(local_map_type=lib.MAP_PROJECTIVE, height=16, width=64)
    assert call(proj)[0] == lib.PLS_E_INVALID
    assert call(ctx)[0] == lib.PLS_OK


def _hall():
    parts = []
    for k in range(0, 60, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.1)[0]))
    return np.concatenate(parts).astype(np.float32), syn.scan(7, 64, 2048).astype(np.float32)


def test_localize_on_the_synthetic_hall():
    m, scan = _hall()
    o = _odometry(max_align=30)
    b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=o.ctx).set_map_pointcloud(m)
    gt = syn.gt_pose(7)
    th = np.deg2rad(120.0)
    prior = gt.copy()
    prior[:3, :3] = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]) @ gt[:3, :3]
    prior[:2, 3] += 15.0 * np.array([np.cos(0.7), np.sin(0.7)])
    cell, step = 0.5, np.deg2rad(5)
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=o.ctx)
    bases = b200.odometry.yaw_sweep(prior, np.pi, step)
    T, sc, ix = km.search_poses(scan, bases, cell, (32, 32), 8)

    def err(T):
        d = np.linalg.inv(gt) @ T
        return np.linalg.norm(d[:2, 3]), abs(np.arctan2(d[1, 0], d[0, 0]))

    e_t, e_r = err(T[0])
    assert e_t <= cell * np.sqrt(2) + 1e-9 and e_r <= step + 1e-9, (e_t, np.rad2deg(e_r))
    res = o.localize(scan, prior, radius=16.0, cell_size=cell, yaw_step=step, num_candidates=8)
    assert len(res) == 8
    e_t, e_r = err(res[0].T)
    assert e_t <= 0.05 and np.rad2deg(e_r) <= 0.1, (e_t, np.rad2deg(e_r))
    assert [r.coarse_rank for r in res] != [] and res[0].score >= max(r.score for r in res if r.status != lib.PLS_E_SINGULAR)
    # the refined poses are register_new_frame's from the same float32 T0s
    for r in res:
        _, T1, _ = o.register_new_frame(scan, r.T0.astype(np.float32))
        assert np.array_equal(T1[0].astype(np.float64), r.T)
