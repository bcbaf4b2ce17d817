"""pls_kdmap_pose_search_scans on the GPU against per-scan pls_kdmap_pose_search on the same context, bit for bit:
volumes and candidates for S = 1, 2, 64 and 300 (and, up to S = 64, every scan's volume against the float64 reference,
since both calls run the same pipeline), mixed bases, rows and windows (0 x 0, and the score kernel's word and tile edges), NaN rows and scans without a valid row, plateaus with K = 0, 1 and 1024, a batch crossing the 2^29 flag
chunk inside one scan's volume, scans far apart on the 2 km map, host, device and mixed pointers; every refusal, each
leaving the outputs unwritten and the context unchanged; and ICPFrameToModel.localize_scans against a loop of
localize on the scene and the 2 km map."""
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
from oracle import pose_search_reference as ref  # noqa: E402

pytestmark = pytest.mark.gpu


def _map_ctx(points):
    ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    pts = np.ascontiguousarray(points, np.float32)
    ctx.call("pls_kdmap_set_points", lib.ptr(pts), 0, pts.shape[0])
    return ctx


def _single(ctx, scan, bases, cell, hx, hy, K):
    """pls_kdmap_pose_search: (volume, T, score, index)."""
    A = bases.shape[0]
    vol = np.zeros((A, 2 * hy + 1, 2 * hx + 1), np.int32)
    T, sc = np.zeros((max(K, 1), 4, 4)), np.zeros(max(K, 1), np.int32)
    ix, num = np.zeros(max(K, 1), np.int64), C.c_int(-1)
    b = np.ascontiguousarray(bases, np.float64)
    st = lib.load().pls_kdmap_pose_search(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(b), A, float(cell), hx, hy,
                                          K, lib.ptr(vol), lib.ptr(T), lib.ptr(sc), lib.ptr(ix), C.byref(num))
    assert st == lib.PLS_OK, lib.load().pls_last_error(ctx.handle)
    k = num.value
    return vol.reshape(-1), T[:k], sc[:k], ix[:k]


SENTINEL = -7


def _outs(S, V, K, device=False):
    Kc = max(K, 1)
    mk = (lambda a: torch.from_numpy(a).cuda()) if device else (lambda a: a)
    return dict(vol=mk(np.full(V, SENTINEL, np.int32)), T=mk(np.full((S, Kc, 4, 4), SENTINEL, np.float64)),
                score=mk(np.full((S, Kc), SENTINEL, np.int32)), index=mk(np.full((S, Kc), SENTINEL, np.int64)),
                num=mk(np.full(S, SENTINEL, np.int32)))


def _host(o):
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in o.items()}


def _raw(ctx, scans, bases, cell, hxs, hys, K, outs=None, S=None, cat=None, num_bases=None, scores=True):
    """pls_kdmap_pose_search_scans: (status, outputs).  scans and bases entries may be numpy or CUDA tensors."""
    S = len(scans) if S is None else S
    addresses = np.array([lib.ptr(s) or 0 for s in scans], dtype=np.uint64)
    rows = np.array([10 if s is None else s.shape[0] for s in scans], dtype=np.int64)
    if cat is None:
        cat = np.ascontiguousarray(np.concatenate([np.asarray(b, np.float64).reshape(-1, 16) for b in bases]))
    if num_bases is None:
        num_bases = np.array([b.shape[0] for b in bases], dtype=np.int32)
    hx, hy = np.asarray(hxs, np.int32), np.asarray(hys, np.int32)
    V = int(sum(int(a) * (2 * int(x) + 1) * (2 * int(y) + 1) for a, x, y in zip(num_bases, hx, hy)))
    o = _outs(len(scans), max(V, 1), K) if outs is None else outs
    st = lib.load().pls_kdmap_pose_search_scans(
        ctx.handle, lib.ptr(addresses), lib.ptr(rows), S, lib.ptr(cat), lib.ptr(num_bases), float(cell), lib.ptr(hx),
        lib.ptr(hy), K, lib.ptr(o["vol"]) if scores else None, lib.ptr(o["T"]), lib.ptr(o["score"]),
        lib.ptr(o["index"]), lib.ptr(o["num"]))
    torch.cuda.synchronize()
    return st, o


def _check(ctx, scans, bases, cell, hxs, hys, K, want_volumes=None, **kw):
    """The batched call equals the single call per scan, and writes nothing past out_num[s]; returns the candidate
    counts.  want_volumes: each scan's reference score volume, which its part of the batched volume must equal."""
    st, o = _raw(ctx, scans, bases, cell, hxs, hys, K, **kw)
    assert st == lib.PLS_OK, lib.load().pls_last_error(ctx.handle)
    o = _host(o)
    at, nums = 0, []
    for s in range(len(scans)):
        scan = scans[s].cpu().numpy() if isinstance(scans[s], torch.Tensor) else scans[s]
        b = bases[s].cpu().numpy() if isinstance(bases[s], torch.Tensor) else bases[s]
        vol, T, sc, ix = _single(ctx, scan, b, cell, int(hxs[s]), int(hys[s]), K)
        assert np.array_equal(o["vol"][at:at + vol.size], vol), s
        if want_volumes is not None:
            assert np.array_equal(o["vol"][at:at + vol.size], want_volumes[s].reshape(-1)), s
        at += vol.size
        k = int(o["num"][s])
        assert k == len(ix), s
        assert np.array_equal(o["T"][s, :k].reshape(-1, 4, 4), T) and np.array_equal(o["score"][s, :k], sc), s
        assert np.array_equal(o["index"][s, :k], ix), s
        assert np.all(o["score"][s, k:] == SENTINEL) and np.all(o["index"][s, k:] == SENTINEL)
        assert np.all(o["T"][s, k:] == SENTINEL)
        nums.append(k)
    return nums


def _bases(A, rng, spread=2.0, at=(0.0, 0.0)):
    th = rng.uniform(-np.pi, np.pi, A)
    B = np.tile(np.eye(4), (A, 1, 1))
    B[:, 0, 0], B[:, 0, 1], B[:, 1, 0], B[:, 1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    B[:, :3, 3] = rng.uniform(-spread, spread, (A, 3)) * [1, 1, 0.2]
    B[:, :2, 3] += at
    return B


def _scene_map(rng, extent=12.0, cell=0.5):
    return rng.uniform([-extent, -extent, -1.5], [extent, extent, 1.5],
                       (int(3 * (2 * extent / cell) ** 2), 3)).astype(np.float32)


def _scan(n, rng, extent=6.0, bad=True):
    scan = rng.uniform([-extent, -extent, -1.2], [extent, extent, 1.2], (n, 3)).astype(np.float32)
    if bad and n > 3:
        k = rng.choice(n, max(1, n // 50), replace=False)
        scan[k, rng.randint(0, 3, k.size)] = rng.choice([np.nan, np.inf, -np.inf], k.size)
    return scan


# windows (half_x, half_y): 0 x 0, and Wx = 31, 32 (never: odd), 33 / Wy = 7, 9 around the 32-lane and 8-row tiles
WINDOWS = [(0, 0), (15, 3), (16, 4), (1, 1), (0, 5), (7, 0), (32, 2), (3, 16)]


@pytest.mark.parametrize("S", [1, 2, 64, 300])
def test_equals_the_single_call_per_scan(S):
    rng = np.random.RandomState(S)
    m = _scene_map(rng)
    ctx = _map_ctx(m)
    scans, bases, hxs, hys = [], [], [], []
    for s in range(S):
        n = int(rng.choice([1, 7, 255, 256, 1025, 3000] if S <= 64 else [1, 31, 200]))
        scans.append(_scan(n, rng))
        bases.append(_bases(int(rng.randint(1, 5 if S <= 64 else 3)), rng))
        hx, hy = WINDOWS[s % len(WINDOWS)]
        hxs.append(hx)
        hys.append(hy)
    # both calls run the same code: for S <= 64 every scan's volume is also checked against the float64 reference
    want = [ref.score_volume(scans[s], bases[s], 0.5, hxs[s], hys[s], m) for s in range(S)] if S <= 64 else None
    for K in (0, 1, 8, 1024):
        nums = _check(ctx, scans, bases, 0.5, hxs, hys, K, want_volumes=want)
        assert K == 0 or sum(nums) > 0


def test_nan_scans_and_scans_without_a_valid_row():
    rng = np.random.RandomState(5)
    ctx = _map_ctx(_scene_map(rng))
    nan = np.full((40, 3), np.nan, np.float32)
    inf = np.full((3, 3), np.inf, np.float32)
    scans = [nan, _scan(500, rng), inf, _scan(100, rng)]
    bases = [_bases(2, rng) for _ in scans]
    nums = _check(ctx, scans, bases, 0.5, [2, 3, 0, 1], [1, 0, 2, 1], 8)
    assert nums[0] == 0 and nums[2] == 0 and nums[1] > 0
    # every scan without a valid row: all-zero volumes, no candidate
    st, o = _raw(ctx, [nan, inf], bases[:2], 0.5, [1, 2], [1, 0], 4)
    assert st == lib.PLS_OK
    assert np.all(o["vol"][:2 * 9 + 2 * 5] == 0) and o["num"].tolist() == [0, 0]


def test_plateaus_with_many_candidates():
    """A map of every other cell: most poses score alike, thousands of candidates per scan."""
    cell = 1.0
    g = np.stack(np.meshgrid(np.arange(-30, 31, 2), np.arange(-30, 31, 2), [0], indexing="ij"), -1).reshape(-1, 3)
    ctx = _map_ctx(g.astype(np.float32))
    rng = np.random.RandomState(6)
    scans = [np.zeros((1, 3), np.float32), (rng.randint(-3, 4, (20, 3)) * [2, 2, 0]).astype(np.float32)]
    bases = [np.tile(np.eye(4), (3, 1, 1)), np.tile(np.eye(4), (2, 1, 1))]
    for K in (0, 1, 1024):
        nums = _check(ctx, scans, bases, cell, [30, 16], [30, 15], K)
    assert min(nums) > 100


def test_a_batch_crossing_the_flag_chunk_inside_a_scan():
    """Sum V > 2^29 with the chunk boundary of the flag scan inside scan 3's volume."""
    rng = np.random.RandomState(7)
    ctx = _map_ctx(_scene_map(rng, extent=40.0, cell=1.0))
    h = 700
    V = 72 * (2 * h + 1) ** 2
    assert 3 * V < (1 << 29) < 4 * V
    scans = [_scan(60, rng) for _ in range(4)]
    bases = [b200.odometry.yaw_sweep(_bases(1, rng)[0], np.pi, np.deg2rad(5)) for _ in range(4)]
    _check(ctx, scans, bases, 1.0, [h] * 4, [h] * 4, 8)


def _wide_map():
    rng = np.random.RandomState(8)
    return rng.uniform([-1000, -1000, -5], [1000, 1000, 15], (1_000_000, 3)).astype(np.float32)


def test_scans_far_apart_on_the_2km_map():
    ctx = _map_ctx(_wide_map())
    rng = np.random.RandomState(9)
    at = [(-900, -900), (900, 900), (-900, 900), (0, 0), (850, -880)]
    scans = [_scan(2000, rng, extent=30.0) for _ in at]
    bases = [_bases(3, rng, at=a) for a in at]
    _check(ctx, scans, bases, 1.0, [10, 4, 0, 20, 7], [10, 9, 3, 0, 7], 8)


def test_host_device_and_mixed_pointers():
    rng = np.random.RandomState(10)
    ctx = _map_ctx(_scene_map(rng))
    scans = [_scan(n, rng) for n in (300, 1, 2000)]
    bases = [_bases(a, rng) for a in (3, 1, 2)]
    hxs, hys = [4, 0, 16], [3, 2, 4]
    want = _raw(ctx, scans, bases, 0.5, hxs, hys, 8)[1]
    cat = np.ascontiguousarray(np.concatenate([b.reshape(-1, 16) for b in bases]))
    dev_scans = [torch.from_numpy(s).cuda() for s in scans]
    mixed = [dev_scans[0], scans[1], dev_scans[2]]
    for sc, bb, dev_out in ((dev_scans, torch.from_numpy(cat).cuda(), True), (mixed, cat, False),
                            (scans, torch.from_numpy(cat).cuda(), True), (mixed, torch.from_numpy(cat).cuda(), False)):
        outs = _outs(3, want["vol"].size, 8, device=dev_out)
        st, o = _raw(ctx, sc, bases, 0.5, hxs, hys, 8, outs=outs, cat=bb)
        assert st == lib.PLS_OK
        o = _host(o)
        for k in want:
            assert np.array_equal(o[k], want[k]), k
    _check(ctx, mixed, bases, 0.5, hxs, hys, 8)


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


def test_every_refusal_leaves_outputs_and_context_unchanged():
    a, b = _odometry(), _odometry()
    for k in range(4):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
    before = _state(a)
    rng = np.random.RandomState(11)
    scans = [syn.scan(4, 32, 512).astype(np.float32), syn.scan(5, 32, 512).astype(np.float32)]
    B = [_bases(4, rng, 1.0), _bases(3, rng, 1.0)]
    ok_st, _ = _raw(a.ctx, scans, B, 0.5, [3, 3], [3, 3], 4)
    assert ok_st == lib.PLS_OK
    L = lib.load()

    def refused(expect=None, **kw):
        args = dict(scans=scans, bases=B, cell=0.5, hxs=[3, 3], hys=[3, 3], K=4)
        args.update(kw)
        outs = _outs(2, 4096, 8)
        st, o = _raw(a.ctx, outs=outs, **args)
        assert st == lib.PLS_E_INVALID, kw
        msg = L.pls_last_error(a.ctx.handle).decode()
        if expect:
            assert expect in msg, (kw, msg)
        for v in _host(o).values():
            assert np.all(v == SENTINEL), kw
        return msg

    bad, far = [x.copy() for x in B], [x.copy() for x in B]
    bad[1][2, 2, 1] = np.nan
    far[1][0, 0, 3] = 1e12
    empty = np.zeros((0, 3), np.float32)
    refused("scan 1", scans=[scans[0], None])
    refused("scan 1", scans=[scans[0], empty])
    refused("scan 0", num_bases=np.array([0, 3], np.int32))
    refused("scan 1", num_bases=np.array([4, -1], np.int32))
    refused("scan 1", hxs=[3, -1])
    refused("scan 0", hys=[-1, 3])
    refused("scan 1", hxs=[0, 1 << 30])
    refused("scan 1", bases=[B[0], np.tile(np.eye(4), (3, 1, 1))], hxs=[0, 23170], hys=[0, 23170],
            num_bases=np.array([4, 2], np.int32))
    refused("scan 1", bases=bad)
    refused("scan 1", bases=far)
    refused("scan 0", cell=1e-4, hxs=[0, 0], hys=[0, 0])               # scan 0's own occupancy box is too large
    refused("S must be > 0", S=0)
    refused(None, K=-1)
    refused(None, K=1025)
    refused(None, cell=0.0)
    refused(None, cell=float("nan"))
    # sum V >= 2^31 although each volume is below it
    one = [np.eye(4)[None], np.eye(4)[None]]
    refused("2^31", bases=one, hxs=[23000, 23000], hys=[23000, 23000])
    # the union of two reachable boxes over the bit limit, each scan's own box within it
    far2 = [B[0].copy(), B[1].copy()]
    far2[1][:, 0, 3] += 20000.0
    far2[1][:, 1, 3] += 20000.0
    assert _raw(a.ctx, scans[:1], far2[:1], 0.5, [0], [0], 4)[0] == lib.PLS_OK
    assert _raw(a.ctx, scans[1:], far2[1:], 0.5, [0], [0], 4)[0] == lib.PLS_OK
    msg = refused("shared occupancy box", bases=far2, cell=0.5, hxs=[0, 0], hys=[0, 0])
    assert "PLS_POSE_SEARCH_MAX_BITS" in msg
    # NULL arrays
    addresses = np.array([lib.ptr(s) for s in scans], dtype=np.uint64)
    rows = np.array([s.shape[0] for s in scans], dtype=np.int64)
    cat = np.ascontiguousarray(np.concatenate([x.reshape(-1, 16) for x in B]))
    nb, hx = np.array([4, 3], np.int32), np.array([1, 1], np.int32)
    o = _outs(2, 100, 4)
    full = [lib.ptr(addresses), lib.ptr(rows), 2, lib.ptr(cat), lib.ptr(nb), 0.5, lib.ptr(hx), lib.ptr(hx), 4,
            None, lib.ptr(o["T"]), lib.ptr(o["score"]), lib.ptr(o["index"]), lib.ptr(o["num"])]
    for i in (0, 1, 3, 4, 6, 7, 10, 11, 12, 13):
        args = list(full)
        args[i] = None
        assert L.pls_kdmap_pose_search_scans(a.ctx.handle, *args) == lib.PLS_E_INVALID, i
    for v in _host(o).values():
        assert np.all(v == SENTINEL)
    fresh = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
    assert L.pls_kdmap_pose_search_scans(fresh.handle, *full) == lib.PLS_E_INVALID
    proj = lib.Context(local_map_type=lib.MAP_PROJECTIVE, height=16, width=64)
    assert L.pls_kdmap_pose_search_scans(proj.handle, *full) == lib.PLS_E_INVALID
    _equal(before, _state(a))
    _equal(before, _state(b))
    for k in range(4, 7):
        for o in (a, b):
            o.process_next_frame({"numpy_pc": syn.scan(k, 32, 512)})
        assert np.array_equal(a._pose_out, b._pose_out)
        _equal(_state(a), _state(b))


def test_search_poses_scans_halves_a_refused_batch():
    """Scans 8 km apart at a fine cell: the shared grid is refused, the Python layer halves the batch."""
    rng = np.random.RandomState(12)
    ctx = _map_ctx(_scene_map(rng))
    km = b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    scans = [_scan(400, rng) for _ in range(3)]
    bases = [_bases(2, rng, at=a) for a in ((4000.0, 4000.0), (0.0, 0.0), (-4000.0, -4000.0))]
    got = km.search_poses_scans(scans, bases, 0.1, (2, 2), 8)
    for s in range(3):
        want = km.search_poses(scans[s], bases[s], 0.1, (2, 2), 8)
        for g, w in zip(got[s], want):
            assert np.array_equal(g, w)


def _same_candidates(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert (g.score, g.coarse_score, g.coarse_rank, g.iterations, g.status) == \
            (w.score, w.coarse_score, w.coarse_rank, w.iterations, w.status)
        assert np.array_equal(g.T, w.T) and np.array_equal(g.T0, w.T0)


def _localize_case(cloud, offset, monkeypatch):
    """Four scans at their ground-truth poses (moved by `offset` with the map's scene), priors off by known amounts;
    scan 2's window is routed to the pyramid."""
    monkeypatch.setattr(b200.odometry, "POSE_SEARCH_PYRAMID_MIN_POSES", 100_000)
    o = _odometry(max_align=20)
    b200.odometry.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=o.ctx).set_map_pointcloud(cloud)
    frames = [3, 7, 11, 15]
    scans = [syn.scan(k, 64, 2048).astype(np.float32) for k in frames]
    scans[1] = torch.from_numpy(scans[1]).cuda()
    priors = np.stack([syn.gt_pose(k).astype(np.float64) for k in frames])
    priors[:, :2, 3] += offset
    shifts = np.array([[3.0, -2.0], [-4.0, 1.0], [9.0, 7.0], [1.0, 4.0]])
    for s, th in enumerate(np.deg2rad([20.0, -35.0, 50.0, 10.0])):
        R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
        priors[s, :3, :3] = R @ priors[s, :3, :3]
        priors[s, :2, 3] += shifts[s]
    radius = np.array([5.0, 5.0, 12.0, 5.0])
    assert 72 * (2 * 24 + 1) ** 2 >= 100_000 > 72 * (2 * 10 + 1) ** 2
    got = o.localize_scans(scans, priors, radius, cell_size=0.5, num_candidates=4)
    for s in range(4):
        want = o.localize(scans[s], priors[s], radius[s], cell_size=0.5, num_candidates=4)
        assert len(want) > 0
        _same_candidates(got[s], want)


def test_localize_scans_equals_a_loop_of_localize_on_the_scene(monkeypatch):
    parts = []
    for k in range(0, 60, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.1)[0]))
    _localize_case(np.concatenate(parts).astype(np.float32), np.zeros(2), monkeypatch)


def test_localize_scans_equals_a_loop_of_localize_on_the_2km_map(monkeypatch):
    from prior_map_bench import make_maps
    maps, _ = make_maps()
    wide = maps["wide2km"].copy()
    offset = np.array([430.0, -270.0])
    wide[:200_000, :2] += np.float32(offset)
    _localize_case(wide, offset, monkeypatch)
