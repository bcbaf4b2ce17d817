"""Every spherical-projection z-buffer per pixel, bit for bit, against oracle/projection_reference.py.

The device's atan2f / asinf are not correctly rounded, so no host evaluation of a pixel coordinate is exact.  The exact
layer therefore takes the float32 row and column pls_project_pixels computes -- the same inlined project_point every
float32 z-buffer runs -- and applies the z-buffer's rule to them on the host: rint half-to-even, the four bounds,
r > 0, closest first and the lowest index on an exact range tie, the range being range32 in the z-buffer's own
RangeOrder.  Every pixel of every image must then match exactly.  The tolerance layer checks those coordinates against
a float64 evaluation within row_col_bound, and the float64 paths (scan ingestion, a float64 frame) against the float64
pixel rule wherever no candidate lies within that bound of a rounding boundary.

Constructed probes put in one pixel two points whose float32 ranges swap order between kYFirst and kXFirst, exact range
ties, the +-0.0 seam, coordinates of exactly k + 0.5, the H - 1 / W - 1 borders and non-finite points, so that a z-buffer
with the wrong order, rounding, bound or tie rule keeps a different point.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import projection_reference as pr

pytestmark = pytest.mark.gpu

UP, DOWN = 3.0, -24.0
F32 = np.float32
CAP = 16 * 132 * 256                      # grid_for's thread cap in projection.cu: the first wrapped grid-stride index


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def syn():
    from pylidar_slam_b200 import synthetic
    return synthetic


# ---------------------------------------------------------------------------------------------------------- driving
def gpu_pixels(lib, ctx, xyz, H, W):
    """pls_project_pixels: the float32 (row, col) of every point, the bits every float32 z-buffer rounds."""
    xyz = np.ascontiguousarray(xyz, F32).reshape(-1, 3)
    out = np.empty((max(len(xyz), 1), 2), F32)
    if len(xyz):
        ctx.call("pls_project_pixels", lib.ptr(xyz), len(xyz), H, W, UP, DOWN, lib.ptr(out))
    return out[: len(xyz), 0], out[: len(xyz), 1]


def build_map(lib, ctx, xyz, channels, H, W, default=None):
    """pls_build_projection_map (default None) or _filled: xyz [B,n,3], channels [B,n,C] or None -> [B,C,H,W]."""
    B, n, _ = xyz.shape
    xyz = np.ascontiguousarray(xyz, F32)
    Cc = 3 if channels is None else channels.shape[2]
    ch = None if channels is None else np.ascontiguousarray(channels, F32)
    out = np.full((B, Cc, H, W), 12345.0, F32)
    if default is None:
        ctx.call("pls_build_projection_map", lib.ptr(xyz), lib.ptr(ch), B, n, Cc, H, W, UP, DOWN, lib.ptr(out))
    else:
        ctx.call("pls_build_projection_map_filled", lib.ptr(xyz), lib.ptr(ch), B, n, Cc, H, W, UP, DOWN, float(default),
                 lib.ptr(out))
    return out


def index_channels(n, C, xyz):
    """C channels that name the point: its index in two exact float32 halves (C >= 2; the index itself for C = 1), then
    x, y, z and further exact functions of the index."""
    i = np.arange(n, dtype=np.int64)
    if C == 1:
        return (i + 1).astype(F32)[:, None]
    ch = np.empty((n, C), F32)
    ch[:, 0] = (i >> 12).astype(F32)
    ch[:, 1] = (i & 4095).astype(F32) + F32(0.5)
    for c in range(2, C):
        ch[:, c] = xyz[:, c - 2] if c < 5 else ((i * c) & 0xFFFFF).astype(F32)
    return ch


def expected_image(rows, cols, xyz, values, H, W, fill, order=pr.Y_FIRST):
    win = pr.expected_winners(pr.pixel_rule(rows, cols, pr.range32(*xyz.T, order), H, W),
                              pr.range32(*xyz.T, order), H, W)
    img = np.full((values.shape[1], H * W), fill, F32)
    ok = win >= 0
    img[:, ok] = values[win[ok]].T
    return img.reshape(-1, H, W), win


def assert_bits_equal(got, want, what):
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = g != w
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())


# ---------------------------------------------------------------------------------------------------------- scenes
def direction(row, col, H, W):
    """A unit vector whose float64 pixel coordinates are (row, col)."""
    kpi, Hf, Wf, ad, fov = pr.proj_consts(H, W, UP, DOWN, True)
    theta = (np.asarray(col, np.float64) / (0.5 * Wf) - 1.0) * kpi
    phi = (1.0 - np.asarray(row, np.float64) / Hf) * fov - ad
    return np.stack([np.cos(phi) * np.cos(-theta), np.cos(phi) * np.sin(-theta), np.sin(phi)], axis=-1)


def dense_cloud(n, H, W, seed):
    """n points spread over the image (and a margin beyond it), ranges 0.5-80 m, about n / (H W) per pixel."""
    rng = np.random.RandomState(seed)
    rows = rng.uniform(-1.0, H, n)
    cols = rng.uniform(-0.7, W - 0.3, n)
    pts = direction(rows, cols, H, W) * rng.uniform(0.5, 80.0, n)[:, None]
    return pts.astype(F32)


def scene(kind, n, H, W, seed, syn):
    if kind == "scan":
        s = syn.scan(seed, max(H, 2), max(W, 2))
        return np.ascontiguousarray(s[:n] if n else s, F32)
    return dense_cloud(n, H, W, seed)


def order_sensitive_pairs(H, W, count, seed):
    """Pairs of points in one pixel (away from every rounding boundary) whose float32 ranges under kYFirst and kXFirst
    order them differently: the winner of the pair depends on the z-buffer's RangeOrder."""
    rng = np.random.RandomState(seed)
    m = 3000000
    rows = rng.randint(0, H, m) + rng.uniform(-0.3, 0.3, m)
    cols = rng.randint(0, W, m) + rng.uniform(-0.3, 0.3, m)
    p = (direction(rows, cols, H, W) * rng.uniform(2.0, 60.0, m)[:, None]).astype(F32)
    q = p.copy()
    for c in range(3):   # a few ulp apart in every coordinate
        q[:, c] = (p[:, c].view(np.int32) + rng.randint(-3, 4, m)).astype(np.int32).view(F32)
    py, px = pr.range32(*p.T, pr.Y_FIRST), pr.range32(*p.T, pr.X_FIRST)
    qy, qx = pr.range32(*q.T, pr.Y_FIRST), pr.range32(*q.T, pr.X_FIRST)
    swap = ((py < qy) & (px > qx)) | ((py > qy) & (px < qx))
    idx = np.nonzero(swap)[0]
    # one pair per pixel
    _, first = np.unique(np.rint(rows[idx]).astype(np.int64) * W + np.rint(cols[idx]).astype(np.int64), return_index=True)
    idx = idx[first][:count]
    return p[idx], q[idx]


def equal_norm_pairs(H, W, seed, count=400):
    """Pairs of distinct integer vectors with the same squared norm (exact in float32 and float64, so their ranges tie
    exactly in every order), less than a pixel apart."""
    rng = np.random.RandomState(seed)
    out = []
    g = np.arange(-6, 7)
    off = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    while len(out) < count:
        c = np.rint(direction(rng.uniform(0, H - 1), rng.uniform(0, W - 1), H, W) * rng.uniform(800, 2500)).astype(np.int64)
        v = c + off
        n2 = (v * v).sum(1)
        order = np.argsort(n2, kind="stable")
        same = np.nonzero(n2[order][1:] == n2[order][:-1])[0]
        if same.size:
            k = same[rng.randint(same.size)]
            out.append((v[order[k]], v[order[k + 1]]))
    a = np.array([o[0] for o in out], F32)
    b = np.array([o[1] for o in out], F32)
    return a, b


def half_probes(lib, ctx, H, W, seed):
    """Points whose GPU row or column is exactly k + 0.5 (selected from a 1-ulp sweep through the boundary, so that
    only the half-to-even rule decides their pixel), at interior pixels and at -0.5, H - 1.5, H - 0.5, W - 1.5, W - 0.5."""
    rng = np.random.RandomState(seed)
    rows_t = np.concatenate([rng.randint(0, H, 6) + 0.5, [-0.5, H - 1.5, H - 0.5]])
    cols_t = np.concatenate([rng.randint(0, W, 6) + 0.5, [0.5, W - 1.5, W - 0.5]])
    pts = []
    steps = np.arange(-600, 601)
    for target_r in rows_t:   # sweep z through the row boundary
        c = np.clip(rng.uniform(0, W - 1), 1, W - 2)
        d = (direction(target_r, c, H, W) * rng.uniform(5, 40)).astype(F32)
        sw = np.repeat(d[None], steps.size, 0)
        sw[:, 2] = (d[2].view(np.int32) + steps).astype(np.int32).view(F32)
        r, _ = gpu_pixels(lib, ctx, sw, H, W)
        pts.append(sw[r == F32(target_r)][:2])
    for target_c in cols_t:   # sweep y through the column boundary
        rr = np.clip(rng.uniform(0, H - 1), 0.2, H - 1.2)
        d = (direction(rr, target_c, H, W) * rng.uniform(5, 40)).astype(F32)
        sw = np.repeat(d[None], steps.size, 0)
        sw[:, 1] = (d[1].view(np.int32) + steps).astype(np.int32).view(F32)
        _, cc = gpu_pixels(lib, ctx, sw, H, W)
        pts.append(sw[cc == F32(target_c)][:2])
    return np.concatenate(pts).astype(F32)


def seam_and_nonfinite(H, W):
    """+0.0 / -0.0 at the +-pi seam (columns 0 and W: the second is dropped), the null point, NaN and +-inf."""
    d = direction(H / 2.0, 0.0, H, W)[None] * 10.0
    plus = np.array([[-abs(d[0, 0]), 0.0, d[0, 2]]], F32)
    minus = plus.copy()
    minus[0, 1] = -0.0
    bad = [[0, 0, 0], [-0.0, 0.0, -0.0]]
    for c in range(3):
        for v in (np.nan, np.inf, -np.inf):
            p = [-5.0, 1.0, -0.5]
            p[c] = v
            bad.append(p)
    return plus, minus, np.array(bad, F32)


@pytest.fixture(scope="module")
def probes(lib, ctx):
    """The probe cloud at (64, 1024): (points, tags) with tags naming each probe's kind."""
    H, W = 64, 1024
    p, q = order_sensitive_pairs(H, W, 1500, 1)
    a, b = equal_norm_pairs(H, W, 2)
    half = half_probes(lib, ctx, H, W, 3)
    plus, minus, bad = seam_and_nonfinite(H, W)
    dup = (direction(np.arange(40) % H + 0.1, np.arange(40) * 25 + 0.2, H, W) * 7.0).astype(F32)
    parts = [("pair_a", p), ("pair_b", q), ("norm_a", a), ("norm_b", b), ("half", half), ("seam_plus", plus),
             ("seam_minus", minus), ("nonfinite", bad), ("dup", dup), ("dup", dup)]
    # which member of an order-sensitive pair is closer under either order is random, so the index does not pick it
    pts = np.concatenate([x for _, x in parts]).astype(F32)
    tags = np.concatenate([[t] * len(x) for t, x in parts])
    return dict(H=H, W=W, pts=pts, tags=tags, n_pairs=len(p), n_norm=len(a), n_half=len(half))


# ---------------------------------------------------------------------------------------------------------- exact layer
CASES = [  # (B, n, C, H, W, scene)
    (1, 0, 3, 64, 1024, "dense"),
    (1, 1, 1, 1, 1, "dense"),
    (1, 2, 4, 1, 7, "dense"),
    (2, 40, 3, 1, 7, "dense"),
    (1, 0, 64, 33, 500, "scan"),
    (1, 0, 3, 33, 500, "scan"),               # no channels: the xyz are scattered
    (2, 60000, 4, 64, 1024, "scan"),
    (5, 16000, 64, 33, 500, "scan"),
    (1, 540671, 4, 128, 2048, "dense"),
    (1, CAP, 1, 128, 2048, "dense"),
    (1, CAP + 1, 3, 64, 1024, "dense"),
    (2, 300000, 4, 64, 1024, "dense"),        # B n across the cap
    (1, 20 * 64 * 1024, 3, 64, 1024, "dense"),  # about 20 points per pixel
    (5, 30000, 3, 128, 2048, "dense"),        # B H W across the cap in the resolve kernel
]


@pytest.mark.parametrize("B,n,C,H,W,kind", CASES)
def test_projection_map_every_pixel(lib, ctx, syn, B, n, C, H, W, kind):
    clouds = [scene(kind, n, H, W, 10 * b + 1, syn) for b in range(B)]
    n = min(len(c) for c in clouds) if kind == "scan" else n
    xyz = np.stack([c[:n] for c in clouds]).reshape(B, n, 3)
    chans = np.stack([index_channels(n, C, xyz[b]) for b in range(B)]).reshape(B, n, C) if C != 3 or kind == "dense" else None
    out = build_map(lib, ctx, xyz, chans, H, W)
    filled = build_map(lib, ctx, xyz, chans, H, W, default=-7.25)
    nan_filled = build_map(lib, ctx, xyz, chans, H, W, default=float("nan"))
    ambiguous = 0
    for b in range(B):
        rows, cols = gpu_pixels(lib, ctx, xyz[b], H, W)
        vals = xyz[b] if chans is None else chans[b]
        want, win = expected_image(rows, cols, xyz[b], vals, H, W, 0.0)
        assert_bits_equal(out[b], want, ("zero default", b))
        want_f, _ = expected_image(rows, cols, xyz[b], vals, H, W, -7.25)
        assert_bits_equal(filled[b], want_f, ("default -7.25", b))
        want_n, _ = expected_image(rows, cols, xyz[b], vals, H, W, np.nan)
        assert_bits_equal(nan_filled[b], want_n, ("NaN default", b))
        if n:
            # tolerance layer: the GPU's coordinates against float64 within the documented bound
            row64, col64, _ = pr.pixels64(xyz[b], H, W, UP, DOWN)
            drow, dcol = pr.row_col_bound(xyz[b], H, W, UP, DOWN)
            fin = np.isfinite(xyz[b]).all(1)
            assert np.all(np.abs(rows[fin].astype(np.float64) - row64[fin]) <= drow[fin]), "row outside row_col_bound"
            assert np.all(np.abs(cols[fin].astype(np.float64) - col64[fin]) <= dcol[fin]), "col outside row_col_bound"
            near = pr.near_half(row64, drow) | pr.near_half(col64, dcol)
            pix64 = pr.pixel_rule(row64, col64, np.ones_like(row64), H, W)
            pix32 = pr.pixel_rule(rows, cols, np.ones_like(row64), H, W)
            assert np.all((pix64 == pix32) | near), "a GPU pixel differs from float64 away from a boundary"
            ambiguous += int(near.sum())
    print(f"[projection] B={B} n={n} C={C} {H}x{W}: boundary-ambiguous points {ambiguous} of {B * n}")
    assert ambiguous <= max(2, 1e-3 * B * n)
    if n and C != 3:
        assert (win >= 0).sum() > 0


def test_probes_in_projection_map(lib, ctx, probes):
    """Each probe's property first, then the exact z-buffer rule on it."""
    H, W, pts, tags = probes["H"], probes["W"], probes["pts"], probes["tags"]
    rows, cols = gpu_pixels(lib, ctx, pts, H, W)
    pix = pr.pixel_rule(rows, cols, pr.range32(*pts.T), H, W)
    pa, pb = np.nonzero(tags == "pair_a")[0], np.nonzero(tags == "pair_b")[0]
    assert len(pa) >= 500
    assert np.array_equal(pix[pa], pix[pb]) and (pix[pa] >= 0).all(), "a pair is not in one pixel"
    ry, rx = pr.range32(*pts.T, pr.Y_FIRST), pr.range32(*pts.T, pr.X_FIRST)
    assert np.all((ry[pa] < ry[pb]) != (rx[pa] < rx[pb])), "a pair's order does not depend on the RangeOrder"
    na, nb = np.nonzero(tags == "norm_a")[0], np.nonzero(tags == "norm_b")[0]
    assert np.all(ry[na] == ry[nb]) and np.all(rx[na] == rx[nb]) and np.all(np.any(pts[na] != pts[nb], axis=1))
    same = pix[na] == pix[nb]
    assert same.sum() >= 50, "too few equal-norm pairs share a pixel"
    hp = tags == "half"
    assert hp.sum() >= 20 and np.all((rows[hp] - np.floor(rows[hp]) == 0.5) | (cols[hp] - np.floor(cols[hp]) == 0.5))
    assert np.any(rows[hp] == F32(-0.5)) and np.any(cols[hp] == F32(W - 0.5)), "the border half-pixels were not hit"
    sp, sm = np.nonzero(tags == "seam_plus")[0], np.nonzero(tags == "seam_minus")[0]
    assert cols[sp][0] == 0.0 and cols[sm][0] == F32(W), (cols[sp], cols[sm])
    assert pix[sp][0] >= 0 and pix[sm][0] == -1
    print(f"[probes] order-sensitive pairs {len(pa)}, equal-norm pairs in one pixel {int(same.sum())}, "
          f"half-pixel points {int(hp.sum())}")
    for C in (1, 3, 64):
        ch = index_channels(len(pts), C, pts)
        out = build_map(lib, ctx, pts[None], ch[None], H, W, default=float("nan"))[0]
        want, win = expected_image(rows, cols, pts, ch, H, W, np.nan)
        assert_bits_equal(out, want, ("probes", C))
    # the winners of the pixels a pair or a tie has to itself: the kYFirst member, the lower index
    alone = np.bincount(pix[pix >= 0], minlength=H * W) == 2
    sel = alone[pix[pa]]
    assert sel.sum() >= 0.9 * len(pa)
    assert np.array_equal(win[pix[pa][sel]], np.where(ry[pa] < ry[pb], pa, pb)[sel])
    tsel = same & (pix[na] >= 0) & alone[np.maximum(pix[na], 0)]
    assert tsel.sum() >= 50
    assert np.array_equal(win[pix[na][tsel]], np.minimum(na, nb)[tsel])


# ---------------------------------------------------------------------------------------------------------- one rule
def _projective_ctx(lib, H, W):
    return lib.Context(height=H, width=W, up_fov_deg=UP, down_fov_deg=DOWN, local_map_type=lib.MAP_PROJECTIVE,
                       local_map_size=1, gn_max_iters=1, max_num_alignments=1)


def _clean_probes(lib, ctx, probes):
    """The finite probes away from every rounding boundary (their pixel cannot depend on the range's last ulp), and a
    background point at the centre of every pixel, far behind them.  A vertex map has one slot per pixel: the probes take
    the first slots, so only the background points of the remaining slots are kept, and the pixels of the first slots
    hold a model candidate only where a probe lands."""
    H, W, pts, tags = probes["H"], probes["W"], probes["pts"], probes["tags"]
    row64, col64, _ = pr.pixels64(pts, H, W, UP, DOWN)
    drow, dcol = pr.row_col_bound(pts, H, W, UP, DOWN)
    keep = np.isfinite(pts).all(1) & ~(pr.near_half(row64, 4 * drow) | pr.near_half(col64, 4 * dcol))
    keep &= np.abs(pts).max(1) > 0
    rr, cc = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    bg = (direction(rr.ravel().astype(np.float64), cc.ravel().astype(np.float64), H, W) * 90.0).astype(F32)
    return pts[keep], tags[keep], bg


def test_every_zbuffer_keeps_its_own_orders_winner(lib, ctx, probes):
    """The model z-buffer (kYFirst, read through pls_projmap_model) and the query z-buffer (kXFirst, read through
    pls_projmap_nn_search's targets in row-major pixel order) at the identity pose, where transform_point is exact."""
    H, W = probes["H"], probes["W"]
    pts, tags, bg = _clean_probes(lib, ctx, probes)
    hw = H * W
    assert len(pts) < hw
    # model: probe i in vertex-map slot i, the background in the remaining slots (index = slot)
    slots = np.concatenate([pts, bg[len(pts):]])
    vm = np.ascontiguousarray(slots.T.reshape(3, H, W))
    moved = pr.transform32(np.eye(4, dtype=F32), slots)
    rows, cols = gpu_pixels(lib, ctx, moved, H, W)
    want, win_model = expected_image(rows, cols, moved, moved, H, W, 0.0, pr.Y_FIRST)
    pm = _projective_ctx(lib, H, W)
    try:
        pm.call("pls_projmap_update", lib.ptr(np.eye(4, dtype=F32).reshape(16)), lib.ptr(vm))
        v = np.empty((1, 3, H, W), F32)
        pm.call("pls_projmap_model", lib.ptr(v), None)
        has_model = np.abs(v[0]).reshape(3, -1).max(0) > 0
        assert_bits_equal(v[0], want, "model z-buffer")
        # query z-buffer: the probes as queries, kXFirst
        q = np.ascontiguousarray(pts)
        nb, nrm, tg, cnt = (np.empty((hw, 3), F32), np.empty((hw, 3), F32), np.empty((hw, 3), F32), C.c_int64(0))
        pm.call("pls_projmap_nn_search", lib.ptr(q), len(q), lib.ptr(nb), lib.ptr(nrm), lib.ptr(tg), C.byref(cnt))
    finally:
        pm.close()
    qr, qc = gpu_pixels(lib, ctx, q, H, W)
    wq = pr.expected_winners(pr.pixel_rule(qr, qc, pr.range32(*q.T, pr.X_FIRST), H, W), pr.range32(*q.T, pr.X_FIRST), H, W)
    # the targets are those of the pixels with a query and a model candidate; every probe pixel has its own candidate
    assert has_model[wq >= 0].mean() > 0.99
    occupied = np.nonzero((wq >= 0) & has_model)[0]
    assert cnt.value == occupied.size
    assert_bits_equal(tg[: cnt.value], q[wq[occupied]], "query z-buffer")
    # the orders differ on the probes: each z-buffer must have decided at least one pair the other way
    pa, pb = np.nonzero(tags == "pair_a")[0], np.nonzero(tags == "pair_b")[0]
    wy = np.where(pr.range32(*q[pa].T, pr.Y_FIRST) < pr.range32(*q[pb].T, pr.Y_FIRST), pa, pb)
    wx = np.where(pr.range32(*q[pa].T, pr.X_FIRST) < pr.range32(*q[pb].T, pr.X_FIRST), pa, pb)
    pix = pr.pixel_rule(qr[pa], qc[pa], np.ones(len(pa)), H, W)
    allp = pr.pixel_rule(qr, qc, np.ones(len(q)), H, W)
    sel = (np.bincount(allp[allp >= 0], minlength=hw) == 2)[pix]      # pixels a pair has to itself
    assert sel.sum() >= 0.9 * len(pa) and np.all(wx != wy)
    assert np.all(win_model[pix[sel]] == wy[sel]) and np.all(wq[pix[sel]] == wx[sel])
    print(f"[one rule] order-sensitive pairs checked: model z-buffer {int(sel.sum())}, query z-buffer {int(sel.sum())}")


def _pose():
    """A float32 pose with every rotation entry and the translation non-trivial."""
    from scipy.spatial.transform import Rotation
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec(np.array([0.3, -0.2, 0.9]) / np.linalg.norm([0.3, -0.2, 0.9]) * 0.4).as_matrix()
    P[:3, 3] = [1.25, -0.75, 0.375]
    return P.astype(F32)


def _transform_y_first(T, p):
    """transform_point with the first two terms swapped, add(fma(z, T2, fma(y, T1, x T0)), T3): a different rounding."""
    T = np.asarray(T, F32).reshape(-1)
    out = np.empty_like(p)
    for c in range(3):
        out[:, c] = pr.add32(pr.fma32(p[:, 2], T[4 * c + 2], pr.fma32(p[:, 1], T[4 * c + 1], pr.mul32(p[:, 0], T[4 * c]))),
                             T[4 * c + 3])
    return out


def test_model_zbuffer_under_a_pose(lib, ctx, probes):
    """The first frame of a projective map is stored with the pose it is given, so the model z-buffer moves every vertex
    with transform_point: the model must be transform32 of the kYFirst winners among the moved points, every pixel, bit
    for bit.  The pixels and ranges are those of the moved points (pls_project_pixels on the exact moved bits), so no
    point needs to be clear of a rounding boundary.  The vertices are the probes moved back by the inverse pose, so
    that the moved cloud again holds the probes' pairs, ties and borders."""
    H, W = probes["H"], probes["W"]
    pts, tags, bg = _clean_probes(lib, ctx, probes)
    hw = H * W
    P = _pose()
    P64 = P.astype(np.float64)
    target = np.concatenate([pts, bg[len(pts):]]).astype(np.float64)
    slots = ((target - P64[:3, 3]) @ np.linalg.inv(P64[:3, :3]).T).astype(F32)
    vm = np.ascontiguousarray(slots.T.reshape(3, H, W))
    moved = pr.transform32(P, slots)
    rows, cols = gpu_pixels(lib, ctx, moved, H, W)
    want, win = expected_image(rows, cols, moved, moved, H, W, 0.0, pr.Y_FIRST)
    # the property: the rounding of the transform decides bits of the model, and the pose keeps order-sensitive pairs
    other = _transform_y_first(P, slots)
    occ = win[win >= 0]
    differ = np.any(other[occ] != moved[occ], axis=1)
    assert differ.sum() >= 1000, "the transform's rounding order does not change the winners' bits"
    ry, rx = pr.range32(*moved.T, pr.Y_FIRST), pr.range32(*moved.T, pr.X_FIRST)
    pa, pb = np.nonzero(tags == "pair_a")[0], np.nonzero(tags == "pair_b")[0]
    pix = pr.pixel_rule(rows, cols, ry, H, W)
    swap = (pix[pa] >= 0) & (pix[pa] == pix[pb]) & ((ry[pa] < ry[pb]) != (rx[pa] < rx[pb]))
    pm = _projective_ctx(lib, H, W)
    try:
        pm.call("pls_projmap_update", lib.ptr(np.ascontiguousarray(P.reshape(16))), lib.ptr(vm))
        v = np.empty((1, 3, H, W), F32)
        pm.call("pls_projmap_model", lib.ptr(v), None)
    finally:
        pm.close()
    assert_bits_equal(v[0], want, "model z-buffer under a pose")
    print(f"[pose] winners whose bits depend on the transform's rounding order {int(differ.sum())} of {occ.size}, "
          f"order-sensitive pairs after the move {int(swap.sum())}")


def test_kd_frame_queries_are_the_zbuffer_winners(lib, ctx, probes, syn):
    """zbuf_points_kernel + FrameInputSelect: a kd frame whose queries are its vertex map's pixels keeps exactly the
    kYFirst winners; a query whose range the selection recomputed in another order would be dropped."""
    H, W = probes["H"], probes["W"]
    pts, tags, _ = _clean_probes(lib, ctx, probes)
    scan = np.ascontiguousarray(syn.scan(0, H, W), F32)
    cloud = np.ascontiguousarray(np.concatenate([scan, pts]))
    rows, cols = gpu_pixels(lib, ctx, cloud, H, W)
    ry = pr.range32(*cloud.T, pr.Y_FIRST)
    pix = pr.pixel_rule(rows, cols, ry, H, W)
    win = pr.expected_winners(pix, ry, H, W)
    # the order-sensitive pairs that hold the two closest points of their pixel (the scan fills every pixel): this
    # z-buffer keeps their kYFirst member, and a selection in kXFirst would drop it for about half of them
    pa, pb = len(scan) + np.nonzero(tags == "pair_a")[0], len(scan) + np.nonzero(tags == "pair_b")[0]
    top = np.maximum(ry[pa], ry[pb])
    order = np.argsort(pix, kind="stable")
    lo, hi = np.searchsorted(pix[order], pix[pa], "left"), np.searchsorted(pix[order], pix[pa], "right")
    two = np.array([p >= 0 and int((ry[order[a:b]] <= t).sum()) == 2 for p, a, b, t in zip(pix[pa], lo, hi, top)])
    two &= pix[pa] == pix[pb]
    assert two.sum() >= 300
    print(f"[one rule] order-sensitive pairs checked: kd frame z-buffer {int(two.sum())}")
    c = lib.Context(height=H, width=W, up_fov_deg=UP, down_fov_deg=DOWN, local_map_type=lib.MAP_KDTREE, local_map_size=1,
                    gn_max_iters=1, max_num_alignments=1)
    try:
        T, params, info, has = np.eye(4, dtype=F32).reshape(16), np.zeros(6, F32), np.zeros(12, np.float64), C.c_int(0)
        for _ in range(2):
            c.call("pls_process_frame", lib.ptr(cloud), lib.INPUT_TENSOR, len(cloud), lib.ptr(np.eye(4, dtype=F32).reshape(16)),
                   lib.ptr(T), lib.ptr(params), C.byref(has), lib.ptr(info))
        # the export accepts exactly the query count of the last search
        c.call("pls_kdmap_last_correspondences", int((win >= 0).sum()), None, None, None, None, None)
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------- float64
def _kitti_correct64(scan):
    """kitti_correct_point on the host: the float32 axis and outer product, the float64 rotation."""
    x, y, z = (scan[:, k].astype(F32) for k in range(3))
    a0, a1 = y, -x
    nrm = np.sqrt(add_f32(a0 * a0, a1 * a1)).astype(F32)
    u0, u1 = (a0 / nrm).astype(F32), (a1 / nrm).astype(F32)
    th = 0.205 * 3.141592653589793 / 180.0
    c, s = np.cos(th), np.sin(th)
    o00, o01, o11 = (u0 * u0).astype(np.float64), (u0 * u1).astype(np.float64), (u1 * u1).astype(np.float64)
    k = 1.0 - c
    px, py, pz = x.astype(np.float64), y.astype(np.float64), z.astype(np.float64)
    rows = [(c + k * o00, k * o01, s * u1.astype(np.float64)), (k * o01, c + k * o11, s * (-u0).astype(np.float64)),
            (s * (-u1).astype(np.float64), s * u0.astype(np.float64), np.full_like(px, c))]
    out = np.stack([r0 * px + r1 * py + r2 * pz for r0, r1, r2 in rows], 1)
    mag = np.stack([np.abs(r0 * px) + np.abs(r1 * py) + np.abs(r2 * pz) for r0, r1, r2 in rows], 1)
    return out, mag


def add_f32(a, b):
    return (a.astype(np.float64) + b.astype(np.float64)).astype(F32)


def winners64(xyz, H, W):
    """The float64 two-pass winner of every pixel, exact where decidable: (winners, pixels left undecided).  Pixels a
    boundary-ambiguous point may reach are undecided; near range ties are settled with the exactly rounded range."""
    row, col, r = pr.pixels64(xyz, H, W, UP, DOWN, f32_consts=False)
    # the host's own float64 evaluation errs by up to the same bound: a point is decided beyond twice the bound
    drow, dcol = (2 * b for b in pr.row_col_bound(xyz, H, W, UP, DOWN, f32=False))
    near = pr.near_half(row, drow) | pr.near_half(col, dcol)
    fin = np.isfinite(xyz).all(1)
    pix = pr.pixel_rule(row, col, r, H, W)
    pix[~fin] = -1
    key = r.copy()
    ok = pix >= 0
    lo = np.full(H * W, np.inf)
    np.minimum.at(lo, pix[ok], r[ok])
    close = ok & (r <= lo[np.maximum(pix, 0)] * (1 + 2.0 ** -48))
    for i in np.nonzero(close)[0]:
        key[i] = pr.range64_exact(*xyz[i])
    win = pr.expected_winners(pix, key, H, W)
    undecided = np.zeros(H * W, bool)
    amb = np.nonzero(near & fin)[0]
    if amb.size:
        reach = pr.pixels_within(row[amb], col[amb], drow[amb], dcol[amb], H, W).ravel()
        undecided[reach[reach >= 0]] = True
    return win, undecided, int(close.sum())


def float64_probes(H, W):
    """Duplicates and equal-norm integer vectors (exact float64 ties: the lowest index wins), and pairs whose float32
    ranges tie while their float64 ranges do not (the float64 winner, placed at the higher index, must win)."""
    a, b = equal_norm_pairs(H, W, 5, 200)
    rng = np.random.RandomState(6)
    m = 200000
    p = (direction(rng.randint(0, H, m) + rng.uniform(-0.3, 0.3, m), rng.randint(0, W, m) + rng.uniform(-0.3, 0.3, m),
                   H, W) * rng.uniform(3, 50, m)[:, None]).astype(F32)
    q = p.copy()
    q[:, 0] = np.nextafter(p[:, 0], F32(np.inf) * np.sign(p[:, 0]))   # one float32 ulp further out in x
    tie32 = pr.range32(*p.T) == pr.range32(*q.T)
    p, q = p[tie32][:600], q[tie32][:600]
    # q is farther in float64; put it first so that a lowest-index rule on float32 ranges would keep it
    return np.concatenate([a, b, a[:50], q, p]).astype(F32), dict(n_norm=len(a), n_far=len(q))


@pytest.mark.parametrize("correct,stride", [(0, 3), (0, 4), (1, 3), (1, 4)])
def test_ingest_scan_float64_winners(lib, ctx, syn, correct, stride):
    H, W = 64, 1024
    probe, info = float64_probes(H, W)
    base = syn.scan(7, H, W)
    base = base[np.isfinite(base).all(1)]
    pts = np.concatenate([base, base[::5], probe]).astype(F32)
    scan = np.concatenate([pts, np.arange(len(pts), dtype=F32)[:, None]], 1) if stride == 4 else pts
    scan = np.ascontiguousarray(scan, F32)
    xyz = np.empty((len(scan), 3), np.float64)
    vm = np.empty((3, H, W), np.float64)
    ctx.call("pls_ingest_scan", lib.ptr(scan), len(scan), stride, correct, H, W, UP, DOWN, lib.ptr(xyz), lib.ptr(vm))
    if correct:
        want, mag = _kitti_correct64(pts)
        fin = np.isfinite(want).all(1)
        assert np.all(np.isnan(xyz[~fin])), "a point on the vertical axis must come out NaN"
        assert np.all(np.abs(xyz[fin] - want[fin]) <= 4 * 2.0 ** -53 * mag[fin]), "kitti correction beyond float64 rounding"
    else:
        assert np.array_equal(xyz, pts.astype(np.float64))
    win, undecided, exact = winners64(xyz, H, W)
    want_vm = np.zeros((3, H * W))
    ok = win >= 0
    want_vm[:, ok] = xyz[win[ok]].T
    got = vm.reshape(3, -1)
    bad = np.any(got.view(np.uint64) != want_vm.view(np.uint64), 0) & ~undecided
    print(f"[ingest] correct={correct} stride={stride}: undecided pixels {int(undecided.sum())} of {H * W}, "
          f"ranges settled exactly {exact}")
    assert not bad.any(), (int(bad.sum()), np.nonzero(bad)[0][:5])
    assert undecided.sum() <= 1e-3 * H * W
    if not correct:
        # the float32 tie that float64 breaks: the farther point comes first, the nearer one must win
        nf, n0 = info["n_far"], len(pts) - 2 * info["n_far"]
        far, near = np.arange(n0, n0 + nf), np.arange(n0 + nf, n0 + 2 * nf)
        r32 = pr.range32(*pts.T)
        assert nf >= 100 and np.all(r32[far] == r32[near])
        assert all(pr.range64_exact(*xyz[i]) > pr.range64_exact(*xyz[j]) for i, j in zip(far, near))
        allpix = pr.pixel_rule(*pr.pixels64(xyz, H, W, UP, DOWN, False)[:2], np.ones(len(xyz)), H, W)
        pix = allpix[near]
        assert np.array_equal(allpix[far], pix), "a float32-tied pair is not in one pixel"
        # the scan fills every pixel: the pixels where the pair holds the two closest points are the pair's
        r64 = pr.pixels64(xyz, H, W, UP, DOWN, False)[2]
        two = np.array([p >= 0 and int(((allpix == p) & (r64 <= r64[f])).sum()) == 2 for p, f in zip(pix, far)])
        mine = two & ~undecided[np.maximum(pix, 0)]
        assert mine.sum() >= 100
        assert np.array_equal(win[pix[mine]], near[mine])
        assert_bits_equal(np.ascontiguousarray(got[:, pix[mine]]), np.ascontiguousarray(xyz[near[mine]].T),
                          "float64 tie broken by float64")


def test_float64_frame_vertex_map(lib, syn):
    """A float64 cloud through the frame input (launch_projection_f64): the first kd frame inserts its vertex map's
    pixels with |p| > 0.01, row-major, each the float32 rounding of the float64 winner."""
    import pylidar_slam_b200 as b200
    H, W = 64, 1024
    probe, _ = float64_probes(H, W)
    base = syn.scan(4, H, W).astype(np.float64) * (1 + 1e-9)
    base = base[np.isfinite(base).all(1)]
    pc = np.ascontiguousarray(np.concatenate([base, probe.astype(np.float64)]))
    win, undecided, _ = winners64(pc, H, W)
    cfg = b200.ICPFrameToModelConfig(local_map=b200.KdTreeLocalMapConfig(local_map_size=4), max_num_alignments=1,
                                     data_key="numpy_pc", alignment=b200.GaussNewtonPointToPlaneConfig())
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=UP, down_fov=DOWN),
                                device="cuda:0")
    try:
        algo.init()
        algo.process_next_frame({"numpy_pc": pc})
        m = C.c_int64(0)
        algo.ctx.call("pls_kdmap_size", C.byref(m))
        got = np.zeros((m.value, 3), F32)
        algo.ctx.call("pls_kdmap_points", lib.ptr(got))
    finally:
        algo.ctx.close()
    assert not undecided.any() or undecided.sum() <= 10
    occ = np.nonzero(win >= 0)[0]
    want = pc[win[occ]].astype(F32)
    keep = np.linalg.norm(want, axis=1) > 0.01
    if not undecided.any():
        assert_bits_equal(got, np.ascontiguousarray(want[keep]), "float64 frame vertex map")
    else:
        assert got.shape[0] == keep.sum()


# ---------------------------------------------------------------------------------------------------------- neighbours
def neighbour_scene(K, Cf, H, W, seed):
    """Target and K reference maps: random vertices, null targets, all-null pixels, null candidates between live ones,
    dyadic exact ties (every distance exact in float32), near ties."""
    rng = np.random.RandomState(seed)
    hw = H * W
    t = (rng.standard_normal((3, hw)) * 10).astype(F32)
    ref = (t[None] + rng.standard_normal((K, 3, hw)).astype(F32) * F32(0.5)).astype(F32)
    null_c = rng.uniform(size=(K, hw)) < 0.25
    ref.transpose(0, 2, 1)[null_c] = 0.0
    t[:, rng.uniform(size=hw) < 0.05] = 0.0                   # null targets
    ref[:, :, rng.uniform(size=hw) < 0.05] = 0.0              # every reference null: index 0
    # dyadic ties: target on a 2^-8 grid, candidates at equal-length dyadic offsets (permuted / sign-flipped)
    tie = np.nonzero(rng.uniform(size=hw) < 0.1)[0]
    t[:, tie] = np.round(t[:, tie] * 256) / 256
    offs = np.array([[0.5, 0.25, 0.125], [0.25, 0.5, -0.125], [-0.125, 0.25, 0.5], [0.5, -0.125, -0.25]], F32)
    for k in range(K):
        ref[k][:, tie] = t[:, tie] + offs[rng.randint(0, 4, tie.size)].T
    fields = None if Cf == 0 else rng.standard_normal((K, Cf, hw)).astype(F32)
    return t.reshape(1, 3, H, W), ref.reshape(K, 3, H, W), None if fields is None else fields.reshape(K, Cf, H, W)


@pytest.mark.parametrize("K", [1, 2, 5, 20])
@pytest.mark.parametrize("Cf", [0, 1, 4])
def test_compute_neighbors_argmin(lib, ctx, K, Cf):
    H, W = 33, 500
    hw = H * W
    t, ref, fields = neighbour_scene(K, Cf, H, W, 100 * K + Cf)
    nb = np.empty((1, 3, H, W), F32)
    nf = None if Cf == 0 else np.empty((1, Cf, H, W), F32)
    ctx.call("pls_compute_neighbors", lib.ptr(t), lib.ptr(ref), lib.ptr(fields), K, Cf, H, W, lib.ptr(nb), lib.ptr(nf))
    tt = t.reshape(3, hw).astype(np.float64)
    rr = ref.reshape(K, 3, hw).astype(np.float64)
    d = np.sqrt(((tt[None] - rr) ** 2).sum(1))
    d[np.abs(rr).max(1) == 0] = np.inf
    t_ok = np.abs(tt).max(0) > 0
    kexp = np.argmin(d, 0)                                    # the first minimum
    ds = np.sort(d, 0)
    # float32 error of each distance: the rounded differences, squares and sums, about 3u relative
    gap_ok = (ds[1] - ds[0] > 8 * 2.0 ** -24 * ds[1]) | (ds[1] == ds[0]) | ~np.isfinite(ds[1]) if K > 1 else np.ones(hw, bool)
    exact_tie = (K > 1) & (ds[0] == ds[1]) if K > 1 else np.zeros(hw, bool)
    # the dyadic ties are exact in float32 too: they must pick the first minimum; other exact float64 ties are rare
    got = nb.reshape(3, hw)
    want = np.where(t_ok, rr[kexp, :, np.arange(hw)].T, 0.0).astype(F32)
    decided = gap_ok | exact_tie
    bad = np.any(got.view(np.uint32) != want.view(np.uint32), 0) & decided & t_ok
    assert not bad.any(), (int(bad.sum()), np.nonzero(bad)[0][:5])
    assert np.array_equal(got[:, ~t_ok], np.zeros((3, int((~t_ok).sum())), F32))
    amb = ~decided & t_ok
    for p in np.nonzero(amb)[0]:                              # one of the two near-equal candidates
        assert any(np.array_equal(got[:, p], ref.reshape(K, 3, hw)[k, :, p]) for k in np.argsort(d[:, p])[:2])
    print(f"[neighbours] K={K} Cf={Cf}: ambiguous pixels {int(amb.sum())} of {hw}, exact ties {int(exact_tie.sum())}")
    assert amb.sum() <= 1e-3 * hw
    if Cf:
        kd = np.where(t_ok, kexp, 0)
        fw = fields.reshape(K, Cf, hw)[kd, :, np.arange(hw)].T
        sel = decided | ~t_ok
        assert_bits_equal(nf.reshape(Cf, hw)[:, sel], np.ascontiguousarray(fw[:, sel]), "neighbour fields")
