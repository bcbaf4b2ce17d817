"""oracle/projection_reference.py without a GPU: its exact float32 arithmetic against rational arithmetic, its pixel and
winner rules against the CPU oracle's Projector and the reference's projection goldens, and its error bound against
float64 evaluations at higher precision."""
from fractions import Fraction
import math

import numpy as np
import pytest
import torch

from oracle import icp_oracle as orc
from oracle import projection_reference as pr

F32 = np.float32


def _exact32(v: Fraction) -> np.float32:
    """The float32 nearest to the rational v (ties to even), by exhaustive neighbour comparison."""
    if abs(v) >= 2 ** 128 - 2 ** 103:                   # IEEE 754: at or past the overflow threshold rounds to inf
        return F32(np.inf) if v > 0 else F32(-np.inf)
    f = F32(float(v))                     # float(Fraction) is correctly rounded to float64: within one float32 step
    best = None
    for c in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - v)
        if best is None or d < best[0] or (d == best[0] and (int(c.view(np.uint32)) & 1) == 0):
            best = (d, c)
    return best[1]


def _fma_exact(a, b, c):
    return _exact32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _range_exact(x, y, z, order):
    a, b = (y, x) if order == pr.Y_FIRST else (x, y)
    aa = _exact32(Fraction(float(a)) ** 2)
    t = _fma_exact(z, z, _fma_exact(b, b, aa))
    # the square root of a float32, rounded: compare the squares of the candidates' midpoints
    s = F32(math.sqrt(float(t)))
    best = min((np.nextafter(s, F32(-np.inf)), s, np.nextafter(s, F32(np.inf))),
               key=lambda c: (abs(Fraction(float(c)) ** 2 - Fraction(float(t))), int(c.view(np.uint32)) & 1))
    return best


def _adversarial_fma(rng, n):
    """(a, b, c) whose product plus c in float64 lands on a float32 midpoint with a non-zero remainder: the case where
    rounding p + c to float64 first and then to float32 goes the wrong way."""
    # a b = 2^m (1 + t)(1 - t) = 2^m - 2^m t^2 with t = k 2^-23: half an ulp of an odd c in [2^(m+24), 2^(m+25)), less a
    # remainder far below float64's ulp there.  In float64 the sum is exactly the midpoint, which ties to the even
    # neighbour; the exact value lies below it and rounds to c.
    out = []
    for _ in range(n):
        m, k, sign = rng.randint(-60, 60), rng.randint(1, 300), rng.choice([-1.0, 1.0])
        a = F32(sign * 2.0 ** m * (1 + k * 2.0 ** -23))
        b = F32(1 - k * 2.0 ** -23)
        c = F32(sign * 2.0 ** (m + 24) * (1 + (2 * rng.randint(0, 2 ** 22) + 1) * 2.0 ** -23))
        out.append((a, b, c))
    return np.array(out, F32)


@pytest.fixture(scope="module")
def fma_cases():
    rng = np.random.RandomState(7)
    rnd = rng.standard_normal((400, 3)).astype(F32) * F32(10.0) ** rng.randint(-8, 9, (400, 3)).astype(F32)
    sub = np.array([[1e-45, 1e-45, 0.0], [1.2e-38, 1.1e-38, -1e-45], [3e-20, 3e-20, 1e-40], [-3e-23, 5e-23, 1e-45],
                    [1.8e19, 1.8e19, 3e38], [1.8e19, 1.9e19, -3.4e38], [3e38, 1.0, 3.3e38], [0.0, -1.0, 0.0]], F32)
    return np.concatenate([rnd, sub, _adversarial_fma(rng, 200)])


def test_fma32_is_correctly_rounded(fma_cases):
    a, b, c = fma_cases.T
    got = pr.fma32(a, b, c)
    # the adversarial rows are the ones where the naive float64 evaluation double-rounds: they must be among the cases
    with np.errstate(over="ignore"):
        naive = (a.astype(np.float64) * b + c).astype(F32)
    assert int((naive != got).sum()) >= 100, "the adversarial cases no longer exercise double rounding"
    for k in range(len(a)):
        want = _fma_exact(a[k], b[k], c[k])
        assert got[k].view(np.uint32) == want.view(np.uint32), (k, a[k], b[k], c[k], got[k], want)


@pytest.mark.parametrize("order", [pr.Y_FIRST, pr.X_FIRST])
def test_range32_is_the_rounded_formula(order):
    rng = np.random.RandomState(3 if order == pr.Y_FIRST else 4)
    p = rng.standard_normal((300, 3)).astype(F32) * F32(10.0) ** rng.randint(-6, 7, (300, 1)).astype(F32)
    p = np.concatenate([p, np.array([[0, 0, 0], [1e-45, 0, 0], [3e-23, 4e-23, 0], [1e19, 1e19, 1e19],
                                     [3, 4, 12], [-0.0, 0.0, -0.0], [1.5e-20, -2.5e-22, 7e-21]], F32)])
    got = pr.range32(p[:, 0], p[:, 1], p[:, 2], order)
    for k in range(len(p)):
        want = _range_exact(*p[k], order)
        assert got[k].view(np.uint32) == want.view(np.uint32), (k, p[k], got[k], want)


def test_range32_orders_differ_where_the_sum_rounds():
    """The two orders are different functions: on random points they disagree in the last ulp for a few percent."""
    rng = np.random.RandomState(11)
    p = (rng.standard_normal((20000, 3)) * 30).astype(F32)
    ry, rx = pr.range32(*p.T, pr.Y_FIRST), pr.range32(*p.T, pr.X_FIRST)
    diff = ry != rx
    assert 0.001 < diff.mean() < 0.5, diff.mean()
    assert np.all(np.abs(ry[diff].view(np.int32) - rx[diff].view(np.int32)) == 1)


def test_transform32_is_the_rounded_formula():
    rng = np.random.RandomState(5)
    T = np.eye(4, dtype=F32)
    T[:3, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0].astype(F32)
    T[:3, 3] = rng.uniform(-20, 20, 3).astype(F32)
    p = (rng.standard_normal((200, 3)) * 40).astype(F32)
    got = pr.transform32(T, p)
    for k in range(len(p)):
        x, y, z = (Fraction(float(v)) for v in p[k])
        for c in range(3):
            t0 = _exact32(y * Fraction(float(T[c, 1])))
            t1 = _fma_exact(p[k, 0], T[c, 0], t0)
            t2 = _fma_exact(p[k, 2], T[c, 2], t1)
            want = _exact32(Fraction(float(t2)) + Fraction(float(T[c, 3])))
            assert got[k, c].view(np.uint32) == want.view(np.uint32), (k, c)
    # the identity moves nothing
    assert np.array_equal(pr.transform32(np.eye(4, dtype=F32), p), p)


def test_round32_breaks_midpoints_by_the_remainder():
    one = 1.0
    half_ulp = 2.0 ** -24                                  # midpoint between 1 and 1 + 2^-23
    assert pr.round32(one + half_ulp, 0.0) == F32(1.0)     # exact tie: to even
    assert pr.round32(one + half_ulp, 1e-30) == np.nextafter(F32(1), F32(2))
    assert pr.round32(one + 3 * half_ulp, -1e-30) == np.nextafter(F32(1), F32(2))
    assert pr.round32(2.0 ** 128 - 2.0 ** 103, -1e-300) == np.finfo(F32).max
    assert np.isinf(pr.round32(2.0 ** 128 - 2.0 ** 103, 0.0))


def test_pixel_rule_half_to_even_bounds_and_range():
    H, W = 4, 6
    row = np.array([-0.5, -0.0, 0.5, 1.5, 2.5, 3.5, 3.49999976, 0.0, 0.0, 0.0, np.nan, 1.0, 1.0], F32)
    col = np.array([0.0, 0.0, 5.5, 4.5, -0.5, 0.0, 5.49999952, 6.5, -0.50000006, 0.0, 0.0, np.inf, 1.0], F32)
    r = np.array([1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, np.nan], F32)
    pix = pr.pixel_rule(row, col, r, H, W)
    assert pix.tolist() == [0, 0, -1, 2 * W + 4, 2 * W + 0, -1, 3 * W + 5, -1, -1, -1, -1, -1, -1]


def test_expected_winners_closest_then_lowest_index():
    pix = np.array([3, 3, 3, 0, -1, 0, 5, 5], np.int64)
    r = np.array([2.0, 1.0, 1.0, 0.5, 0.1, 0.5, np.inf, 7.0], F32)
    w = pr.expected_winners(pix, r, 2, 4)
    assert w.tolist() == [3, -1, -1, 1, -1, 7, -1, -1]
    w64 = pr.expected_winners(pix, r.astype(np.float64), 2, 4)
    assert np.array_equal(w, w64)


def _oracle_pixels(H, W, pts):
    row, col = orc.Projector(H, W).pixels(torch.from_numpy(pts)[None])
    return row[0].numpy(), col[0].numpy(), torch.from_numpy(pts).norm(dim=1).numpy()


def _vmap_of(winners, values, H, W):
    out = np.zeros((values.shape[1], H * W), values.dtype)
    ok = winners >= 0
    out[:, ok] = values[winners[ok]].T
    return out.reshape(-1, H, W)


def test_rules_rebuild_the_oracle_projection(golden_helpers):
    """pixel_rule + expected_winners on the oracle's own coordinates and ranges are the oracle's build_projection_map."""
    from pylidar_slam_b200 import synthetic as syn
    for H, W, pts in ((16, 256, golden_helpers["a3_points"]), (64, 1024, syn.scan(3, 64, 1024)), (33, 500, syn.scan(1, 33, 500))):
        pts = np.ascontiguousarray(pts, F32)
        pts = np.concatenate([pts, pts[::7]])   # duplicates: exact range ties at higher indices
        row, col, r = _oracle_pixels(H, W, pts)
        win = pr.expected_winners(pr.pixel_rule(row, col, r, H, W), r, H, W)
        ref = orc.Projector(H, W).build_projection_map(torch.from_numpy(pts)[None])[0].numpy()
        np.testing.assert_array_equal(_vmap_of(win, pts, H, W), ref)
        assert (win >= 0).sum() > H * W // 4


def test_rules_rebuild_the_golden_projection(golden_helpers, golden_misc):
    """On the reference's own float32 pixel coordinates, the rules reproduce its vertex map."""
    g = golden_helpers
    pts, pix = g["a3_points"], g["a3_pixels"]
    H, W = g["a3_vmap"].shape[1:]
    r = torch.from_numpy(pts).norm(dim=1).numpy()
    win = pr.expected_winners(pr.pixel_rule(pix[:, 0], pix[:, 1], r, H, W), r, H, W)
    np.testing.assert_array_equal(_vmap_of(win, pts, H, W), g["a3_vmap"])
    m = golden_misc
    cloud = m["proj_cloud"]
    H, W = m["proj_map"].shape[1:]
    row, col, r = _oracle_pixels(H, W, np.ascontiguousarray(cloud[:, :3]))
    win = pr.expected_winners(pr.pixel_rule(row, col, r, H, W), r, H, W)
    want = _vmap_of(win, cloud[:, :3], H, W)
    want[:, win.reshape(H, W) < 0] = m["proj_default"]
    np.testing.assert_array_equal(want, m["proj_map"])


def test_pixels64_is_the_oracle_formula_in_float64():
    from pylidar_slam_b200 import synthetic as syn
    pts = syn.scan(2, 64, 1024).astype(np.float64)
    pts = pts[np.isfinite(pts).all(1)]
    row, col, r = pr.pixels64(pts, 64, 1024, f32_consts=False)
    orow, ocol = orc.Projector(64, 1024).pixels(torch.from_numpy(pts)[None])
    np.testing.assert_allclose(row, orow[0].numpy(), rtol=0, atol=1e-9)
    np.testing.assert_allclose(col, ocol[0].numpy(), rtol=0, atol=1e-9)


def test_row_col_bound_covers_the_float32_oracle():
    """The bound covers torch's float32 evaluation of the same formula (whose atan2 / asin are at least as accurate as
    the device's on x86), and is tight: a few ulp of the coordinate, far below a pixel."""
    from pylidar_slam_b200 import synthetic as syn
    H, W = 64, 2048
    pts = syn.scan(5, H, W)
    pts = pts[np.isfinite(pts).all(1) & (np.abs(pts).sum(1) > 0)]
    row, col, _ = pr.pixels64(pts, H, W)
    drow, dcol = pr.row_col_bound(pts, H, W)
    orow, ocol = orc.Projector(H, W).pixels(torch.from_numpy(np.ascontiguousarray(pts, F32))[None])
    assert np.all(np.abs(orow[0].numpy() - row) <= drow)
    assert np.all(np.abs(ocol[0].numpy() - col) <= dcol)
    assert np.percentile(drow, 99) < 1e-3 and np.percentile(dcol, 99) < 2e-3
    # float64: the same analysis at u = 2^-53
    drow64, dcol64 = pr.row_col_bound(pts, H, W, f32=False)
    assert np.all(drow64 < drow * 1e-8) and np.all(dcol64 < dcol * 1e-8)
    # the null point is exact, a non-finite one unbounded
    d0 = pr.row_col_bound(np.array([[0, 0, 0], [np.inf, 0, 0], [1, np.nan, 0]]), H, W)
    assert d0[0].tolist()[0] == 0 and np.isinf(d0[0][1:]).all() and np.isinf(d0[1][1:]).all()
