"""Test infrastructure only: exact and bounded host models of the spherical projection's z-buffers.

Nothing here runs in the library.  tests/test_projection_pixels_gpu.py uses it to say, per pixel, which point every
z-buffer of projection_device.cuh must keep, and tests/test_projection_reference_cpu.py pins it without a GPU.

What is exact and what is not
-----------------------------
* The range and the pose transform are explicitly rounded float32 formulas (projection_device.cuh: range_rn,
  transform_point), so `range32` and `transform32` reproduce them bit for bit.  A float32 product is exact in float64
  (24 + 24 bits < 53), and a float32 sum, product or square root evaluated in float64 and rounded once to float32 is
  correctly rounded (53 >= 2 * 24 + 2).  A float32 fma is not: p + c in float64 can round onto a float32 midpoint and
  then round again.  `fma32` evaluates p + c with TwoSum, s + e == p + c exactly, and breaks a midpoint s by the sign
  of e, so every fma is rounded once, correctly.
* atan2f and asinf are not correctly rounded on the device, so the host cannot reproduce a pixel coordinate.  The exact
  layer takes the float32 row and column the GPU computed (pls_project_pixels runs the inlined project_point of every
  z-buffer) and applies `pixel_rule` -- rint half-to-even, the four bounds, r > 0 -- and `expected_winners` -- closest
  first, the lowest index on an exact range tie -- to them.  Both are exact.
* `pixels64` evaluates the same formula in float64; `row_col_bound` bounds how far the device's float32 (or float64)
  row and column can lie from the exact real value of that formula.  That is the only tolerance here.

Derivation of `row_col_bound`
-----------------------------
u is the unit roundoff (2^-24 for float32, 2^-53 for float64); a correctly rounded operation (.rn) errs by at most
u |result|, and ulp(v) <= 2 u |v|.  The CUDA Math API appendix gives atan2f 3 ulp and asinf 2 ulp (float32), atan2
and asin 2 ulp (float64).  The inputs x, y, z are exact, the constants (pi, W, H, |fov_down|, fov) are the ones the
kernel uses, so only the kernel's own roundings enter.  With every partial error propagated to first order:

    r      = sqrt(fma(z, z, fma(b, b, a a)))   three roundings of a sum of non-negative terms (relative 3u), the
                                               square root halves it and adds its own: |dr| <= 2.5 u r
    q      = z / r                             |dq| <= |q| (2.5 u + u)
    phi    = asin(q)                           |dphi| <= |dq| / sqrt(1 - (|q| + |dq|)^2) + A_asin 2u |phi|
    s1     = phi + |fov_down|                  |ds1| <= |dphi| + u |s1|
    s2     = s1 / fov                          |ds2| <= |ds1| / fov + u |s2|
    s3     = 1 - s2                            |ds3| <= |ds2| + u |s3|
    row    = s3 H                              |drow| <= H |ds3| + u |row|
    theta  = -atan2(y, x)                      |dtheta| <= A_atan2 2u |theta|
    t      = theta / pi                        |dt| <= |dtheta| / pi + u |t|
    a      = t + 1                             |da| <= |dt| + u |a|
    col    = (0.5 a) W                         |dcol| <= 0.5 W |da| + u |col|      (0.5 a is exact)

The bound multiplies the first-order sum by 1 + 2^-10, which covers the products of error terms (each O(u^2)).  A
point whose |q| + |dq| reaches 1 gets an infinite row bound: its row is not bounded by this analysis.

The bound covers the device's error, not that of `pixels64` itself.  Against a float32 kernel the host's float64 error
(about 2^-29 of the bound) is absorbed by the 2^-10 slack.  Against a float64 kernel it is not: `pixels64` performs the
same operations in float64, with numpy's arctan2 and arcsin, which are within the same 2 ulp, so it errs by up to the
same bound, and a float64 point is decided only beyond twice the bound from a rounding boundary.
"""
from fractions import Fraction
import math

import numpy as np

F32, F64 = np.float32, np.float64
U32, U64 = 2.0 ** -24, 2.0 ** -53
Y_FIRST, X_FIRST = "y_first", "x_first"   # RangeOrder::kYFirst, RangeOrder::kXFirst
PI32 = float(np.float32(np.pi))           # project_point's kPi


# ------------------------------------------------------------------------------------------------ exact float32 ops
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def round32(s, e):
    """The float32 nearest to the exact value s + e (s, e float64, |e| <= ulp(s) / 2, as TwoSum gives them)."""
    s, e = np.asarray(s, F64), np.asarray(e, F64)
    with np.errstate(over="ignore", invalid="ignore"):
        r = s.astype(F32)
        rd = r.astype(F64)
        rd = np.where(np.isinf(r) & np.isfinite(s), np.copysign(2.0 ** 128, s), rd)  # the overflow threshold's upper end
        d = s - rd
        other = np.nextafter(r, np.where(d > 0, np.inf, -np.inf).astype(F32)).astype(F32)
        mid = (rd + other.astype(F64)) * 0.5
        tie = np.isfinite(s) & (d != 0) & (s == mid) & (e != 0)
        toward = tie & (np.sign(e) == np.sign(d))   # the exact value lies past the midpoint, on the other's side
    return np.where(toward, other, r).astype(F32)


def mul32(a, b):
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)).astype(F32)   # exact product, one rounding


def add32(a, b):
    return (np.asarray(a, F32).astype(F64) + np.asarray(b, F32).astype(F64)).astype(F32)


def fma32(a, b, c):
    """fmaf(a, b, c), correctly rounded."""
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)
        s, e = _two_sum(p, np.asarray(c, F32).astype(F64))
    return round32(s, np.where(np.isfinite(e), e, 0.0))


def sqrt32(a):
    with np.errstate(invalid="ignore"):
        return np.sqrt(np.asarray(a, F32).astype(F64)).astype(F32)


def range32(x, y, z, order=Y_FIRST):
    """range_rn in float32: sqrt_rn(fma_rn(z, z, fma_rn(b, b, mul_rn(a, a)))), (a, b) = (y, x) for kYFirst."""
    x, y, z = (np.asarray(v, F32) for v in (x, y, z))
    a, b = (y, x) if order == Y_FIRST else (x, y)
    return sqrt32(fma32(z, z, fma32(b, b, mul32(a, a))))


def transform32(T, p):
    """transform_point: row c of the row-major pose T rounded as add(fma(z, T2, fma(x, T0, y T1)), T3).  p [n,3]."""
    T = np.asarray(T, F32).reshape(-1)[:12]
    p = np.asarray(p, F32).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    out = np.empty_like(p)
    for c in range(3):
        out[:, c] = add32(fma32(z, T[4 * c + 2], fma32(x, T[4 * c], mul32(y, T[4 * c + 1]))), T[4 * c + 3])
    return out


# ---------------------------------------------------------------------------------------- exact float64 range (slow)
def range64_exact(x, y, z):
    """range_rn in float64 for one point, every fma correctly rounded (Fraction -> float is correctly rounded)."""
    x, y, z = float(x), float(y), float(z)
    if not all(math.isfinite(v) for v in (x, y, z)):
        return math.sqrt(z * z + x * x + y * y) if not any(math.isnan(v) for v in (x, y, z)) else math.nan
    t = float(Fraction(x) * Fraction(x) + Fraction(y * y))
    return math.sqrt(float(Fraction(z) * Fraction(z) + Fraction(t)))


# ------------------------------------------------------------------------------------------------- pixels, winners
def proj_consts(H, W, up=3.0, down=-24.0, f32=True):
    """(kPi, Hf, Wf, abs_down, fov) as the kernel holds them: make_proj_const (float32) or ProjConst64."""
    d = abs(float(down) / 180.0 * 3.141592653589793)
    u = abs(float(up) / 180.0 * 3.141592653589793)
    if f32:
        return PI32, float(F32(H)), float(F32(W)), float(F32(d)), float(F32(d + u))
    return 3.141592653589793, float(H), float(W), d, d + u


def pixel_rule(row, col, r, H, W):
    """project_to_pixel's rule on given coordinates: rint half-to-even, 0 <= row <= H-1, 0 <= col <= W-1, r > 0.
    Returns the flat pixel (row * W + col), -1 where the point is dropped."""
    row, col, r = np.asarray(row), np.asarray(col), np.asarray(r)
    with np.errstate(invalid="ignore"):
        pr, pc = np.rint(row), np.rint(col)
        ok = (pr >= 0) & (pr <= H - 1) & (pc >= 0) & (pc <= W - 1) & (r > 0)
    pix = np.full(row.shape, -1, np.int64)
    pix[ok] = pr[ok].astype(np.int64) * W + pc[ok].astype(np.int64)
    return pix


def expected_winners(pix, key_r, H, W):
    """The z-buffer's winner of every pixel: the smallest key_r (float32 or float64), the lowest index on an exact tie.
    pix [n] from pixel_rule; returns [H*W] point indices, -1 for an empty pixel."""
    pix, key_r = np.asarray(pix), np.asarray(key_r)
    win = np.full(H * W, -1, np.int64)
    sel = np.nonzero(pix >= 0)[0]
    if sel.size == 0:
        return win
    order = sel[np.lexsort((sel, key_r[sel], pix[sel]))]
    p = pix[order]
    first = np.ones(order.size, bool)
    first[1:] = p[1:] != p[:-1]
    win[p[first]] = order[first]
    return win


def pixels64(p, H, W, up=3.0, down=-24.0, f32_consts=True):
    """Row, column and range of every point of p [n,3], the projection formula evaluated in float64 with the kernel's
    constants (float32 ones for the float32 kernels).  The null point gives (-1, -1), like project_point."""
    p = np.asarray(p, F64).reshape(-1, 3)
    kpi, Hf, Wf, ad, fov = proj_consts(H, W, up, down, f32_consts)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        r = np.sqrt(z * z + x * x + y * y)
        null = r == 0
        rr = np.where(null, 0.001, r)
        theta = -np.arctan2(y, x)
        phi = np.arcsin(z / rr)
        col = 0.5 * (theta / kpi + 1.0) * Wf
        row = (1.0 - (phi + ad) / fov) * Hf
    return np.where(null, -1.0, row), np.where(null, -1.0, col), r


def row_col_bound(p, H, W, up=3.0, down=-24.0, f32=True):
    """Worst-case |device - exact| of project_point's row and column (float32 kernels) or of project_to_pixel_f64's
    (f32=False), from the documented maximum errors; derivation in the module docstring.  inf where not bounded."""
    p = np.asarray(p, F64).reshape(-1, 3)
    u = U32 if f32 else U64
    a_atan2, a_asin = (3.0, 2.0) if f32 else (2.0, 2.0)
    kpi, Hf, Wf, ad, fov = proj_consts(H, W, up, down, f32)
    row, col, r = pixels64(p, H, W, up, down, f32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = z / np.where(r == 0, 0.001, r)
        dq = np.abs(q) * 3.5 * u
        reach = np.abs(q) + dq
        deriv = np.where(reach < 1.0, 1.0 / np.sqrt(1.0 - np.minimum(reach, 1.0) ** 2), np.inf)
        phi = np.arcsin(q)
        dphi = dq * deriv + a_asin * 2 * u * np.abs(phi)
        s1 = phi + ad
        ds1 = dphi + u * np.abs(s1)
        s2 = s1 / fov
        ds2 = ds1 / fov + u * np.abs(s2)
        s3 = 1.0 - s2
        ds3 = ds2 + u * np.abs(s3)
        drow = Hf * ds3 + u * np.abs(row)
        theta = -np.arctan2(y, x)
        dth = a_atan2 * 2 * u * np.abs(theta)
        t = theta / kpi
        dt = dth / kpi + u * np.abs(t)
        a = t + 1.0
        da = dt + u * np.abs(a)
        dcol = 0.5 * Wf * da + u * np.abs(col)
    slack = 1.0 + 2.0 ** -10
    finite = np.isfinite(p).all(axis=1)
    null = r == 0
    drow = np.where(null, 0.0, np.where(finite, drow * slack, np.inf))
    dcol = np.where(null, 0.0, np.where(finite, dcol * slack, np.inf))
    return drow, dcol


def near_half(v, bound):
    """True where v lies within bound of a rounding boundary k + 0.5 (or is not finite)."""
    v = np.asarray(v, F64)
    with np.errstate(invalid="ignore"):
        return ~np.isfinite(v) | ~np.isfinite(bound) | (np.abs(v - np.floor(v) - 0.5) <= bound)


def pixels_within(row, col, drow, dcol, H, W):
    """Every pixel (flat, -1 for dropped) a point may take when its row and column may be off by drow, dcol; [n, 4]."""
    out = np.full((np.size(row), 4), -1, np.int64)
    k = 0
    for sr in (-1, 1):
        for sc in (-1, 1):
            with np.errstate(invalid="ignore"):
                out[:, k] = pixel_rule(row + sr * drow, col + sc * dcol, np.ones_like(row), H, W)
            k += 1
    return out
