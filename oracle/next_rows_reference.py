"""TEST INFRASTRUCTURE ONLY -- float64 references of the kernels beside the odometry hot path: the training loss
(training.cu), the a4 normal map (projmap.cu normal_map_kernel), the stand-alone Gauss-Newton alignments (gn.cu) and the
weighted Procrustes registration (registration.cu).  numpy only; the product path never imports it.

  * p2plane_loss_f64      the unsupervised point-to-plane loss and its gradients, per batch element, with the pixel,
                          the z-buffer winner and an `ambiguous` flag for every target point, and first-order bounds of
                          what float32 rounding of the transform can move;
  * normal_map_f32_emulated  a bit-exact numpy emulation of normal_map_kernel's documented float32 operation order;
  * gn_sums_f64 / gn_step_f64 / gn_align_f64  the 30 normal-equation accumulators, one solve, the iteration loop;
    gn_f32_step_bound    what float32 evaluation of the per-correspondence terms can move one step by;
  * procrustes_f64        LAPACK's SVD with the reference's sign rule.

Semantics follow the header comments of the CUDA files (themselves restating slam/training/loss_modules.py,
slam/common/geometry.py, slam/common/optimization.py and slam/common/registration.py of the reference).
"""
from fractions import Fraction

import numpy as np

U = 2.0 ** -24  # float32 unit roundoff
NACC = 30
SCHEMES = {"default": 0, "least_square": 1, "huber": 2, "exp": 3, "neighborhood": 4, "geman_mcclure": 5,
           "square_geman_mcclure": 6, "cauchy": 7}
PIX_BAND = 2e-3     # px: a row / column this close to a .5 boundary may round either way on the GPU
RANGE_BAND = 4e-6   # relative: two ranges this close in one pixel may swap their z-buffer order


# ----------------------------------------------------------------------------------------------- pose algebra
def euler_to_mat(e):
    cx, sx, cy, sy, cz, sz = np.cos(e[0]), np.sin(e[0]), np.cos(e[1]), np.sin(e[1]), np.cos(e[2]), np.sin(e[2])
    return np.array([[cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx],
                     [sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx],
                     [-sy, cy * sx, cy * cx]])


def build_pose(x):
    """(tx, ty, tz, ex, ey, ez) -> 4x4, R = Rz Ry Rx (pose_device.cuh build_pose), float64."""
    x = np.asarray(x, np.float64)
    T = np.eye(4)
    T[:3, :3] = euler_to_mat(x[3:])
    T[:3, 3] = x[:3]
    return T


def euler_jacobian(e):
    """dR/de_k, k = x, y, z: [3,3,3] (pose_device.cuh euler_jacobian), float64."""
    cx, sx, cy, sy, cz, sz = np.cos(e[0]), np.sin(e[0]), np.cos(e[1]), np.sin(e[1]), np.cos(e[2]), np.sin(e[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Jx = np.array([[0, 0, 0], [0, -sx, -cx], [0, cx, -sx]])
    Jy = np.array([[-sy, 0, cy], [0, 0, 0], [-cy, 0, -sy]])
    Jz = np.array([[-sz, -cz, 0], [cz, -sz, 0], [0, 0, 0]])
    return np.stack([Rz @ Ry @ Jx, Rz @ Jy @ Rx, Jz @ Ry @ Rx])


# ----------------------------------------------------------------------------------------------- training loss
def proj_consts(H, W, up_deg, down_deg):
    """ProjConst of projection_device.cuh: the float32 scalars the kernel projects with, as float64 values."""
    up = float(np.float32(up_deg)) / 180.0 * np.pi
    down = float(np.float32(down_deg)) / 180.0 * np.pi
    return dict(H=H, W=W, abs_down=float(np.float32(abs(down))), fov=float(np.float32(abs(down) + abs(up))),
                pi=float(np.float32(np.pi)))


def pixel_coords_f64(pm, pc):
    """Float row / column / range of points pm [N,3] (float64), the kernel's formula evaluated in float64."""
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.sqrt((pm * pm).sum(1))
        rr = np.where(r == 0.0, 0.001, r)
        theta = -np.arctan2(pm[:, 1], pm[:, 0])
        phi = np.arcsin(pm[:, 2] / rr)
        col = 0.5 * (theta / pc["pi"] + 1.0) * pc["W"]
        row = (1.0 - (phi + pc["abs_down"]) / pc["fov"]) * pc["H"]
    return row, col, r


def loss_cost(scheme, sigma, a, d2):
    """C(a), dC/da, dC/d(d2) of training_device.cuh loss_cost (a = |r|, d2 = |p' - q|^2), vectorised float64."""
    s = SCHEMES[scheme] if isinstance(scheme, str) else scheme
    z = np.zeros_like(a)
    with np.errstate(over="ignore", invalid="ignore"):
        if s in (0, 1):
            return a * a, 2 * a, z
        if s == 2:
            q = a < sigma
            return np.where(q, a * a, 2 * sigma * a - sigma * sigma), np.where(q, 2 * a, 2 * sigma), z
        if s == 3:
            e = np.exp(-a * a / (sigma * sigma))
            return a * a * e, 2 * a * e * (1 - a * a / (sigma * sigma)), z
        if s == 4:
            w = np.exp(-d2 / (sigma * sigma))
            return a * a * w, 2 * a * w, -a * a * w / (sigma * sigma)
        if s == 5:
            t = sigma + a * a
            return sigma * a * a / t, 2 * sigma * sigma * a / (t * t), z
        if s == 6:
            t = sigma + a * a
            return a * a * (sigma / t) * (sigma / t), 2 * a * sigma * sigma * (sigma - a * a) / (t * t * t), z
        return np.log(1 + a * a / (sigma * sigma)), 2 * a / (sigma * sigma + a * a), z


def loss_pixel_terms(scheme, sigma, pw, q, n):
    """training_device.cuh loss_pixel_terms over rows: mask, C^2 and g = d(C^2)/d(pw) (float64)."""
    ok = (n != 0).any(1) & (q != 0).any(1) & (pw != 0).any(1)
    d = q - pw
    r = (d * n).sum(1)
    C, dCa, dCd2 = loss_cost(scheme, sigma, np.abs(r), (d * d).sum(1))
    ka = 2.0 * C * dCa * np.sign(r)
    kd = 2.0 * C * dCd2 * 2.0
    g = -ka[:, None] * n - kd[:, None] * d
    return ok.astype(np.float64), np.where(ok, C * C, 0.0), np.where(ok[:, None], g, 0.0)


def p2plane_loss_f64(vt, vr, nr, mats, H, W, up, down, scheme, sigma, params=None, transform_ulps=4.0):
    """The training loss of training.cu in float64.

    vt / vr / nr: [B,3,H,W] float32 target vertex, reference vertex and reference normal maps; mats [B,4,4] the pose
    matrices (float64 values; pass the float32 matrices, or build_pose(params) for the parameter path); params [B,6]
    adds the parameter gradient.  Every target point p moves to p' = R p + t (float64); its pixel is rint of the float64
    row / column; the closest p' of a pixel wins, an exact range tie goes to the lower point index; the winner books
    C^2 and the mask; every point that landed in a pixel receives that pixel's g (index_put's backward).

    A point is `ambiguous` when its row or column lies within PIX_BAND + 8u H (or W) px of a .5 boundary, or its range lies within
    RANGE_BAND relative of another point of its pixel without being equal to it: float32 atan2f / asinf / sqrtf and a
    possibly contracted transform may decide those differently.

    Bounds: the kernel transforms in float32, so every p' carries an error of at most
    delta = transform_ulps * u * (|R||p| + |t|) per coordinate.  loss_bound = sum_pix |g| . delta / M;
    grad bounds use the change of g over +-delta along each axis (central differences of the pixel terms).  Summation
    order and the float32 outputs are the caller's to add.
    Returns a dict of [B, ...] arrays: loss_per_batch, grad_mats [B,4,4], grad_params [B,6] (or None), pixel,
    winner, landed, ambiguous [B,HW], loss_bound, grad_mats_bound, grad_params_bound, and loss = mean of the batch."""
    vt = np.asarray(vt, np.float32)
    B = vt.shape[0]
    HW = H * W
    pc = proj_consts(H, W, up, down)
    sigma = float(np.float32(sigma))
    out = {k: [] for k in ("loss_per_batch", "grad_mats", "grad_params", "pixel", "winner", "landed", "ambiguous",
                           "loss_bound", "grad_mats_bound", "grad_params_bound")}
    mats = np.asarray(mats, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):  # an element without a valid pixel has M = 0, as in the kernel
        for b in range(B):
            _loss_element(b, B, H, W, vt, vr, nr, mats, pc, scheme, sigma, params, transform_ulps, out)
    res = {k: (np.stack(v) if v[0] is not None else None) for k, v in out.items()}
    res["loss"] = float(res["loss_per_batch"].mean())
    return res


def _loss_element(b, B, H, W, vt, vr, nr, mats, pc, scheme, sigma, params, transform_ulps, out):
    HW = H * W
    R, t = mats[b, :3, :3], mats[b, :3, 3]
    P = vt[b].reshape(3, HW).T.astype(np.float64)
    alive = (P != 0).any(1)
    with np.errstate(invalid="ignore"):
        pm = P @ R.T + t
    finite = np.isfinite(pm).all(1)
    row, col, rng_ = pixel_coords_f64(np.where(finite[:, None], pm, 0.0), pc)
    prow, pcol = np.rint(row), np.rint(col)
    landed = alive & finite & (prow >= 0) & (prow <= H - 1) & (pcol >= 0) & (pcol <= W - 1) & (rng_ > 0)
    pix = np.where(landed, prow * W + pcol, -1).astype(np.int64)
    # float32 rows / columns carry a few ulps of H / W on top of the band (1/64 px at W = 135 169)
    near = lambda v, m: np.abs(v - np.floor(v) - 0.5) < PIX_BAND + 8 * U * m  # noqa: E731
    reach = (row > -0.5 - 0.01) & (row < H - 0.5 + 0.01) & (col > -0.5 - 0.01) & (col < W - 0.5 + 0.01)
    amb = alive & finite & reach & (near(row, H) | near(col, W))
    idx = np.nonzero(landed)[0]
    order = idx[np.lexsort((idx, rng_[idx], pix[idx]))]
    ps = pix[order]
    head = np.ones(len(order), bool)
    head[1:] = ps[1:] != ps[:-1]
    rs = rng_[order]
    same = ~head[1:]
    dr = rs[1:] - rs[:-1]
    close = same & (dr > 0) & (dr <= RANGE_BAND * rs[1:])
    amb[order[1:][close]] = True
    amb[order[:-1][close]] = True
    winner = np.full(HW, -1, np.int64)
    winner[ps[head]] = order[head]
    wpix = np.nonzero(winner >= 0)[0]
    q = vr[b].reshape(3, HW).T.astype(np.float64)
    n = nr[b].reshape(3, HW).T.astype(np.float64)
    pw = np.zeros((HW, 3))
    pw[wpix] = pm[winner[wpix]]
    mask, c2, g = loss_pixel_terms(scheme, sigma, pw, q, n)
    M = mask.sum()
    lb = c2.sum() / M
    sc = 1.0 / (M * B)
    gl = g[pix[landed]]
    Pl = P[landed]
    G = np.zeros((4, 4))
    G[:3, :3] = gl.T @ Pl * sc
    G[:3, 3] = gl.sum(0) * sc
    # bounds: delta per point, the pixel's terms moved by +-delta of its winner along each axis
    delta = transform_ulps * U * (np.abs(P) @ np.abs(R).T + np.abs(t))
    dw = np.zeros((HW, 3))
    dw[wpix] = delta[winner[wpix]]
    dg = np.zeros((HW, 3))
    for k in range(3):
        e = np.zeros((HW, 3))
        e[:, k] = dw[:, k]
        _, _, gp = loss_pixel_terms(scheme, sigma, pw + e, q, n)
        _, _, gm = loss_pixel_terms(scheme, sigma, pw - e, q, n)
        dg += np.abs(gp - gm)  # covers |dg/dp'_k| delta_k on both sides, kinks included
    loss_bound = (np.abs(g) * dw).sum() / M
    dgl = dg[pix[landed]]
    Gb = np.zeros((4, 4))
    Gb[:3, :3] = dgl.T @ np.abs(Pl) * sc + 1e-12 * (np.abs(gl).T @ np.abs(Pl)) * sc
    Gb[:3, 3] = dgl.sum(0) * sc + 1e-12 * np.abs(gl).sum(0) * sc
    gp_, gpb = None, None
    if params is not None:
        dR = euler_jacobian(np.asarray(params[b], np.float64)[3:])
        gp_ = np.concatenate([G[:3, 3], [(G[:3, :3] * dR[k]).sum() for k in range(3)]])
        # the kernel evaluates dR in float32: a few ulp of |dR| on top of the propagated matrix bound
        gpb = np.concatenate([Gb[:3, 3], [(Gb[:3, :3] * np.abs(dR[k])).sum() + 8 * U * (np.abs(G[:3, :3]) * np.abs(dR[k])).sum()
                                          for k in range(3)]])
    for k, v in (("loss_per_batch", lb), ("grad_mats", G), ("grad_params", gp_), ("pixel", pix), ("winner", winner),
                 ("landed", landed), ("ambiguous", amb), ("loss_bound", loss_bound), ("grad_mats_bound", Gb),
                 ("grad_params_bound", gpb)):
        out[k].append(v)


# ----------------------------------------------------------------------------------------------- normal map
def _is_f32_midpoint(s):
    """True where the float64 value s lies exactly halfway between two adjacent float32 values."""
    r = s.astype(np.float32)
    other = np.nextafter(r, np.where(s > r.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    with np.errstate(invalid="ignore", over="ignore"):
        return (r.astype(np.float64) != s) & ((r.astype(np.float64) + other.astype(np.float64)) * 0.5 == s)


def _round_fraction_to_f32(x):
    """Correctly rounded (ties to even) float32 of an exact rational."""
    f = np.float32(float(x))
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.uint32)) & 1))
    return np.float32(best)


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c) of float32 arrays: the float64 product is exact (24 + 24 bits); the sum
    is redone with Fraction where the float64 sum is inexact AND lands on a float32 rounding midpoint (the only case
    where rounding twice differs from rounding once)."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)  # two-sum: exact error of the float64 addition
    out = s.astype(np.float32)
    bad = (err != 0) & _is_f32_midpoint(s)
    for i in zip(*np.nonzero(bad)):
        out[i] = _round_fraction_to_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
    return out


def normal_map_f32_emulated(vm, ksize, return_det=False):
    """normal_map_kernel bit for bit: vm [B,3,H,W] float32 -> [B,3,H,W] float32.
      zero-padded k x k window; box sums as sequential float32 adds, rows outer / columns inner, of separately rounded
      products; cofactor rows fma(a1, b2, -(a2 * b1)); det = ((d0 + d1) + d2) / 3 with |det| > 1e-6f; n_i =
      ((c0_i / det) sx + (c1_i / det) sy) + (c2_i / det) sz; norm = sqrt(fma(n2, n2, fma(n1, n1, n0 * n0))), 0 -> 1;
      a null centre vertex gives a null normal."""
    vm = np.asarray(vm, np.float32)
    assert ksize % 2 == 1 and 1 <= ksize <= 9
    B, _, H, W = vm.shape
    r = ksize // 2
    f = np.float32
    pad = np.zeros((B, 3, H + 2 * r, W + 2 * r), f)
    pad[:, :, r:r + H, r:r + W] = vm
    S = {k: np.zeros((B, H, W), f) for k in ("x", "y", "z", "xx", "xy", "xz", "yy", "yz", "zz")}
    for dy in range(ksize):
        for dx in range(ksize):
            px, py, pz = (pad[:, c, dy:dy + H, dx:dx + W] for c in range(3))
            S["x"] = S["x"] + px
            S["y"] = S["y"] + py
            S["z"] = S["z"] + pz
            S["xx"] = S["xx"] + px * px
            S["xy"] = S["xy"] + px * py
            S["xz"] = S["xz"] + px * pz
            S["yy"] = S["yy"] + py * py
            S["yz"] = S["yz"] + py * pz
            S["zz"] = S["zz"] + pz * pz
    A0, A1, A2 = (S["xx"], S["xy"], S["xz"]), (S["xy"], S["yy"], S["yz"]), (S["xz"], S["yz"], S["zz"])

    def cross(a, b):
        return (fma32(a[1], b[2], -(a[2] * b[1])), fma32(a[2], b[0], -(a[0] * b[2])), fma32(a[0], b[1], -(a[1] * b[0])))

    def dot3(a0, b0, a1, b1, a2, b2):
        return (a0 * b0 + a1 * b1) + a2 * b2

    c0, c1, c2 = cross(A1, A2), cross(A2, A0), cross(A0, A1)
    d0 = dot3(c0[0], A0[0], c0[1], A0[1], c0[2], A0[2])
    d1 = dot3(c1[0], A1[0], c1[1], A1[1], c1[2], A1[2])
    d2 = dot3(c2[0], A2[0], c2[1], A2[1], c2[2], A2[2])
    det = ((d0 + d1) + d2) / f(3.0)
    ok = np.abs(det) > f(1e-6)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        dd = np.where(ok, det, f(1.0))
        n = [dot3(c0[i] / dd, S["x"], c1[i] / dd, S["y"], c2[i] / dd, S["z"]) for i in range(3)]
        nn = np.sqrt(fma32(n[2], n[2], fma32(n[1], n[1], n[0] * n[0])))
        nn = np.where(nn == 0, f(1.0), nn)
        n = [np.where(ok, v / nn, f(0.0)) for v in n]
    null = (vm == 0).all(1)
    out = np.stack([np.where(null, f(0.0), v) for v in n], 1).astype(f)
    return (out, det) if return_det else out


# ----------------------------------------------------------------------------------------------- Gauss-Newton
def ls_weight(scheme, sigma, r, d=None):
    """gn_device.cuh ls_weight in float64: sqrt(cost(r)) / max(|r|, 1e-4); d = |p' - q| for the neighbourhood scheme."""
    s = SCHEMES[scheme] if isinstance(scheme, str) else scheme
    a = np.abs(r)
    if s in (0, 1):
        return np.ones_like(r)
    with np.errstate(over="ignore", under="ignore"):
        if s == 2:
            cost = np.where(a < sigma, r * r, 2 * sigma * a - sigma * sigma)
        elif s == 3:
            cost = r * r * np.exp(-(r * r) / (sigma * sigma))
        elif s == 4:
            cost = r * r * np.exp(-(d * d) / (sigma * sigma))
        elif s == 5:
            cost = sigma * r * r / (sigma + r * r)
        elif s == 6:
            cost = r * r * (sigma / (sigma + r * r)) ** 2
        else:
            cost = np.log1p((r / sigma) ** 2)
    return np.sqrt(cost) / np.maximum(a, 1e-4)


def _weight_rounding(scheme, sigma, r, dist):
    """Relative error, in units of u, that float32 evaluation of the weight's transcendental adds: the argument of
    exp carries r^2 / sigma^2 (exp) or d^2 / sigma^2 (neighbourhood) ulps; log(1 + s^2) loses (1 + s^2) / log(1 + s^2)
    of its relative accuracy to the rounding of 1 + s^2 (Cauchy)."""
    s = SCHEMES[scheme]
    rel = np.ones_like(r)
    if s == 3:
        rel += r * r / sigma ** 2
    if s == 4:
        rel += dist * dist / sigma ** 2
    if s == 7:
        s2 = (r / sigma) ** 2
        rel += (1 + s2) / np.maximum(np.log1p(s2), 1e-300)
    return rel


def gn_terms_f64(ref, tgt, nrm, x, scheme, sigma):
    """Per correspondence r, J [n,6], w at pose x (float64).  nrm None selects the point-to-point cost, whose
    Jacobian is the reference's [d, (dR_k p) . d] (r times dr/dx, optimization.py:485-501)."""
    p, q = np.asarray(tgt, np.float64), np.asarray(ref, np.float64)
    T = build_pose(x)
    dR = euler_jacobian(np.asarray(x, np.float64)[3:])
    pm = p @ T[:3, :3].T + T[:3, 3]
    D = np.stack([p @ dR[k].T for k in range(3)], 1)  # [n,3(k),3]
    if nrm is not None:
        nn = np.asarray(nrm, np.float64)
        r = ((pm - q) * nn).sum(1)
        J = np.concatenate([nn, (D * nn[:, None, :]).sum(2)], 1)
    else:
        d = pm - q
        r = np.sqrt((d * d).sum(1))
        J = np.concatenate([d, (D * d[:, None, :]).sum(2)], 1)
    w = ls_weight(scheme, sigma, r, np.sqrt(((p - q) ** 2).sum(1)))
    return r, J, w


def gn_sums_f64(ref, tgt, nrm, x, scheme, sigma):
    """The 30 accumulators in the ICP order: 21 upper (wJ)(wJ)^T row-major, 6 (wJ)(wr), sum (wr)^2, sum r^2, count;
    and the per-element (w r)^2."""
    r, J, w = gn_terms_f64(ref, tgt, nrm, x, scheme, sigma)
    wj = J * w[:, None]
    wr = w * r
    s = np.zeros(NACC)
    k = 0
    for a in range(6):
        for b in range(a, 6):
            s[k] = (wj[:, a] * wj[:, b]).sum()
            k += 1
    s[21:27] = wj.T @ wr
    s[27], s[28], s[29] = (wr * wr).sum(), (r * r).sum(), float(len(r))
    return s, wr * wr


def normal_matrix(sums):
    H = np.zeros((6, 6))
    k = 0
    for a in range(6):
        for b in range(a, 6):
            H[a, b] = H[b, a] = sums[k]
            k += 1
    return H, sums[21:27].copy()


def gn_step_f64(sums):
    """One solve of gn_solve_kernel's rules: ('tiny', None) when sqrt(sum r^2) < 1e-7, ('singular', None) when
    |det H| < 1e-7, else ('ok', dx) with H dx = -g."""
    if np.sqrt(sums[28]) < 1e-7:
        return "tiny", None
    H, g = normal_matrix(sums)
    if not abs(np.linalg.det(H)) >= 1e-7:
        return "singular", None
    return "ok", np.linalg.solve(H, -g)


def gn_align_f64(ref, tgt, nrm, scheme, sigma, max_iters=1, norm_stop=1e-3, x0=None, f32=False):
    """The iteration of align_impl: x += dx until |dx| < norm_stop or max_iters.  f32 rounds dx and x to float32 after
    each step as the float32 kernel stores them.  Returns (status, x, iterations, per-element (w r)^2 of the last
    evaluated step)."""
    x = np.zeros(6) if x0 is None else np.asarray(x0, np.float64).copy()
    loss, status = None, "ok"
    for it in range(max(max_iters, 1)):
        sums, loss = gn_sums_f64(ref, tgt, nrm, x, scheme, sigma)
        status, dx = gn_step_f64(sums)
        if status != "ok":
            return status, x, it + 1, loss
        if f32:
            dx = dx.astype(np.float32).astype(np.float64)
            x = (x.astype(np.float32) + dx.astype(np.float32)).astype(np.float64)
        else:
            x = x + dx
        if np.sqrt((dx * dx).sum()) < norm_stop:
            return "ok", x, it + 1, loss
    return status, x, max(max_iters, 1), loss


def gn_f32_step_bound(ref, tgt, nrm, scheme, sigma):
    """Elementwise bound on |x_f32 - x_f64| of ONE float32 step from x = 0 (R = I, t = 0 and dR exact in float32).

    Per correspondence the float32 kernel rounds p - q, the residual, the Jacobian row and the weight; relative to the
    float64 values these carry e_r <= 5u sum|p - q||n| (point: 3u r + 2u |p - q|), e_J <= 6u sum|dR_k||p||n|, and the
    weight moves by its own change over r +- e_r plus 8u |w| (1 + r^2/sigma^2 for exp, + d^2/sigma^2 for the
    neighbourhood weight: the float32 argument of exp).  These give first-order bounds dH, dg of the float64-accumulated
    normal equations, and dx <= |H^-1| (dg + dH |dx|): the conditioning of H decides how far float32 terms move the
    step.  A factor 2 covers second order; 2u |dx| the two float32 stores of x."""
    p, q = np.asarray(tgt, np.float64), np.asarray(ref, np.float64)
    x = np.zeros(6)
    r, J, w = gn_terms_f64(ref, tgt, nrm, x, scheme, sigma)
    dR = euler_jacobian(x[3:])
    ad = np.abs(p - q)
    if nrm is not None:
        an = np.abs(np.asarray(nrm, np.float64))
        e_r = 5 * U * (ad * an).sum(1)
        e_J = np.concatenate([np.zeros_like(an), np.stack([6 * U * ((np.abs(p) @ np.abs(dR[k]).T) * an).sum(1) for k in range(3)], 1)], 1)
    else:
        e_r = 3 * U * r + 2 * U * ad.sum(1)
        e_d = 2 * U * ad
        Dp = np.stack([p @ dR[k].T for k in range(3)], 1)
        e_J = np.concatenate([e_d, np.stack([6 * U * ((np.abs(p) @ np.abs(dR[k]).T) * ad).sum(1) + (np.abs(Dp[:, k]) * e_d).sum(1)
                                             for k in range(3)], 1)], 1)
    dist = np.sqrt((ad * ad).sum(1))
    s = SCHEMES[scheme]
    wp, wm = ls_weight(scheme, sigma, r + e_r, dist), ls_weight(scheme, sigma, r - e_r, dist)
    rel = _weight_rounding(scheme, sigma, r, dist)
    dw = np.maximum(np.abs(wp - w), np.abs(wm - w)) + 8 * U * np.abs(w) * rel
    wj, wr = J * w[:, None], w * r
    dwj = np.abs(w)[:, None] * e_J + np.abs(J) * dw[:, None] + U * np.abs(wj)
    dwr = np.abs(w) * e_r + np.abs(r) * dw + U * np.abs(wr)
    dH = np.abs(wj).T @ dwj + dwj.T @ np.abs(wj)
    dg = np.abs(wj).T @ dwr + dwj.T @ np.abs(wr)
    sums, _ = gn_sums_f64(ref, tgt, nrm, x, scheme, sigma)
    H, g = normal_matrix(sums)
    dx = np.linalg.solve(H, -g)
    return 2 * np.abs(np.linalg.inv(H)) @ (dg + dH @ np.abs(dx)) + 2 * U * np.abs(dx)


# ----------------------------------------------------------------------------------------------- Procrustes
def procrustes_f64(tgt, ref, w=None):
    """T (4x4 float64) with T tgt ~ ref: weighted centroids, UNWEIGHTED cross-covariance, numpy.linalg.svd, and
    R = U diag(1, 1, sign(det U det V)) V^T (registration.py:15-76)."""
    pt, pr = np.asarray(tgt, np.float64), np.asarray(ref, np.float64)
    ww = np.ones(len(pt)) if w is None else np.asarray(w, np.float64).reshape(-1)
    mu_t = (pt * ww[:, None]).sum(0) / ww.sum()
    mu_r = (pr * ww[:, None]).sum(0) / ww.sum()
    Cm = (pr - mu_r).T @ (pt - mu_t)
    Um, _, Vt = np.linalg.svd(Cm)
    S = np.eye(3)
    if np.linalg.det(Um) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    T = np.eye(4)
    T[:3, :3] = Um @ S @ Vt
    T[:3, 3] = mu_r - T[:3, :3] @ mu_t
    return T


def gn_loss_bound(ref, tgt, nrm, x, scheme, sigma, u):
    """Per-element bound on the kernel's (w r)^2 against gn_sums_f64's, for unit roundoff u (2^-24 or 2^-53): the
    residual carries e_r <= 8u (|R||p| + |t| + |q|) . (|n| or 1); the bound is the change of (w r)^2 over r +- e_r
    (the scheme's own weight, kinks included) plus 16u of the value for the transcendental weight's rounding."""
    p, q = np.asarray(tgt, np.float64), np.asarray(ref, np.float64)
    T = build_pose(x)
    r, _, w = gn_terms_f64(ref, tgt, nrm, x, scheme, sigma)
    mag = np.abs(p) @ np.abs(T[:3, :3]).T + np.abs(T[:3, 3]) + np.abs(q)
    e_r = 8 * u * ((mag * np.abs(np.asarray(nrm, np.float64))).sum(1) if nrm is not None else mag.sum(1))
    dist = np.sqrt(((p - q) ** 2).sum(1))
    f0 = (w * r) ** 2
    fp = (ls_weight(scheme, sigma, r + e_r, dist) * (r + e_r)) ** 2
    fm = (ls_weight(scheme, sigma, r - e_r, dist) * (r - e_r)) ** 2
    rel = _weight_rounding(scheme, sigma, r, dist)
    return 2 * np.maximum(np.abs(fp - f0), np.abs(fm - f0)) + 16 * u * f0 * rel + 1e-300


# ----------------------------------------------------------------------------------------------- loss scenes
def _inverse_projection(row, col, rng_, pc):
    phi = (1.0 - row / pc["H"]) * pc["fov"] - pc["abs_down"]
    theta = (2.0 * col / pc["W"] - 1.0) * pc["pi"]
    return np.stack([rng_ * np.cos(phi) * np.cos(-theta), rng_ * np.cos(phi) * np.sin(-theta), rng_ * np.sin(phi)], -1)


def loss_scene(B, H, W, seed, up=3.0, down=-24.0, scheme="geman_mcclure", sigma=0.5, tie_probe=True):
    """Inputs of one training-loss call: target / reference vertex maps, reference normals [B,3,H,W] float32, pose
    parameters [B,6] and their float32 matrices [B,4,4].  Every batch element has its own pose, scene, null-pixel
    pattern and (odd elements) a NaN row; points land anywhere in the image, some beyond the vertical field of view,
    several per pixel.  Probes: points on the centres of the first / last row and column.  Element 0 carries, when W
    is even and W >= 8, two points of bit-identical range in one pixel (R = I, t = (0.3, 0, 0) and mirrored y, so
    that the float32 ranges agree whatever the transform's contraction); its reference normal (0, 1, 0) makes the
    winner move the residual by 2|y|.  Ambiguous points (see p2plane_loss_f64) are nulled until none remain."""
    rs = np.random.RandomState(seed)
    pc = proj_consts(H, W, up, down)
    HW = H * W
    params = np.zeros((B, 6))
    params[:, :3] = rs.normal(0, 0.5, (B, 3))
    params[:, 3:] = rs.normal(0, 0.05, (B, 3))
    tie = tie_probe and W % 2 == 0 and W >= 8
    if tie:
        params[0] = [0.3, 0, 0, 0, 0, 0]
    params = params.astype(np.float32)
    mats = np.stack([build_pose(params[b].astype(np.float64)) for b in range(B)]).astype(np.float32)
    vt = np.zeros((B, 3, H, W), np.float32)
    probes = []
    for b in range(B):
        row = rs.uniform(-0.45, H - 0.55, HW)
        col = rs.uniform(-0.45, W - 0.55, HW)
        out = rs.rand(HW) < 0.03                    # beyond the vertical field of view
        row[out] = np.where(rs.rand(out.sum()) < 0.5, rs.uniform(-4, -0.7, out.sum()), rs.uniform(H - 0.3, H + 4, out.sum()))
        rg = rs.uniform(2.0, 40.0, HW)
        k = min(HW, 8)
        border = rs.choice(HW, k, replace=False)   # exactly on the centres of the first / last row and column
        row[border] = np.array([0, 0, H - 1, H - 1, 0, H - 1, rs.randint(H), rs.randint(H)])[:k]
        col[border] = np.array([0, W - 1, 0, W - 1, rs.randint(W), rs.randint(W), 0, W - 1])[:k]
        pm = _inverse_projection(row, col, rg, pc)
        R, t = mats[b, :3, :3].astype(np.float64), mats[b, :3, 3].astype(np.float64)
        P = ((pm - t) @ R).astype(np.float32)
        P[rs.rand(HW) < 0.1] = 0.0                   # null target pixels
        if b % 2 == 1 and H > 1:
            r0 = rs.randint(H)
            P.reshape(H, W, 3)[r0] = np.nan          # a NaN row of the target map
        vt[b] = P.T.reshape(3, H, W)
        if b == 0 and tie:
            i1, i2 = np.sort(rs.choice(HW, 2, replace=False))
            p1 = _inverse_projection(np.array([(H - 1) // 2]), np.array([W / 2 - 0.3]), np.array([12.0]), pc)[0]
            p1 = np.array([p1[0] - 0.3, p1[1], p1[2]], np.float32)  # column W/2 - 0.3, its mirror W/2 + 0.3
            p2 = p1.copy()
            p2[1] = -p1[1]
            vt[0, :, i1 // W, i1 % W] = p1
            vt[0, :, i2 // W, i2 % W] = p2
            probes = [i1, i2]
    vr = np.zeros_like(vt)
    nr = np.zeros_like(vt)
    for _ in range(6):
        res = p2plane_loss_f64(vt, vr, nr, mats.astype(np.float64), H, W, up, down, scheme, sigma)
        amb = res["ambiguous"].copy()
        if tie:  # the probe pixel belongs to the two probes alone
            tp = res["pixel"][0, probes[0]]
            assert tp >= 0 and tp == res["pixel"][0, probes[1]], "tie probe points must share a pixel"
            amb[0] |= (res["pixel"][0] == tp)
            amb[0, probes] = False
        if not amb.any():
            break
        vt.reshape(B, 3, HW)[np.nonzero(amb)[0], :, np.nonzero(amb)[1]] = 0.0
    else:
        raise AssertionError("loss_scene: ambiguous points remain")
    for b in range(B):
        win = res["winner"][b]
        pw = np.zeros((HW, 3))
        P = vt[b].reshape(3, HW).T.astype(np.float64)
        R, t = mats[b, :3, :3].astype(np.float64), mats[b, :3, 3].astype(np.float64)
        has = win >= 0
        pw[has] = P[win[has]] @ R.T + t
        q = np.where(has[:, None], pw + rs.normal(0, 0.25, (HW, 3)), rs.normal(0, 10, (HW, 3)))
        n = rs.normal(0, 1, (HW, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        q[rs.rand(HW) < 0.05] = 0.0
        n[rs.rand(HW) < 0.05] = 0.0
        if b == 0 and tie:
            tp = res["pixel"][0, probes[0]]
            n[tp] = [0.0, 1.0, 0.0]
            q[tp] = pw[tp] + [0.0, 0.05, 0.0]
        vr[b] = q.T.reshape(3, H, W).astype(np.float32)
        nr[b] = n.T.reshape(3, H, W).astype(np.float32)
    return dict(vt=vt, vr=vr, nr=nr, params=params, mats=mats, tie=probes if tie else None, up=up, down=down)
