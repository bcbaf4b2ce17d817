"""TEST INFRASTRUCTURE ONLY -- a float64 reference of ONE ICP iteration on the kd map.

Given the float32 map (insertion order), the float32 queries and the float32 pose the iteration linearised at, it
computes in float64 what the CUDA iteration computes in float32 (kdmap.cu: kd_residual_kernel / kd_icp_refine_kernel):

  * the exact 1-NN of every transformed query and its runner-up distance (scipy cKDTree on the float64 map);
  * the normal of every matched map point from its exact k nearest other points (the construction of
    test_a9_normals_per_point_bound, with its eigen-gap);
  * the 30 accumulators with accumulate_normal_equations' definitions: wj = J w, JtJ upper from wj, Jtr from
    wj (w r), sum (w r)^2, sum r^2, count.

Residual, Jacobian and weights are the oracle's own (icp_oracle.p2plane_residual / p2plane_jacobian / ls_weights)
evaluated in float64 at x = 0.
"""
import numpy as np
import torch
from scipy.spatial import cKDTree

from oracle import icp_oracle as orc

NACC = 30
_UPPER = [(a, b) for a in range(6) for b in range(a, 6)]


def transform(T, pts):
    """float64 image of float32 points under a float32 4x4 pose (no rounding on the way)."""
    T = np.asarray(T, np.float64).reshape(4, 4)
    return np.asarray(pts, np.float64) @ T[:3, :3].T + T[:3, 3]


def residuals(p, q, n, scheme, sigma, r_shift=0.0, d_scale=None):
    """(r [N], J [N,6], w [N]) in float64 through the oracle's residual, Jacobian and weights at x = 0.  r_shift is
    added to every residual and d_scale [N] scales p - q inside the `neighborhood` weight (how the tolerance of a
    float32 evaluation is probed)."""
    p, q, n = (torch.from_numpy(np.ascontiguousarray(a, np.float64))[None] for a in (p, q, n))
    x = torch.zeros(1, 6, dtype=torch.float64)
    r = orc.p2plane_residual(x, p, q, n) + torch.as_tensor(r_shift, dtype=torch.float64)
    J = orc.p2plane_jacobian(x, p, n)
    ref = q if d_scale is None else p - (p - q) * torch.from_numpy(np.asarray(d_scale, np.float64))[None, :, None]
    w = orc.ls_weights(scheme, sigma, r, p, ref).expand_as(r)
    return r[0].numpy(), J[0].numpy(), w[0].numpy()


def terms(p, q, n, scheme, sigma, r_shift=0.0, d_scale=None):
    """Per correspondence: the 30 accumulator terms [N, 30] (float64), accumulate_normal_equations' definitions."""
    r, J, w = residuals(p, q, n, scheme, sigma, r_shift, d_scale)
    wj = J * w[:, None]
    wr = w * r
    out = np.empty((wj.shape[0], NACC))
    for k, (a, b) in enumerate(_UPPER):
        out[:, k] = wj[:, a] * wj[:, b]
    out[:, 21:27] = wj * wr[:, None]
    out[:, 27] = wr * wr
    out[:, 28] = r * r
    out[:, 29] = 1.0
    return out


def accumulate(p, q, n, scheme, sigma):
    """The 30 accumulators of the correspondences (p, q, n), float64."""
    return terms(p, q, n, scheme, sigma).sum(0)


def float32_tolerance(p, q, n, scheme, sigma, e):
    """Per accumulator, how far a float32 evaluation of the same correspondences may land from accumulate(p, q, n):
    e [N] bounds the float32 error of the residual r, of the distance |p - q| and of each component of p x n (the
    Jacobian's rotation part; its translation part is n itself).  The worst deviation of every term with r and |p - q|
    moved by +-e, plus the first-order effect of +-e on J[3:6], summed over the correspondences, plus 1e-6 of the sum
    of |term| for the rounding of the weight and of the products (a few float32 ulp)."""
    e = np.asarray(e, np.float64)
    t0 = terms(p, q, n, scheme, sigma)
    d = np.linalg.norm(np.asarray(p, np.float64) - np.asarray(q, np.float64), axis=1)
    dev = np.zeros_like(t0)
    for sr in (1.0, -1.0):
        for sd in (1.0, -1.0):
            scale = np.where(d > 0, (d + sd * e) / np.where(d > 0, d, 1.0), 1.0)
            dev = np.maximum(dev, np.abs(terms(p, q, n, scheme, sigma, r_shift=sr * e, d_scale=scale) - t0))
    r, J, w = residuals(p, q, n, scheme, sigma)
    eJ = np.zeros_like(J)
    eJ[:, 3:] = e[:, None]
    aJ = np.abs(J)
    for k, (a, b) in enumerate(_UPPER):
        dev[:, k] += w * w * (aJ[:, a] * eJ[:, b] + aJ[:, b] * eJ[:, a] + eJ[:, a] * eJ[:, b])
    dev[:, 21:27] += (w * w * np.abs(r))[:, None] * eJ
    return dev.sum(0) + 1e-6 * np.abs(t0).sum(0)


def gauss_newton_step(sums):
    """x = -H^-1 g from the accumulators (float64), H from the 21 upper entries."""
    H = np.zeros((6, 6))
    for k, (a, b) in enumerate(_UPPER):
        H[a, b] = H[b, a] = sums[k]
    return -np.linalg.solve(H, np.asarray(sums[21:27], np.float64))


def exact_normals(map_f32, tree, idx, k):
    """float64 normals of the map points `idx` from their exact k nearest other points.  Returns (normals [n,3],
    gap [n] = (lambda_mid - lambda_min) / lambda_max, unique [n]: no distance tie at the k-th neighbour)."""
    m = np.asarray(map_f32)
    d, nb = tree.query(m[idx].astype(np.float64), k=k + 2, workers=-1)
    unique = d[:, k + 1] > d[:, k] * (1 + 1e-6)
    diff = (m[nb[:, 1:k + 1]] - m[idx][:, None, :]).astype(np.float64)
    C = np.einsum("nki,nkj->nij", diff, diff) / k
    w, v = np.linalg.eigh(C)
    gap = (w[:, 1] - w[:, 0]) / np.maximum(w[:, 2], 1e-300)
    return v[:, :, 0], gap, unique


def kd_icp_iteration(map_f32, queries_f32, T_f32, scheme, sigma, k=10, tree=None):
    """One ICP iteration in float64.  Returns a dict: p [N,3] transformed queries, match [N] insertion index of the
    exact 1-NN, d1 / d2 [N] nearest and runner-up distance, normals [N,3] of the matched points (float64, sign
    arbitrary), gap / unique [N] of those normals, sums [30]."""
    m64 = np.asarray(map_f32, np.float64)
    tree = tree if tree is not None else cKDTree(m64)
    p = transform(T_f32, queries_f32)
    d, nb = tree.query(p, k=2, workers=-1)
    match = nb[:, 0]
    u, inv = np.unique(match, return_inverse=True)
    nrm, gap, unique = exact_normals(map_f32, tree, u, k)
    out = dict(p=p, match=match, d1=d[:, 0], d2=d[:, 1], normals=nrm[inv], gap=gap[inv], unique=unique[inv])
    out["sums"] = accumulate(p, m64[match], out["normals"], scheme, sigma)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# The (k+1)-NN lists and second moments of the kd map's normals (kdmap_device.cuh: warp_knn, warp_second_moments).
#
# The kernel orders a map point's neighbours by the 64-bit key (float32 d^2 bits, sorted position): the sorted
# position is the point's index in the array the index build sorts by the Morton code of its level-0 cell (insertion
# order inside a cell).  warp_second_moments then sums the float32 outer products of entries 1..k sequentially in that
# order and divides by k -- numpy's `.mean(axis=1)` of the reference's float32 differences.
KD_COORD_MAX = 8191
KD_B0 = 3
KD_CELL_MARGIN = np.float32(2e-3)
U32 = 2.0 ** -24        # float32 unit roundoff
EPS64 = 2.0 ** -52
# float32 d^2 of the kernel (dist2_point: three rounded differences, their squares summed with at most three roundings)
# is within D2_REL * d^2 of the float64 d^2 of the same float32 coordinates: 2 u from the rounded differences (squared),
# 3 u from the products and sums, and one u of slack.
D2_REL = 6 * U32


def _spread10(x):
    x = x.astype(np.uint32) & np.uint32(0x3FF)
    x = (x | (x << np.uint32(16))) & np.uint32(0x030000FF)
    x = (x | (x << np.uint32(8))) & np.uint32(0x0300F00F)
    x = (x | (x << np.uint32(4))) & np.uint32(0x030C30C3)
    x = (x | (x << np.uint32(2))) & np.uint32(0x09249249)
    return x


def kernel_grid(map_f32, cell_target=0.2):
    """kd_grid_header_kernel in float32: (mn [3], scale).  The bounding box is the exact min / max of the points; the
    scale makes a level-0 cell (8 quantisation units) `cell_target` metres wide unless the 13-bit range must cover a
    wider extent."""
    m = np.asarray(map_f32, np.float32)
    mn, mx = m.min(0), m.max(0)
    ext = np.float32(max(float((mx - mn).max()), float(np.float32(1e-6))))
    scale = min(np.float32(8) / np.float32(cell_target), np.float32(KD_COORD_MAX) / ext)
    return mn, np.float32(scale)


def kernel_quantise(map_f32, mn, scale):
    """kd_cell_key_kernel's quantised coordinates [M, 3] (uint32): clamp to [0, 8191] in float32, truncate."""
    f = (np.asarray(map_f32, np.float32) - mn) * scale
    return np.minimum(np.maximum(f, np.float32(0)), np.float32(KD_COORD_MAX)).astype(np.uint32)


def kernel_cell_ids(q):
    """Morton id of the level-0 cell of quantised coordinates q [M, 3]."""
    c = q >> np.uint32(KD_B0)
    return _spread10(c[:, 0]) | (_spread10(c[:, 1]) << np.uint32(1)) | (_spread10(c[:, 2]) << np.uint32(2))


def kernel_sort_positions(map_f32, cell_target=0.2):
    """Each map point's position in the kernel's `sorted` array: a stable sort of the level-0 Morton ids."""
    mn, scale = kernel_grid(map_f32, cell_target)
    order = np.argsort(kernel_cell_ids(kernel_quantise(map_f32, mn, scale)), kind="stable")
    pos = np.empty(len(order), np.int64)
    pos[order] = np.arange(len(order))
    return pos


def _d2_exact_in_float32(m, qv, nb):
    """True where the float32 d^2 of dist2_point involves no rounding (every difference, square and partial sum is a
    float32 value), so it equals the float64 d^2 whatever the order of the additions."""
    d32 = m[nb] - qv[:, None, :]                               # float32 differences
    d64 = m[nb].astype(np.float64) - qv[:, None, :].astype(np.float64)
    ok = (d32.astype(np.float64) == d64).all(-1)
    sq = d64 * d64
    ok &= (sq.astype(np.float32).astype(np.float64) == sq).all(-1)
    s1 = sq[..., 0] + sq[..., 1]
    s2 = s1 + sq[..., 2]
    return ok & (s1.astype(np.float32) == s1) & (s2.astype(np.float32) == s2)


def knn_lists(map_f32, queries, k, positions, tree=None):
    """The exact (k+1)-NN of each query in the kernel's order (float64 d^2 of the float32 coordinates, then sorted
    position).  Returns (idx [n, k+1] insertion index or -1 past the map's size, pos [n, k+1] or -1, d2 [n, k+1] float64
    or inf, ambiguous [n]).

    A query is ambiguous when two of its entries, or its last entry and the next point, have float64 d^2 within
    2 D2_REL of each other without being two equal d^2 that float32 computes exactly: there the kernel's float32 d^2 may
    order them differently.  Exact ties of exactly computed d^2 are decided by the position, as in the kernel."""
    m = np.asarray(map_f32, np.float32)
    qv = np.asarray(queries, np.float32)
    M, n, K = m.shape[0], qv.shape[0], k + 1
    tree = tree if tree is not None else cKDTree(m.astype(np.float64))
    want = min(M, K + 1)                                    # the list and the point after it
    kq = min(M, K + 8)
    while True:
        d, nb = tree.query(qv.astype(np.float64), k=kq, workers=-1)
        d, nb = d.reshape(n, kq), nb.reshape(n, kq)
        if kq == M:
            break
        # every point tied (within the band) with the last one needed must be among the candidates
        need = d[:, want - 1] * (1 + 4 * D2_REL) + 1e-30
        if (d[:, kq - 1] > need).all():
            break
        kq = min(M, 2 * kq)
    diff = m[nb].astype(np.float64) - qv[:, None, :].astype(np.float64)
    d2 = (diff * diff).sum(-1)
    p = positions[nb]
    order = np.lexsort((p, d2), axis=1)
    nb = np.take_along_axis(nb, order, 1)
    d2 = np.take_along_axis(d2, order, 1)
    p = np.take_along_axis(p, order, 1)
    exact = _d2_exact_in_float32(m, qv, nb)
    a, b = d2[:, :want - 1], d2[:, 1:want]
    close = (b - a) <= 2 * D2_REL * b
    tie_ok = (a == b) & exact[:, :want - 1] & exact[:, 1:want]
    ambiguous = (close & ~tie_ok).any(1)
    idx = np.full((n, K), -1, np.int64)
    pos = np.full((n, K), -1, np.int64)
    dd = np.full((n, K), np.inf)
    f = min(K, M)
    idx[:, :f], pos[:, :f], dd[:, :f] = nb[:, :f], p[:, :f], d2[:, :f]
    return idx, pos, dd, ambiguous


def reference_covs(map_f32, centre_idx, lists, k):
    """Second moments [n, 3, 3] (float32) about map points centre_idx of entries 1..k of their neighbour lists, with the
    reference's own expression (local_map.py:411-413, icp_oracle.KdTreeLocalMap._normals_for): float32 differences,
    outer products, `.mean(axis=1)`.  An entry -1 (a map of at most k points) stands for a zero difference: the sum of
    the found - 1 others divided by k, which is what warp_second_moments computes there."""
    m = np.asarray(map_f32, np.float32)
    centre = m[np.asarray(centre_idx)]
    nb = np.asarray(lists)[:, 1:k + 1]
    pts = np.where((nb >= 0)[:, :, None], m[np.maximum(nb, 0)], centre[:, None, :])
    d = pts - centre[:, None, :]
    return (d[:, :, :, None] * d[:, :, None, :]).mean(axis=1)


def tight_normal_bound(covs64):
    """Permitted |sin| between a normal the kernel computes from these (float32-valued) moments and the float64 eigh
    eigenvector of the same moments.  Returns (bound [n], gap [n] = (lambda_mid - lambda_min) / lambda_max).

    The moments are the same numbers on both sides, so only two errors remain:
      * the float32 rounding of the three components of the float64 unit vector the solver returns: each moves by at
        most u |n_i|, so the direction by at most u; sqrt(3) u is taken;
      * the float64 solve, on either side.  Jacobi rotations and the row cross products of the closed form, like
        LAPACK's eigh, are backward stable: a perturbation of c eps64 lambda_max of the matrix turns the vector by
        c eps64 lambda_max / gap (c = 16 covers the three solvers).  The closed form also takes lambda_min from
        acos(r) / 3: near r = +-1 (small gap) an error dr of r moves lambda_min by (2/3) p^2 dr / gap with
        p <= lambda_max, and the vector by that over the gap; dr <= 12 eps64 gives 8 eps64 (lambda_max / gap)^2.  The
        solver uses the closed form only where gap >= 1e-3 (lambda_max - lambda_min) (0.5e-3 here for margin), and
        Jacobi below, where the acos term does not apply."""
    C = np.asarray(covs64, np.float64)
    w = np.linalg.eigvalsh(C)
    lmax = np.maximum(np.abs(w[:, 2]), 1e-300)
    gap_abs = w[:, 1] - w[:, 0]
    gap = gap_abs / lmax
    inv = np.minimum(lmax / np.maximum(gap_abs, 1e-300), 1e100)   # degenerate: unbounded in effect
    closed = gap_abs >= 0.5e-3 * np.maximum(w[:, 2] - w[:, 0], 1e-300)
    bound = np.sqrt(3) * U32 + 16 * EPS64 * inv + np.where(closed, 8 * EPS64 * inv * inv, 0.0)
    return bound, gap


def level0_paths(map_f32, queries, k, kth_d2, cell_target=0.2):
    """warp_probe_block at level 0 in float32, per query: (candidates [n] = points in the 27-cell block, exact [n] =
    k+1 candidates and the (k+1)-th float32 d^2 `kth_d2` within the block's exactness radius).  The selection path
    follows: <= 64 candidates knn_select_small<2>, 65 ... 128 knn_select_small<4>, more the streaming filter with at
    least (candidates / 32 - 1) merges of 32 keys; a query that is not exact goes on to the coarser levels."""
    m = np.asarray(map_f32, np.float32)
    qv = np.asarray(queries, np.float32)
    mn, scale = kernel_grid(m, cell_target)
    cells = kernel_quantise(m, mn, scale).astype(np.int64) >> KD_B0
    cmax = KD_COORD_MAX >> KD_B0
    key = lambda c: (c[..., 0] * (cmax + 1) + c[..., 1]) * (cmax + 1) + c[..., 2]
    ids, counts = np.unique(key(cells), return_counts=True)
    f = np.minimum(np.maximum((qv - mn) * scale, np.float32(-1e6)), np.float32(1e6))
    c = np.clip(np.floor(f).astype(np.int64) >> KD_B0, 0, cmax)
    total = np.zeros(len(qv), np.int64)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                cc = c + np.array([dx, dy, dz])
                inside = ((cc >= 0) & (cc <= cmax)).all(1)
                kk = key(np.clip(cc, 0, cmax))
                j = np.minimum(np.searchsorted(ids, kk), len(ids) - 1)
                total += np.where(inside & (ids[j] == kk), counts[j], 0)
    side = np.float32(1 << KD_B0)
    lo = f - c.astype(np.float32) * side
    hi = (c + 1).astype(np.float32) * side - f
    own = np.maximum(np.minimum(lo, hi).min(1), np.float32(0))
    inv_scale = np.float32(1) / scale
    cell = ((side + own).astype(np.float64) * np.float64(inv_scale) - np.float64(KD_CELL_MARGIN)).astype(np.float32)
    r2 = np.where(cell > 0, cell * cell, np.float32(-1))
    exact = (total >= k + 1) & (np.asarray(kth_d2, np.float32) <= r2)
    return total, exact
