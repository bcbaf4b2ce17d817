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
