"""TEST INFRASTRUCTURE ONLY -- a float64 reference of ONE ICP iteration on the projective map, and of the model rebuild.

Given the exported model (pls_projmap_model: planar [K,3,H,W] vertices and normals, the GPU's own bits), the float32
queries and the float32 pose T the iteration linearises at, it computes in float64 what projmap.cu computes in float32:

  * the transformed queries, z-buffered with the oracle projector's pixel math (closest range wins, exact range ties
    go to the lowest query index);
  * per pixel the arg-min over the K candidates by the reference's rule (geometry.py:424-428): float32 square roots of
    the distances, the first minimum wins, all-zero candidates do not compete;
  * the 30 accumulators with kd_icp_reference.terms, and a tolerance from kd_icp_reference.float32_tolerance.

A query is *ambiguous* when the float32 evaluation could put it into another pixel or change its z-buffer rank; a
pixel is ambiguous when its top two candidates lie within the float32 error of each other.  Their spread goes into the
tolerance.  A comparison whose float32 evaluation is exact (dyadic coordinates: every difference, square and partial
sum representable) is decided exactly, the way the kernel decides it.
"""
import numpy as np
import torch

from oracle import icp_oracle as orc
from oracle import kd_icp_reference as kdr

NACC = kdr.NACC
U = 2.0 ** -24  # float32 unit roundoff
CHUNK = 1 << 14


def _f32_exact(x):
    x = np.asarray(x, np.float64)
    return np.asarray(x.astype(np.float32).astype(np.float64) == x)


def _norm2_exact(d):
    """d [...,3] float64 differences of float32 values: True where the float32 d.d is exact in every summation order."""
    s = d * d
    ok = _f32_exact(d).all(-1) & _f32_exact(s).all(-1)
    for a, b in ((0, 1), (0, 2), (1, 2)):
        ok &= _f32_exact(s[..., a] + s[..., b])
    return ok & _f32_exact(s.sum(-1))


def transform_error(T, q):
    """Bound of |p32 - p| per coordinate for the kernel's float32 transform of the queries q (0 at the identity)."""
    T = np.asarray(T, np.float32).reshape(4, 4)
    if np.array_equal(T, np.eye(4, dtype=np.float32)):
        return np.zeros(q.shape[0])
    s = np.abs(np.asarray(q, np.float64)).sum(1) + np.abs(T[:3, 3].astype(np.float64)).sum()
    return 4 * np.sqrt(3) * U * s


def pixels(p, H, W, up=3.0, down=-24.0, perr=None):
    """Float64 pixel of every point p [N,3] by the oracle projector.  Returns (pix [N] or -1, alternatives [N,3] pixel
    or -1: where a float32 evaluation could round the row or the column the other way, r [N])."""
    p = np.asarray(p, np.float64)
    n = p.shape[0]
    perr = np.zeros(n) if perr is None else np.asarray(perr, np.float64)
    row, col = orc.Projector(H, W, up, down).pixels(torch.from_numpy(p)[None])
    row, col = row[0].numpy(), col[0].numpy()
    r = np.linalg.norm(p, axis=1)
    rxy = np.maximum(np.hypot(p[:, 0], p[:, 1]), 1e-30)
    fov = abs(down / 180.0 * np.pi) + abs(up / 180.0 * np.pi)
    # float32 pixel coordinates: the transform moves the direction by perr / r, atan2f / asinf / the products by a few ulp
    m_row = H / fov * (2 * perr / np.maximum(r, 1e-30) + 64 * U) + 8 * U * H
    m_col = W / (2 * np.pi) * (2 * perr / rxy + 64 * U) + 8 * U * W

    def side(x, m, hi):
        c = np.rint(x)
        frac = x - np.floor(x)
        near = np.abs(frac - 0.5) <= m
        other = np.where(c > x, c - 1, c + 1)
        ok = (c >= 0) & (c <= hi)
        ok_o = near & (other >= 0) & (other <= hi)
        return c, ok, other, ok_o

    rc, rok, ro, rook = side(row, m_row, H - 1)
    cc, cok, co, cook = side(col, m_col, W - 1)
    live = r > 0
    pix = np.where(live & rok & cok, rc * W + cc, -1).astype(np.int64)
    alt = np.full((n, 3), -1, np.int64)
    alt[:, 0] = np.where(live & rook & cok, ro * W + cc, -1)
    alt[:, 1] = np.where(live & rok & cook, rc * W + co, -1)
    alt[:, 2] = np.where(live & rook & cook, ro * W + co, -1)
    # a point whose validity itself is in doubt (rounding across the image border) has its nominal pixel in doubt too
    doubt = live & ((rook & ~rok) | (cook & ~cok))
    alt[doubt & (pix >= 0), 0] = pix[doubt & (pix >= 0)]
    return pix, alt, r


def zbuffer(p, perr, H, W, up=3.0, down=-24.0):
    """Closest-wins z-buffer of the points p.  Returns (winner [HW] query index or -1, ambiguous [HW] bool, pairs: (query,
    pixel) arrays of every query that may end up in a pixel)."""
    n = p.shape[0]
    pix, alt, r = pixels(p, H, W, up, down, perr)
    hw = H * W
    win = np.full(hw, -1, np.int64)
    ok = np.nonzero(pix >= 0)[0]
    order = ok[np.lexsort((ok, r[ok], pix[ok]))]
    first = np.ones(order.shape[0], bool)
    first[1:] = pix[order][1:] != pix[order][:-1]
    win[pix[order[first]]] = order[first]
    amb = np.zeros(hw, bool)
    # a query that may land elsewhere leaves both pixels in doubt
    aq = np.nonzero((alt >= 0).any(1))[0]
    for c in range(3):
        sel = aq[alt[aq, c] >= 0]
        amb[alt[sel, c]] = True
    amb[pix[aq[pix[aq] >= 0]]] = True
    # rank: the runner-up of a pixel within the float32 error of the range (exact equal float32 norms decide by index)
    second = np.nonzero(~first)[0]
    second = second[(second > 0) & first[second - 1]]
    a, b = order[second - 1], order[second]
    tol = 8 * U * r[a] + 2 * (perr[a] + perr[b])
    exact_tie = (perr[a] == 0) & (perr[b] == 0) & _norm2_exact(p[a]) & _norm2_exact(p[b]) & (r[a] == r[b])
    close = (r[b] - r[a] <= tol) & ~exact_tie
    amb[pix[a[close]]] = True
    qs = [np.arange(n)[pix >= 0]] + [aq[alt[aq, c] >= 0] for c in range(3)]
    ps = [pix[pix >= 0]] + [alt[aq[alt[aq, c] >= 0], c] for c in range(3)]
    return win, amb, (np.concatenate(qs), np.concatenate(ps))


def argmin(model_v, pix, p, perr):
    """The reference's arg-min at pixels pix [M] for the points p [M,3].  model_v planar [K,3,H,W] float32.  Returns
    (k [M] or -1, admissible [M,K] bool: the candidates a float32 evaluation may pick, margin [M]: runner-up distance
    minus best distance)."""
    K = model_v.shape[0]
    flat = model_v.reshape(K, 3, -1)
    v = np.transpose(flat[:, :, pix], (2, 0, 1)).astype(np.float64)      # [M,K,3]
    live = np.abs(v).max(-1) > 0
    d = p[:, None, :] - v
    d2 = (d * d).sum(-1)
    root = np.where(live, np.sqrt(d2).astype(np.float32), np.float32(np.inf))
    k = np.argmin(root, axis=1)                                         # first minimum
    k = np.where(live.any(1), k, -1)
    rows = np.arange(pix.shape[0])
    dist = np.sqrt(d2)
    best = dist[rows, np.maximum(k, 0)]
    exact = _norm2_exact(d) & (perr[:, None] == 0)
    tol = 8 * U * best + 2 * perr
    adm = live & (dist <= (best + tol)[:, None])
    # pairs decided exactly: both squares exact -> the float32 roots of the exact squares decide, as in the kernel
    both = exact & exact[rows, np.maximum(k, 0)][:, None]
    adm &= ~both | (np.arange(K)[None, :] == k[:, None])
    adm[k < 0] = False
    other = np.where(live & (np.arange(K)[None, :] != k[:, None]), dist, np.inf)
    margin = other.min(1) - best
    return k, adm, margin


def _normals(model_n, k, pix):
    K = model_n.shape[0]
    flat = model_n.reshape(K, 3, -1)
    return flat[k, :, pix].astype(np.float64)


def proj_icp_iteration(model_v, model_n, queries_f32, T_f32, scheme, sigma, up=3.0, down=-24.0):
    """One projective ICP iteration in float64.  Returns a dict: sums [30], tol [30] (float32 rounding plus the spread of
    every ambiguous choice), count_tol (pixels whose count may differ), win [HW] query per pixel, k [HW] winning
    candidate, amb_query [HW] / amb_pixel [HW] ambiguity masks, p [N,3] the transformed queries."""
    K, _, H, W = model_v.shape
    q = np.asarray(queries_f32, np.float32)
    T = np.asarray(T_f32, np.float32).reshape(4, 4)
    p = kdr.transform(T, q)
    perr = transform_error(T, q)
    win, amb_q, (pq, pp) = zbuffer(p, perr, H, W, up, down)
    hw = H * W
    kk = np.full(hw, -1, np.int64)
    amb_k = np.zeros(hw, bool)
    sums = np.zeros(NACC)
    tol = np.zeros(NACC)
    px = np.nonzero(win >= 0)[0]
    for s in range(0, px.shape[0], CHUNK):
        pix = px[s:s + CHUNK]
        qi = win[pix]
        k, adm, _ = argmin(model_v, pix, p[qi], perr[qi])
        kk[pix] = k
        m = k >= 0
        pix, qi, k, adm = pix[m], qi[m], k[m], adm[m]
        if pix.shape[0] == 0:
            continue
        pm, qm, nm = p[qi], model_v.reshape(K, 3, -1)[k, :, pix].astype(np.float64), _normals(model_n, k, pix)
        sums += kdr.terms(pm, qm, nm, scheme, sigma).sum(0)
        e = 16 * U * (np.linalg.norm(pm, axis=1) + np.linalg.norm(qm, axis=1)) + 2 * perr[qi]
        tol += kdr.float32_tolerance(pm, qm, nm, scheme, sigma, e)
        # candidate ambiguity (query certain): the spread between the admissible choices
        several = (adm.sum(1) > 1) & ~amb_q[pix]
        amb_k[pix[several]] = True
        if several.any():
            t = []
            for j in range(K):
                use = several & adm[:, j]
                if not use.any():
                    continue
                kj = np.full(pix.shape[0], j)
                tj = np.full((pix.shape[0], NACC), np.nan)
                qj = model_v.reshape(K, 3, -1)[kj[use], :, pix[use]].astype(np.float64)
                tj[use] = kdr.terms(pm[use], qj, _normals(model_n, kj[use], pix[use]), scheme, sigma)
                t.append(tj)
            t = np.stack(t)[:, several]
            tol += (np.nanmax(t, 0) - np.nanmin(t, 0)).sum(0)
    # query ambiguity: any query that may land in such a pixel, with any admissible candidate, or nothing at all
    count_tol = int(amb_q.sum())
    sel = amb_q[pp]
    if sel.any():
        qa, pa = pq[sel], pp[sel]
        k, adm, _ = argmin(model_v, pa, p[qa], perr[qa])
        upix, slot = np.unique(pa, return_inverse=True)
        big = np.zeros((upix.shape[0], NACC))
        for j in range(K):
            use = adm[:, j]
            if not use.any():
                continue
            kj = np.full(use.sum(), j)
            qj = model_v.reshape(K, 3, -1)[kj, :, pa[use]].astype(np.float64)
            tj = np.abs(kdr.terms(p[qa[use]], qj, _normals(model_n, kj, pa[use]), scheme, sigma))
            np.maximum.at(big, slot[use], tj)
        tol += 2 * big.sum(0)
    return dict(sums=sums, tol=tol, count_tol=count_tol, win=win, k=kk, amb_query=amb_q, amb_pixel=amb_k, p=p)


def rebuild_model(vmaps, nmaps, poses, pose_err, H, W, up=3.0, down=-24.0):
    """Float64 rebuild of model_zbuf_kernel / model_resolve_kernel.  vmaps / nmaps [K,3,H,W] float32 source frames (oldest
    first), poses [K,4,4] float64 frame -> newest frame, pose_err [K] bound of the float32 pose chain's error (per unit
    of |v|_1 + |t|_1 + 1).  Returns (vertices [K,3,H,W], normals [K,3,H,W], occupied [K,H,W], ambiguous [K,H,W], err [K,H,W]
    bound of the vertex error)."""
    K = vmaps.shape[0]
    hw = H * W
    V = np.zeros((K, 3, hw))
    N = np.zeros((K, 3, hw))
    occ = np.zeros((K, hw), bool)
    amb = np.zeros((K, hw), bool)
    err = np.zeros((K, hw))
    for k in range(K):
        v = vmaps[k].reshape(3, hw).T.astype(np.float64)
        n = nmaps[k].reshape(3, hw).T.astype(np.float64)
        live = np.nonzero(np.abs(v).max(1) > 0)[0]
        P = np.asarray(poses[k], np.float64)
        p = v[live] @ P[:3, :3].T + P[:3, 3]
        s = np.abs(v[live]).sum(1) + np.abs(P[:3, 3]).sum()
        e = pose_err[k] * (s + 1) + 8 * U * s
        win, a, _ = zbuffer(p, e, H, W, up, down)
        has = win >= 0
        V[k][:, has] = p[win[has]].T
        N[k][:, has] = (n[live][win[has]] @ P[:3, :3].T).T
        occ[k] = has
        amb[k] = a
        err[k][has] = e[win[has]]
    return V.reshape(K, 3, H, W), N.reshape(K, 3, H, W), occ.reshape(K, H, W), amb.reshape(K, H, W), err.reshape(K, H, W)
