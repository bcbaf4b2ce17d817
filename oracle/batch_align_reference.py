"""TEST INFRASTRUCTURE ONLY -- float64 reference of the batched stand-alone alignments (gn.cu, pls_align_*_batch).

GaussNewton.compute (slam/common/optimization.py:296-344) iterates all B elements of a batch together:

  1. each element's residuals, Jacobian and weights at its own x[b];
  2. if the norm of all B*N unweighted residuals is below 1e-7: warn, every x unchanged;
  3. if any element's |det H| is below 1e-7: raise;
  4. x[b] += dx[b] for every element; stop all once the norm of all B*6 increments is below norm_stop.

Per element this reuses next_rows_reference's gn_sums_f64 (the 30 accumulators from gn_terms_f64) and normal_matrix; the
joint rules are restated here.  numpy only; the product path never imports it.
"""
import numpy as np

from . import next_rows_reference as nrr


def element_step(sums):
    """(det H, dx) of one element's normal equations H dx = -g (gn_step_f64 without its per-element residual guard,
    which the batch applies jointly)."""
    H, g = nrr.normal_matrix(sums)
    det = np.linalg.det(H)
    return det, (np.linalg.solve(H, -g) if abs(det) >= 1e-7 else np.full(6, np.nan))


def gn_align_batch_f64(ref, tgt, nrm, scheme, sigma, max_iters=1, norm_stop=1e-3, x0=None, f32=False):
    """ref / tgt / nrm [B,N,3] (nrm None: point-to-point).  f32 rounds dx and x to float32 after each step as the
    float32 kernel stores them.  Returns (status in {"ok", "tiny", "singular"}, x [B,6], iterations executed,
    per-element (w r)^2 [B,N] of the last evaluated step)."""
    ref, tgt = np.asarray(ref, np.float64), np.asarray(tgt, np.float64)
    B = ref.shape[0]
    x = np.zeros((B, 6)) if x0 is None else np.array(x0, np.float64).reshape(B, 6)
    loss = None
    iters = max(max_iters, 1)
    for it in range(iters):
        terms = [nrr.gn_sums_f64(ref[b], tgt[b], None if nrm is None else nrm[b], x[b], scheme, sigma) for b in range(B)]
        sums = np.stack([t[0] for t in terms])
        loss = np.stack([t[1] for t in terms])
        if np.sqrt(sums[:, 28].sum()) < 1e-7:
            return "tiny", x, it + 1, loss
        steps = [element_step(s) for s in sums]
        if not all(abs(det) >= 1e-7 for det, _ in steps):
            return "singular", x, it + 1, loss
        dx = np.stack([d for _, d in steps])
        if f32:
            dx = dx.astype(np.float32).astype(np.float64)
            x = (x.astype(np.float32) + dx.astype(np.float32)).astype(np.float64)
        else:
            x = x + dx
        if np.sqrt((dx * dx).sum()) < norm_stop:
            return "ok", x, it + 1, loss
    return "ok", x, iters, loss
