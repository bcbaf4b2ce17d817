"""TEST INFRASTRUCTURE ONLY -- a float64 restatement of pls_kdmap_evaluate_poses (include/plslam_b200.h).

Given one pose's float32 transformed valid rows p' (transform_point's bits), the float32 map point each was matched to
and that point's float32 normal, it forms the row the kernel writes:

  * d^2 = ((dx dx + dy dy) + dz dz) in float64, dx = float64(p'_x) - float64(q_x): numpy's element-wise float64
    operations, each rounded once, give the kernel's bits;
  * a query is an inlier when it has a match and d^2 <= max_distance * max_distance (float64);
  * [0..29] the accumulators of kd_icp_reference.terms (accumulate_normal_equations' definitions) over the inliers,
    [30] sum d^2 over the inliers, [31] the number of valid rows.

The sums are float64 sums in numpy's order, not the kernel's block order: they agree with the kernel to float64
summation error, the inlier set and the counts exactly (the residual terms themselves are float64 images of the
oracle's residual, so they carry the float32 differences kd_icp_reference.float32_tolerance bounds).
"""
import numpy as np

from oracle import kd_icp_reference as kref

EVAL_STATS = 32


def match_d2(p, q):
    """The kernel's float64 d^2 of float32 points p [N,3] and their matches q [N,3] (float64 inputs are taken as they
    are: the float64 images kd_icp_reference works with)."""
    d = np.asarray(p).astype(np.float64) - np.asarray(q).astype(np.float64)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def inliers(p, q, matched, max_distance):
    """Boolean [N]: matched and d^2 <= max_distance^2 (float64).  Unmatched rows' q may hold anything."""
    matched = np.asarray(matched, bool)
    qq = np.where(matched[:, None], np.asarray(q), 0)
    md = np.float64(max_distance)
    return matched & (match_d2(p, qq) <= md * md)


def evaluate_row(p, q, normals, matched, max_distance, scheme, sigma):
    """The PLS_EVAL_STATS row of one pose: p [N,3] its transformed valid rows, q / normals [N,3] the matched points
    and their normals (float32), matched [N] whether a row found a match."""
    p = np.asarray(p)
    keep = inliers(p, q, matched, max_distance)
    row = np.zeros(EVAL_STATS)
    if keep.any():
        pk, qk = p[keep], np.asarray(q)[keep]
        row[:30] = kref.terms(pk, qk, np.asarray(normals)[keep], scheme, sigma).sum(0)
        row[30] = match_d2(pk, qk).sum()
    row[31] = p.shape[0]
    return row, keep
