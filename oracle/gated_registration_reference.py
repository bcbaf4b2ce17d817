"""TEST INFRASTRUCTURE ONLY -- a float64 restatement of one gated ICP iteration of pls_register_scans_gated
(include/plslam_b200.h), and of the scene the gate is for.

  * gate_bound / dmax32: the float32 bounds kd_gate_of derives from max_distance (KdGate, kdmap_device.cuh);
  * gated_iteration: matches in (the float32 transformed rows p', their matched map points and normals), the gated
    accumulators, inlier count and Gauss-Newton step out.  The inlier test and the sums are those of
    oracle/evaluate_poses_reference.evaluate_row at the same gate: d^2 in float64, every operation rounded once;
  * brute_force_gated_nn: for small maps, every query's exact 1-NN with the map's tie rule (d^2, then sorted position),
    -1 for an outlier, and whether float32 rounding could change the winner;
  * changed_map_scene / icp: a prior map that no longer matches the world (an object the map lacks stands in the
    scan, 3 m in front of a wall) and a float64 point-to-plane ICP with and without the gate.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle import evaluate_poses_reference as er
from oracle import kd_icp_reference as kref


def _f32_up(v):
    """The least float32 >= v (float64), +inf above FLT_MAX."""
    v = np.float64(v)
    if not v <= np.float64(np.finfo(np.float32).max):
        return np.float32(np.inf)
    f = np.float32(v)
    return np.nextafter(f, np.float32(np.inf)) if np.float64(f) < v else f


def gate_bound(max_distance):
    """G: a float32 strictly above every float32 d^2 of an inlier (derivation at KdGate)."""
    d2 = np.float64(max_distance) * np.float64(max_distance)
    return _f32_up(d2 * (1.0 + 2.0 ** -20) + 2.0 ** -126)


def dmax32(max_distance):
    return _f32_up(max_distance)


def gated_iteration(p, q, normals, matched, max_distance, scheme, sigma):
    """One gated iteration from its matches.  Returns dict(sums [30], inliers [N] bool, count, step [6] or None when
    the 6x6 system is singular (|det| < 1e-7, the kernel's test))."""
    row, keep = er.evaluate_row(p, q, normals, matched, max_distance, scheme, sigma)
    sums = row[:30]
    H = np.zeros((6, 6))
    for k, (a, b) in enumerate(kref._UPPER):
        H[a, b] = H[b, a] = sums[k]
    step = None if abs(np.linalg.det(H)) < 1e-7 else kref.gauss_newton_step(sums)
    return dict(sums=sums, inliers=keep, count=int(keep.sum()), step=step)


def brute_force_gated_nn(map_f32, positions, p, max_distance):
    """Exact gated 1-NN of float32 rows p [N,3] by brute force (small maps).  positions [M]: each map point's sorted
    position (kd_icp_reference.kernel_sort_positions), the tie rule's second key.  Returns (match [N] insertion index or
    -1, decided [N]): decided is False where float32 d^2 could order the best two differently or put the winner on the
    other side of the gate (within kd_icp_reference.D2_REL of either)."""
    m = np.asarray(map_f32, np.float32)
    p = np.asarray(p, np.float32)
    md2 = np.float64(max_distance) ** 2
    match = np.full(len(p), -1, np.int64)
    decided = np.ones(len(p), bool)
    for s in range(0, len(p), 256):
        d2 = er.match_d2(np.repeat(p[s:s + 256], len(m), 0), np.tile(m, (len(p[s:s + 256]), 1))).reshape(-1, len(m))
        order = np.lexsort((np.broadcast_to(positions, d2.shape), d2), axis=1)
        best = order[:, 0]
        b1 = d2[np.arange(len(best)), best]
        b2 = d2[np.arange(len(best)), order[:, 1]] if len(m) > 1 else np.full(len(best), np.inf)
        inl = b1 <= md2
        match[s:s + 256] = np.where(inl, best, -1)
        slack = 4 * kref.D2_REL
        near_tie = b2 <= b1 * (1 + slack) + 1e-30
        near_gate = np.abs(b1 - md2) <= slack * max(md2, 1e-30) + 1e-30
        decided[s:s + 256] = ~(inl & near_tie) & ~near_gate
    return match, decided


# -------------------------------------------------------------------------------------------------- the changed map
def _plane(rng, n, origin, u, v):
    a, b = rng.uniform(0, 1, (2, n))
    return np.asarray(origin) + a[:, None] * np.asarray(u) + b[:, None] * np.asarray(v)


def changed_map_scene(seed=0):
    """A 40 m room (floor, four walls) as the prior map; the scan samples the same room and also a 6 x 2.5 m object the
    map lacks (a parked truck's side), standing 3 m in front of the x = +20 wall, 2.5-5 m above the floor, so that its
    nearest map points lie on that wall.  Returns (map [M,3], scan [N,3], truth [4,4], start [4,4]) float32; the truth
    is the identity, the start 0.3 m and 2 degrees off."""
    rng = np.random.RandomState(seed)
    def room(n):
        return np.concatenate([
            _plane(rng, n, [-20, -20, 0], [40, 0, 0], [0, 40, 0]),
            _plane(rng, n // 2, [20, -20, 0], [0, 40, 0], [0, 0, 8]),
            _plane(rng, n // 2, [-20, -20, 0], [0, 40, 0], [0, 0, 8]),
            _plane(rng, n // 2, [-20, 20, 0], [40, 0, 0], [0, 0, 8]),
            _plane(rng, n // 2, [-20, -20, 0], [40, 0, 0], [0, 0, 8])])
    prior = room(40000).astype(np.float32)
    world = room(6000)
    truck = _plane(rng, 6000, [17, -3, 2.5], [0, 6, 0], [0, 0, 2.5])
    scan = np.concatenate([world, truck]).astype(np.float32)
    start = np.eye(4, dtype=np.float32)
    c, s = np.cos(np.deg2rad(2.0)), np.sin(np.deg2rad(2.0))
    start[:2, :2] = [[c, -s], [s, c]]
    start[:3, 3] = [0.3, -0.2, 0.05]
    return np.ascontiguousarray(prior), np.ascontiguousarray(scan), np.eye(4, dtype=np.float32), start


def _rot(w):
    th = np.linalg.norm(w)
    if th < 1e-300:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def icp(map_f32, scan_f32, T0, max_distance=np.inf, iters=30, k=10, scheme="default", sigma=0.3):
    """float64 point-to-plane ICP (exact 1-NN, exact k-NN normals, one Gauss-Newton step per iteration, the step
    applied on the left) with the gate.  Returns (T [4,4] float64, inliers of the last iteration)."""
    m64 = np.asarray(map_f32, np.float64)
    tree = cKDTree(m64)
    T = np.asarray(T0, np.float64).copy()
    q = np.asarray(scan_f32, np.float64)
    count = 0
    for _ in range(iters):
        p = q @ T[:3, :3].T + T[:3, 3]
        _, nb = tree.query(p, k=1, workers=-1)
        u, inv = np.unique(nb, return_inverse=True)
        nrm = kref.exact_normals(map_f32, tree, u, k)[0][inv]
        it = gated_iteration(p, m64[nb], nrm, np.ones(len(p), bool), max_distance, scheme, sigma)
        count = it["count"]
        if it["step"] is None:
            break
        x = it["step"]
        D = np.eye(4)
        D[:3, :3] = _rot(x[3:])
        D[:3, 3] = x[:3]
        T = D @ T
        if np.linalg.norm(x) < 1e-6:
            break
    return T, count


def pose_error(T, truth):
    """(translation error m, rotation error rad)."""
    T, truth = np.asarray(T, np.float64), np.asarray(truth, np.float64)
    dR = truth[:3, :3].T @ T[:3, :3]
    ang = np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1))
    return float(np.linalg.norm(T[:3, 3] - truth[:3, 3])), float(ang)
