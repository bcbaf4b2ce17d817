"""Every ICP iteration on the kd map against a float64 reference (oracle/kd_icp_reference.py), per query.

ICP iterations after a frame's first do not search: a query keeps its match when `(d + eps) * 1.00001 + 1e-6 <
sqrt(second)` proves it (kd_icp_refine_kernel below KD_COLD_MAP_POINTS map points, kd_nn_verify_kernel and three more
launches above), where `second` is the runner-up bound stored by the query's last full search.  A bound a little too
large keeps stale matches that move a pose far less than the pose tolerances of the other tests.  So here:

  * run j of a register call (threshold_delta_pose = 0, max_num_alignments = j, a fresh context on the same map) is
    read back with pls_kdmap_last_correspondences: its matches, normals, search states and accumulators are those of
    iteration j, linearised at the pose run j-1 returned;
  * every query's match is an exact nearest neighbour, every search state's runner-up bound holds, every normal meets
    the test_a9 bound and equals the normal a fresh nn_search computes, the accumulators equal float64 sums of the
    same correspondences within float32 rounding, and the pose update is the float64 solve of those sums.
"""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

pytestmark = pytest.mark.gpu

K_NORMALS = 10
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
REFINE_ROUND = 8 * 132 * 256          # queries one launch of kd_icp_refine_kernel handles in its first round
COLD_MAP_POINTS = 2_000_000           # kdmap.cu: KD_COLD_MAP_POINTS (four launches per later iteration from here)
U = 2.0 ** -24                        # float32 unit roundoff


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def ref():
    from oracle import kd_icp_reference
    return kd_icp_reference


def _perturbed(T, metres, degrees, seed):
    rng = np.random.RandomState(seed)
    axis = rng.randn(3)
    d = rng.randn(3)
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(degrees)).as_matrix()
    P[:3, 3] = d / np.linalg.norm(d) * metres
    return (np.asarray(T, np.float64) @ P).astype(np.float32)


@pytest.fixture(scope="module")
def scene():
    """cfg2-shaped: 20 synthetic 64x2048 frames grid-sampled at 0.3 m in a kd map; the next frame's samples as queries,
    T0 = its ground-truth pose perturbed by 0.3 m / 1 degree."""
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20))
    lm.init()
    for k in range(20):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        s, _ = b200.grid_sample(syn.scan(k, 64, 2048), 0.3)
        lm.update(rel[None], new_pc_data=s)
    m = np.ascontiguousarray(lm.points())
    lm.ctx.close()
    q, _ = b200.grid_sample(syn.scan(20, 64, 2048), 0.3)
    dense = syn.scan(20, 128, 4096)
    dense = np.ascontiguousarray(dense[np.isfinite(dense).all(1) & (np.abs(dense).sum(1) > 0)])
    T_gt = syn.gt_relative_pose(20)
    return dict(m=m, q=np.ascontiguousarray(q), dense=dense, T_gt=T_gt, T0=_perturbed(T_gt, 0.3, 1.0, 0),
                tree=cKDTree(m.astype(np.float64)))


# ---------------------------------------------------------------------------------------------------------- driving
def _context(lib, iters, scheme="geman_mcclure", sigma=0.3, k=K_NORMALS):
    return lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=1, num_neighbors_normals=k,
                       scheme=lib.SCHEMES[scheme], sigma=sigma, gn_max_iters=1, max_num_alignments=iters,
                       threshold_delta_pose=0.0)


def _insert(lib, ctx, m):
    ctx.call("pls_kdmap_update_points", lib.ptr(np.eye(4, dtype=np.float32)), lib.ptr(m), m.shape[0])


def _readback(lib, ctx, n):
    out = dict(idx=np.empty(n, np.int64), nb=np.empty((n, 3), np.float32), nrm=np.empty((n, 3), np.float32),
               state=np.empty((n, 4), np.float32), sums=np.empty(30, np.float64))
    ctx.call("pls_kdmap_last_correspondences", n, lib.ptr(out["idx"]), lib.ptr(out["nb"]), lib.ptr(out["nrm"]),
             lib.ptr(out["state"]), lib.ptr(out["sums"]))
    return out


def _register(lib, ctx, q, T0, iters):
    T, params, losses, it = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(iters, np.float32), C.c_int(0)
    ctx.call("pls_register_frame", lib.ptr(q), q.shape[0], lib.ptr(np.ascontiguousarray(T0, np.float32).reshape(16)),
             lib.ptr(T), lib.ptr(params), lib.ptr(losses), C.byref(it))
    assert it.value == iters
    return dict(T=T.reshape(4, 4), params=params, losses=losses, **_readback(lib, ctx, q.shape[0]))


def _runs(lib, m, q, T0, iters, scheme="geman_mcclure", sigma=0.3, k=K_NORMALS):
    """runs[j - 1] = register call with max_num_alignments = j on a fresh context holding map m."""
    runs = []
    for j in range(1, iters + 1):
        ctx = _context(lib, j, scheme, sigma, k)
        _insert(lib, ctx, m)
        runs.append(_register(lib, ctx, q, T0, j))
        ctx.close()
        if j > 1:  # determinism across contexts: the shared iterations give the same bits
            assert runs[-1]["losses"][:j - 1].tobytes() == runs[-2]["losses"].tobytes(), j
    return runs


def _fresh_normals(lib, m, idx, k=K_NORMALS):
    """Normals kd_normals_warp_kernel computes at the map points idx, in a fresh context (nn_search of the points)."""
    ctx = _context(lib, 1, k=k)
    _insert(lib, ctx, m)
    pts = np.ascontiguousarray(m[idx])
    nb, nrm = np.empty_like(pts), np.empty_like(pts)
    ctx.call("pls_kdmap_nn_search", lib.ptr(pts), pts.shape[0], lib.ptr(nb), lib.ptr(nrm), None)
    ctx.close()
    assert np.array_equal(nb, pts)
    return nrm


# ----------------------------------------------------------------------------------------------------------- checks
_POSITIONS = {}


def _positions(m):
    """kernel_sort_positions of map m (cached by the map's bytes)."""
    from oracle import kd_icp_reference
    key = (m.shape, hash(m.tobytes()))
    if key not in _POSITIONS:
        _POSITIONS[key] = kd_icp_reference.kernel_sort_positions(m)
    return _POSITIONS[key]


def _pose64(T):
    return np.asarray(T, np.float64).reshape(4, 4)


def _euler_round_trip(T):
    import torch
    from oracle import icp_oracle as orc
    prm = orc.from_pose_matrix(torch.from_numpy(T)[None])
    return orc.build_pose_matrix(prm)[0].numpy(), prm[0].numpy()


def _check_iteration(ref, m, tree, q, T_lin, run, scheme, sigma, min_normals_ok=0.9, tag="", k=K_NORMALS):
    """Iteration linearised at the float32 pose T_lin, read back in `run`.  Returns the distinct matched indices."""
    n = q.shape[0]
    T64 = _pose64(T_lin)
    p = ref.transform(T64, q)
    idx = run["idx"]
    m64 = m.astype(np.float64)
    assert (idx >= 0).all() and (idx < m.shape[0]).all(), tag
    assert np.array_equal(run["nb"], m[idx]), tag

    # 1. exact match.  The kernel transforms in float32: each coordinate of its p is the float64 p within 4 roundings
    # of partial sums bounded by s = |q|_1 + |t|_1, so |p32 - p| <= 4 sqrt(3) u s; an exact match for p32 is within
    # d1(p) + 2 |p32 - p| of p (plus the float32 distance comparison, relative 1e-6).
    d1, _ = tree.query(p, k=1, workers=-1)
    s = np.abs(q.astype(np.float64)).sum(1) + np.abs(T64[:3, 3]).sum()
    delta = 2 * 4 * np.sqrt(3) * U * s
    dm = np.linalg.norm(p - m64[idx], axis=1)
    bad = dm > d1 * (1 + 1e-6) + delta
    assert bad.sum() == 0, (tag, "queries whose match is not a nearest neighbour", int(bad.sum()), float((dm - d1)[bad].max()))

    # 2. runner-up bound, from the GPU's own stored position: every other map point is at least sqrt(second) away
    st = run["state"].astype(np.float64)
    dd, ii = tree.query(st[:, :3], k=2, workers=-1)
    d_other = np.where(ii[:, 0] == idx, dd[:, 1], dd[:, 0])
    bad = np.sqrt(st[:, 3]) > d_other * 1.00001 + 1e-6
    assert bad.sum() == 0, (tag, "runner-up bounds above the runner-up", int(bad.sum()),
                            float((np.sqrt(st[:, 3]) - d_other)[bad].max()))

    # 3. normals of every distinct matched point: the test_a9 bound against exact float64 normals, and, where the
    # point's (k+1)-NN list is not ambiguous in float32, tight_normal_bound against the float64 eigenvector of the
    # reference's float32 moments over that list (whichever kernel computed the normal: normals or refine kernel)
    u, first = np.unique(idx, return_index=True)
    gn = run["nrm"][first].astype(np.float64)
    assert np.abs(np.linalg.norm(gn, axis=1) - 1).max() <= 1e-6, tag
    nr, gap, uniq = ref.exact_normals(m, tree, u, k)
    sin = np.linalg.norm(np.cross(gn, nr), axis=1)
    ok = uniq & (gap > 1e-3)
    assert ok.mean() >= min_normals_ok, (tag, ok.mean())
    bad = sin[ok] > 2e-5 / gap[ok] + 2e-7
    assert bad.sum() == 0, (tag, "normals off the a9 bound", int(bad.sum()))
    lists, _, _, amb = ref.knn_lists(m, m[u], k, _positions(m), tree)
    covs = ref.reference_covs(m, u, lists, k).astype(np.float64)
    v = np.linalg.eigh(covs)[1][:, :, 0]
    bound, tgap = ref.tight_normal_bound(covs)
    tsin = np.linalg.norm(np.cross(gn, v), axis=1)
    sure = ~amb & (tgap > 1e-9)
    assert sure.mean() >= min_normals_ok, (tag, sure.mean())
    assert (tsin[sure] <= bound[sure]).all(), (tag, "normals off the tight bound", int((tsin[sure] > bound[sure]).sum()),
                                               float((tsin[sure] / bound[sure]).max()))

    # 4. accumulators: float64 sums of the GPU's own correspondences (its matches, its normals) within the float32
    # rounding of r, |p - q| and p x n (8 ulp of |p| + |q|) plus 1e-6 of sum |term|
    qm = m64[idx]
    nn = run["nrm"].astype(np.float64)
    sums = run["sums"]
    assert sums[29] == n, tag
    exact = ref.accumulate(p, qm, nn, scheme, sigma)
    e = 8 * 2 * U * (np.linalg.norm(p, axis=1) + np.linalg.norm(qm, axis=1))
    tol = ref.float32_tolerance(p, qm, nn, scheme, sigma, e)
    err = np.abs(sums - exact)
    assert (err <= tol).all(), (tag, "accumulators", np.nonzero(err > tol)[0], (err / tol).max())
    return u


def _check_pose_update(ref, T_lin, run, j):
    """losses[j-1] is sums[27] in float32; T_j is the float64 solve of the GPU's sums applied to T_lin through the Euler
    round trip, to float32 resolution."""
    sums = run["sums"]
    assert run["losses"][j - 1] == np.float32(sums[27])
    import torch
    from oracle import icp_oracle as orc
    dx = ref.gauss_newton_step(sums).astype(np.float32).astype(np.float64)  # the kernel applies the step in float32
    dT = orc.build_pose_matrix(torch.from_numpy(dx)[None])[0].numpy()
    T_exp, prm = _euler_round_trip(dT @ _pose64(T_lin))
    T = _pose64(run["T"])
    scale = 1 + np.abs(T_exp[:3, 3]).sum()
    assert np.abs(T[:3, :3] - T_exp[:3, :3]).max() <= 2e-6, np.abs(T[:3, :3] - T_exp[:3, :3]).max()
    assert np.abs(T[:3, 3] - T_exp[:3, 3]).max() <= 2e-6 * scale, np.abs(T[:3, 3] - T_exp[:3, 3]).max()
    assert np.abs(run["params"] - prm).max() <= 2e-6 * scale


def _check_runs(lib, ref, m, tree, q, T0, runs, scheme="geman_mcclure", sigma=0.3, min_normals_ok=0.9, tag="",
                k=K_NORMALS):
    """Every check on every iteration; returns per iteration the set of distinct matched points."""
    matched = []
    for j, run in enumerate(runs, start=1):
        T_lin = T0 if j == 1 else runs[j - 2]["T"]
        matched.append(_check_iteration(ref, m, tree, q, T_lin, run, scheme, sigma, min_normals_ok, f"{tag} it {j}", k))
        _check_pose_update(ref, T_lin, run, j)
    # normals computed in later iterations (inside the refine kernel or by the normals kernel) are the bits a fresh
    # context's nn_search computes at the same map points
    every = np.unique(np.concatenate(matched))
    fresh = _fresh_normals(lib, m, every, k)
    for j, (run, u) in enumerate(zip(runs, matched), start=1):
        rows = np.searchsorted(every, u)
        first = np.unique(run["idx"], return_index=True)[1]
        assert np.array_equal(run["nrm"][first].view(np.uint32), fresh[rows].view(np.uint32)), (tag, j)
    return matched


def _first_matched_late(matched):
    """Map points first matched in iteration 2 or later."""
    return np.setdiff1d(np.unique(np.concatenate(matched[1:])), matched[0]) if len(matched) > 1 else np.array([])


# -------------------------------------------------------------------------------------------------------- scenarios
_CFG2_RUNS = {}


def _cfg2_runs(lib, scene, k):
    """The cfg2 scenario's six register calls at num_neighbors_normals = k."""
    if k not in _CFG2_RUNS:
        _CFG2_RUNS[k] = _runs(lib, scene["m"], scene["q"], scene["T0"], 6, k=k)
    return _CFG2_RUNS[k]


@pytest.fixture(scope="module")
def cfg2_runs(lib, scene):
    return _cfg2_runs(lib, scene, K_NORMALS)


def test_cfg2_six_iterations_refine_kernel(lib, ref, scene, cfg2_runs):
    m, q = scene["m"], scene["q"]
    assert m.shape[0] < COLD_MAP_POINTS
    matched = _check_runs(lib, ref, m, scene["tree"], q, scene["T0"], cfg2_runs, tag="cfg2")
    changed = max(np.mean(a["idx"] != b["idx"]) for a, b in zip(cfg2_runs[:-1], cfg2_runs[1:]))
    assert changed >= 0.01, changed                       # later iterations really re-search
    assert len(_first_matched_late(matched)) >= 100       # ... and compute new normals


@pytest.mark.parametrize("k", [3, 31])
def test_cfg2_six_iterations_refine_kernel_at_other_k(lib, ref, scene, k):
    """The cfg2 scenario with the fewest and the most normal neighbours the map accepts: the normals of iterations 2-6
    come from kd_icp_refine_kernel's own (k+1)-NN searches and meet the tight bound like the first iteration's."""
    runs = _cfg2_runs(lib, scene, k)
    matched = _check_runs(lib, ref, scene["m"], scene["tree"], scene["q"], scene["T0"], runs, tag=f"cfg2 k={k}", k=k)
    assert len(_first_matched_late(matched)) >= 100
    # the normals differ from those at k = 10: the context's k reached the kernels
    base = _cfg2_runs(lib, scene, K_NORMALS)[0]
    assert not np.array_equal(runs[0]["nrm"], base["nrm"])


@pytest.mark.parametrize("scheme", SCHEMES)
def test_every_scheme_two_iterations(lib, ref, scene, scheme):
    sigma = 0.5 if scheme == "default" else 0.3
    runs = _runs(lib, scene["m"], scene["q"], scene["T0"], 2, scheme, sigma)
    _check_runs(lib, ref, scene["m"], scene["tree"], scene["q"], scene["T0"], runs, scheme, sigma, tag=scheme)


def test_refine_kernel_rounds_beyond_the_first(lib, ref, scene):
    """An unsubsampled 128x4096 scan: more queries than the refine kernel's blocks take in one round."""
    q = scene["dense"]
    assert q.shape[0] > REFINE_ROUND and scene["m"].shape[0] < COLD_MAP_POINTS
    runs = _runs(lib, scene["m"], q, scene["T0"], 3)
    _check_runs(lib, ref, scene["m"], scene["tree"], q, scene["T0"], runs, tag="dense")
    late = np.arange(q.shape[0]) >= REFINE_ROUND
    assert (runs[1]["idx"][late] != runs[0]["idx"][late]).any()   # the second round had matches to change


def _filler(scene, runs, need, seed=5, k=K_NORMALS):
    """Points strictly inside the scene map's bounding box, clear of every query (at every pose the runs linearised
    at) by more than its match distance and of every matched point by more than its 11th neighbour: they change no
    match and no normal."""
    m, tree, q = scene["m"], scene["tree"], scene["q"]
    m64 = m.astype(np.float64)
    poses = [scene["T0"]] + [r["T"] for r in runs[:-1]]
    centres, radii = [], []
    for T in poses:
        p = _pose64_transform(T, q)
        d1, _ = tree.query(p, k=1, workers=-1)
        centres.append(p)
        radii.append(d1 * 1.001 + 0.01)
    matched = np.unique(np.concatenate([r["idx"] for r in runs]))
    r12, _ = tree.query(m64[matched], k=k + 2, workers=-1)
    centres.append(m64[matched])
    radii.append(r12[:, -1] * 1.001 + 0.01)
    centres, radii = np.concatenate(centres), np.concatenate(radii)
    lo, hi = m.min(0).astype(np.float64), m.max(0).astype(np.float64)
    margin = 1e-3 * (hi - lo)
    rng = np.random.RandomState(seed)
    cand = rng.uniform(lo + margin, hi - margin, (int(need * 1.6), 3)).astype(np.float32)
    ctree = cKDTree(cand.astype(np.float64))
    bad = np.zeros(cand.shape[0], bool)
    for hits in ctree.query_ball_point(centres, radii, workers=-1):
        bad[hits] = True
    keep = cand[~bad]
    assert keep.shape[0] >= need, (keep.shape[0], need)
    return np.ascontiguousarray(keep[:need]), centres, radii


def _pose64_transform(T, pts):
    T = _pose64(T)
    return pts.astype(np.float64) @ T[:3, :3].T + T[:3, 3]


def test_four_launch_path_on_a_filled_map(lib, ref, scene, cfg2_runs):
    """The cfg2 map filled to >= 2 M points with points that change no match and no normal: the later iterations run
    as verify / queued 1-NN / normals / residual, and give the bits the refine kernel gives on the unfilled map (the
    same bounding box keeps the quantisation and the relative sorted order of the scene points, so ties resolve
    alike)."""
    _four_launch_path(lib, ref, scene, cfg2_runs, K_NORMALS)


def test_four_launch_path_on_a_filled_map_at_k31(lib, ref, scene):
    """The same with 31 normal neighbours: the filler keeps clear of every matched point's 32nd neighbour."""
    _four_launch_path(lib, ref, scene, _cfg2_runs(lib, scene, 31), 31)


def _four_launch_path(lib, ref, scene, cfg2_runs, k):
    m = scene["m"]
    unfilled = cfg2_runs[:4]
    fill, centres, radii = _filler(scene, unfilled, COLD_MAP_POINTS - m.shape[0] + 1000, k=k)
    big = np.ascontiguousarray(np.concatenate([m, fill]))
    assert big.shape[0] >= COLD_MAP_POINTS
    assert (big.min(0) == m.min(0)).all() and (big.max(0) == m.max(0)).all()
    runs = _runs(lib, big, scene["q"], scene["T0"], 4, k=k)
    for j, (a, b) in enumerate(zip(runs, unfilled), start=1):
        for key in ("T", "params", "losses", "idx", "nrm", "sums"):
            assert a[key].tobytes() == b[key].tobytes(), (j, key)
    # filler clearance at the poses the filled runs linearised at (the same bits as the unfilled ones)
    ftree = cKDTree(fill.astype(np.float64))
    df, _ = ftree.query(centres, k=1, workers=-1)
    assert (df > radii).all()
    _check_runs(lib, ref, big, cKDTree(big.astype(np.float64)), scene["q"], scene["T0"], runs, tag=f"filled k={k}", k=k)


def test_later_iterations_across_an_overflowed_level(lib, ref):
    from test_kd_overflow_gpu import _map, _table_cells
    m = _map(0)
    levels = _table_cells(m, local_map_size=1)
    assert levels[0][0] <= levels[0][1] // 2
    assert any(cells > slots for cells, slots in levels[1:]), levels
    rng = np.random.RandomState(11)
    d = rng.randn(*m.shape)
    q = (m + d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.05, 0.5, (m.shape[0], 1))).astype(np.float32)
    T0 = _perturbed(np.eye(4), 0.05, 0.5, 1)
    runs = _runs(lib, m, q, T0, 4)
    matched = _check_runs(lib, ref, m, cKDTree(m.astype(np.float64)), q, T0, runs, tag="overflow")
    assert max(np.mean(a["idx"] != b["idx"]) for a, b in zip(runs[:-1], runs[1:])) > 0
    assert len(matched[0]) > 0


def _on_level0_faces(m, pts):
    """pts with x moved onto a level-0 cell face, as the index quantises it ((x - min) * scale a multiple of 8)."""
    mn = m.min(0)
    ext = np.float32(max(float((m.max(0) - mn).max()), 1e-6))
    scale = min(np.float32(8) / np.float32(0.2), np.float32(8191) / ext)
    out = []
    for p in pts:
        k = np.floor(np.float32(p[0] - mn[0]) * scale / 8)
        x = np.float32(mn[0] + np.float64(8 * k) / np.float64(scale))
        for _ in range(64):
            u = np.float32(np.float32(x - mn[0]) * scale)
            if u == 8 * k:
                out.append([x, p[1], p[2]])
                break
            x = np.nextafter(x, np.float32(np.inf) if u < 8 * k else np.float32(-np.inf))
    return np.asarray(out, np.float32)


def test_queries_outside_the_map_and_on_cell_faces(lib, ref, scene):
    m = scene["m"]
    rng = np.random.RandomState(12)
    base = _pose64_transform(scene["T_gt"], scene["q"]).astype(np.float32)     # registered already: T0 = identity
    lo, hi = m.min(0), m.max(0)
    n_out = base.shape[0] // 20
    # scene queries moved 20-300 m beyond a vertical face of the box (x or y, either side)
    outside = base[rng.choice(base.shape[0], n_out, replace=False)].copy()
    axis, side = rng.randint(0, 2, n_out), rng.randint(0, 2, n_out).astype(bool)
    far = rng.uniform(20, 300, n_out).astype(np.float32)
    rows = np.arange(n_out)
    outside[rows, axis] = np.where(side, hi[axis] + far, lo[axis] - far)
    faces = _on_level0_faces(m, m[rng.choice(m.shape[0], 2000, replace=False)])
    q = np.ascontiguousarray(np.concatenate([base, outside, faces]))
    gap_out = np.maximum(lo - outside, outside - hi).max(1)
    assert (gap_out >= 19.9).all() and faces.shape[0] >= 1000
    T0 = np.eye(4, dtype=np.float32)
    runs = _runs(lib, m, q, T0, 3)
    _check_runs(lib, ref, m, scene["tree"], q, T0, runs, tag="outside")
    sl = slice(base.shape[0], base.shape[0] + n_out)
    assert all((r["idx"][sl] >= 0).sum() == n_out for r in runs)   # every outside query is matched


def test_ties_between_duplicates_and_lattice_neighbours(lib, ref):
    """A lattice on three orthogonal planes (well-defined normals, a regular system) plus exact duplicates; queries
    half-way between lattice neighbours: ties whose runner-up is the tie distance, so the match is never proven."""
    g = np.arange(-20, 21) * 0.5
    a, b = np.meshgrid(g, g, indexing="ij")
    a, b = a.ravel(), b.ravel()
    z = np.zeros_like(a)
    lattice = np.concatenate([np.stack([a, b, z - 10.0], 1), np.stack([a, z - 10.0, b], 1), np.stack([z - 10.0, a, b], 1)])
    rng = np.random.RandomState(13)
    m = np.concatenate([lattice, lattice[rng.choice(lattice.shape[0], lattice.shape[0] // 10, replace=False)]])
    m = np.ascontiguousarray(m.astype(np.float32))
    sel = rng.choice(lattice.shape[0], 4000, replace=False)
    q = lattice[sel].copy()
    plane = np.argmin(np.abs(q - (-10.0)), axis=1)                          # the coordinate fixed at -10
    inplane = (plane + 1) % 3
    q[np.arange(len(q)), inplane] += 0.25                                   # half-way between two neighbours
    q[np.arange(len(q)), plane] += 0.1                                      # off the plane: a residual to solve
    q = np.ascontiguousarray(q.astype(np.float32))
    T0 = np.eye(4, dtype=np.float32)
    runs = _runs(lib, m, q, T0, 3)
    tree = cKDTree(m.astype(np.float64))
    _check_runs(lib, ref, m, tree, q, T0, runs, min_normals_ok=0.0, tag="ties")
    # iteration 1 runs at the identity: the kernel's query positions are the queries themselves
    d, _ = tree.query(q.astype(np.float64), k=2)
    ties = d[:, 0] == d[:, 1]
    assert ties.sum() >= 1
    # the runner-up bound of a tie is the tie distance: the next iteration cannot prove the match, it searches again
    st = runs[0]["state"].astype(np.float64)
    assert np.array_equal(st[:, :3], q.astype(np.float64))
    assert (np.sqrt(st[ties, 3]) <= d[ties, 0] * (1 + 1e-6)).all()


def test_warm_normal_cache_gives_the_same_bits(lib, scene):
    ctx = _context(lib, 6)
    _insert(lib, ctx, scene["m"])
    a = _register(lib, ctx, scene["q"], scene["T0"], 6)
    b = _register(lib, ctx, scene["q"], scene["T0"], 6)     # every normal it needs is cached now
    ctx.close()
    for key in ("T", "params", "losses", "idx", "nrm", "state", "sums"):
        assert a[key].tobytes() == b[key].tobytes(), key


def test_readback_refuses_a_rebuilt_map(lib, scene):
    ctx = _context(lib, 2)
    n = scene["q"].shape[0]
    with pytest.raises(RuntimeError, match="no kd search"):
        ctx.call("pls_kdmap_last_correspondences", n, None, None, None, None, None)
    _insert(lib, ctx, scene["m"])
    _register(lib, ctx, scene["q"], scene["T0"], 2)
    with pytest.raises(AssertionError, match="query count"):
        ctx.call("pls_kdmap_last_correspondences", n + 1, None, None, None, None, None)
    _insert(lib, ctx, scene["m"][:1000])
    with pytest.raises(RuntimeError, match="rebuilt"):
        ctx.call("pls_kdmap_last_correspondences", n, None, None, None, None, None)
    ctx.close()
