"""Every projective ICP iteration against a float64 reference (oracle/proj_icp_reference.py), through its accumulators.

The projective iteration is proj_icp_tma_kernel when H*W is a multiple of 128 (and PLS_PROJ_NO_TMA is unset), else
proj_icp_iter_kernel.  A pose moves by far less than the pose tolerances of the other tests when a few hundred pixels
take the wrong candidate, so here every iteration is checked through the 30 accumulators of its last iteration
(pls_last_icp_sums) against float64 sums of the same model (pls_projmap_model, the GPU's own bits):

  * the count must match exactly where no query or pixel is ambiguous, the other 29 sums within float32 rounding plus
    the spread of the ambiguous choices, and the returned pose must be the float64 solve of the GPU's sums;
  * constructed probes put chosen candidates at chosen pixels (exact ties, the 2^-21 band of the squared-distance
    arg-min, the TMA / direct-load split, null candidates, tile edges, z-buffer ties) so that one wrong choice moves
    sum r^2 by at least 100 times its tolerance;
  * the model rebuild is compared per pixel with a float64 rebuild.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
UP, DOWN = 3.0, -24.0
U = 2.0 ** -24
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
KS = [1, 2, 4, 5, 16, 17, 20]
TMA_SHAPES = [(16, 512), (64, 2048), (128, 4096)]
FALLBACK_SHAPES = [(33, 500), (64, 2047)]
# projmap.cu's launch constants
PT_TILE, NUM_SMS, KDIRECT_MAX, PT_STAGES = 128, 132, 10, 3
PROBE_K = 20
Q = 2.0 ** -14          # grid of the probe coordinates: every difference, square and partial sum is exact in float32


def _lib():
    from pylidar_slam_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def lib():
    return _lib()


@pytest.fixture(scope="module")
def pref():
    from oracle import proj_icp_reference
    return proj_icp_reference


@pytest.fixture(scope="module")
def kdr():
    from oracle import kd_icp_reference
    return kd_icp_reference


# ---------------------------------------------------------------------------------------------------------- driving
def _context(lib, H, W, kcap, iters=1, scheme="geman_mcclure", sigma=0.3):
    return lib.Context(height=H, width=W, up_fov_deg=UP, down_fov_deg=DOWN, local_map_type=lib.MAP_PROJECTIVE,
                       local_map_size=kcap, scheme=lib.SCHEMES[scheme], sigma=sigma, gn_max_iters=1,
                       max_num_alignments=iters, threshold_delta_pose=0.0)


def _update(lib, ctx, rel, vm):
    rel = np.ascontiguousarray(rel, np.float32).reshape(16)
    ctx.call("pls_projmap_update", lib.ptr(rel), None if vm is None else lib.ptr(np.ascontiguousarray(vm, np.float32)))


def _model(lib, ctx, H, W):
    k = C.c_int(0)
    ctx.call("pls_projmap_num_frames", C.byref(k))
    v = np.empty((k.value, 3, H, W), np.float32)
    n = np.empty_like(v)
    ctx.call("pls_projmap_model", lib.ptr(v), lib.ptr(n))
    return v, n


def _last_sums(lib, ctx):
    s, it = np.empty(30, np.float64), C.c_int(-1)
    ctx.call("pls_last_icp_sums", lib.ptr(s), C.byref(it))
    return s, it.value


def _register(lib, ctx, q, T0, iters):
    T, params, losses, it = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(iters, np.float32), C.c_int(0)
    ctx.call("pls_register_frame", lib.ptr(q), q.shape[0], lib.ptr(np.ascontiguousarray(T0, np.float32).reshape(16)),
             lib.ptr(T), lib.ptr(params), lib.ptr(losses), C.byref(it))
    assert it.value == iters
    sums, it2 = _last_sums(lib, ctx)
    assert it2 == iters
    return dict(T=T.reshape(4, 4), params=params, losses=losses, sums=sums)


def _perturbed(T, metres, degrees, seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    axis, d = rng.randn(3), rng.randn(3)
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(degrees)).as_matrix()
    P[:3, 3] = d / np.linalg.norm(d) * metres
    return (np.asarray(T, np.float64) @ P).astype(np.float32)


_FRAMES = {}


def _frames(H, W, n=21):
    """Synthetic vertex maps [n,3,H,W] and relative poses [n,4,4] (float32) of frames 0..n-1."""
    key = (H, W, n)
    if key not in _FRAMES:
        from pylidar_slam_b200 import synthetic as syn
        vms = np.stack([syn.vertex_map_from_scan(syn.scan(k, H, W), H, W)[0] for k in range(n)])
        rels = np.stack([np.eye(4, dtype=np.float32)] + [syn.gt_relative_pose(k).astype(np.float32) for k in range(1, n)])
        _FRAMES.clear()
        _FRAMES[key] = (vms, rels)
    return _FRAMES[key]


def _queries(H, W, k):
    from pylidar_slam_b200 import synthetic as syn
    return np.ascontiguousarray(syn.scan(k, H, W))


# ----------------------------------------------------------------------------------------------------------- checks
def _check_sums(pref, mv, mn, q, T, sums, scheme="geman_mcclure", sigma=0.3, tag="", min_count=1):
    out = pref.proj_icp_iteration(mv, mn, q, T, scheme, sigma, UP, DOWN)
    exact = out["sums"]
    if out["count_tol"] == 0:
        assert sums[29] == exact[29], (tag, sums[29], exact[29])
    else:
        assert abs(sums[29] - exact[29]) <= out["count_tol"], (tag, sums[29], exact[29], out["count_tol"])
    assert sums[29] >= min_count, (tag, sums[29])
    err = np.abs(sums[:29] - exact[:29])
    tol = out["tol"][:29]
    assert (err <= tol).all(), (tag, "accumulators", np.nonzero(err > tol)[0], float((err / tol).max()))
    return out


def _check_pose(kdr, T_lin, run):
    """The returned pose is the float64 solve of the GPU's sums (the kd test's check)."""
    from test_kd_icp_iterations_gpu import _check_pose_update
    _check_pose_update(kdr, T_lin, run, 1)


def _blocks(H, W, K, kdirect=4, stages=2, no_tma=False):
    """projmap_icp_iteration's launch geometry: (TMA path, ktma, blocks)."""
    hw = H * W
    kd = max(0, min(kdirect, KDIRECT_MAX))
    if kd > K - 1:
        kd = K - 1 if K > 1 else 0
    ktma = K - kd
    stage_bytes = (ktma * 3 + 4) * PT_TILE * 4
    use = not no_tma and hw % PT_TILE == 0 and 1 <= stages <= PT_STAGES and stage_bytes * stages <= 200 * 1024
    if not use:
        b = (hw + 255) // 256
        return False, ktma, max(1, min(b, 4 * NUM_SMS))
    per_sm = max(1, min(8, (220 * 1024) // (stage_bytes * stages + 2048)))
    tiles = hw // PT_TILE
    per_cta = -(-tiles // (per_sm * NUM_SMS))
    return True, ktma, max(1, -(-tiles // per_cta))


# ---------------------------------------------------------------------------------------------- a. model rebuild
def test_model_rebuild_per_pixel(lib, pref):
    """Fill to K = local_map_size, evict, one move-only update: every pixel of every model frame after every update."""
    from pylidar_slam_b200 import common
    H, W, kcap = 64, 2048, 5
    vms, rels = _frames(H, W)
    nms = common.compute_normal_map(np.ascontiguousarray(vms[:kcap + 2]))
    ctx = _context(lib, H, W, kcap)
    held = []     # [frame index, float64 pose frame -> newest, compositions]
    for step in range(kcap + 2):
        move_only = step == kcap + 1
        rel = rels[step]
        _update(lib, ctx, rel, None if move_only else vms[step])
        inv = np.linalg.inv(rel.astype(np.float64))
        held = [[f, inv @ P if step else P, m + 1] for f, P, m in held]
        if not move_only:
            held.append([step, np.eye(4), 0])
        held = held[-kcap:]
        mv, mn = _model(lib, ctx, H, W)
        assert mv.shape[0] == len(held)
        idx = [f for f, _, _ in held]
        V, N, occ, amb, err = pref.rebuild_model(vms[idx], nms[idx], np.stack([P for _, P, _ in held]),
                                                 [16 * U * (m + 1) for _, _, m in held], H, W, UP, DOWN)
        got = np.abs(mv).max(1) > 0
        sure = ~amb
        assert sure.mean() > 0.9, (step, sure.mean())
        bad = sure & (got != occ)
        assert not bad.any(), (step, "occupancy", np.argwhere(bad)[:5])
        both = sure & occ
        dv = np.abs(mv.astype(np.float64) - V).max(1)
        assert (dv[both] <= err[both]).all(), (step, "vertices", float((dv[both] / err[both]).max()))
        en = np.array([16 * U * (m + 1) for _, _, m in held])[:, None, None] * np.abs(N).sum(1) + 4 * U
        dn = np.abs(mn.astype(np.float64) - N).max(1)
        assert (dn[both] <= en[both]).all(), (step, "normals", float((dn[both] / en[both]).max()))
        assert (mn[~np.broadcast_to(got[:, None], mn.shape)] == 0).all()
    ctx.close()


# ------------------------------------------------------------------------------------- b/c. iteration accumulators
def _filled(lib, H, W, kcap, K, iters=1, scheme="geman_mcclure", sigma=0.3):
    vms, rels = _frames(H, W)
    ctx = _context(lib, H, W, kcap, iters, scheme, sigma)
    for k in range(K):
        _update(lib, ctx, rels[k], vms[k])
    return ctx


@pytest.mark.parametrize("H,W", TMA_SHAPES + FALLBACK_SHAPES)
def test_first_iteration_every_k(lib, pref, kdr, H, W):
    """K = 1 ... 20 candidates, the model's tile stride local_map_size = 20 (above K) and = K; T0 = identity."""
    vms, rels = _frames(H, W)
    q = _queries(H, W, 20)
    ctx20 = _context(lib, H, W, 20)
    done = 0
    for K in KS:
        while done < K:
            _update(lib, ctx20, rels[done], vms[done])
            done += 1
        for kcap in sorted({20, K}):
            ctx = ctx20 if kcap == 20 else _filled(lib, H, W, kcap, K)
            mv, mn = _model(lib, ctx, H, W)
            assert mv.shape[0] == K
            run = _register(lib, ctx, q, np.eye(4, dtype=np.float32), 1)
            _check_sums(pref, mv, mn, q, np.eye(4, dtype=np.float32), run["sums"], tag=(H, W, K, kcap),
                        min_count=0.3 * H * W)
            _check_pose(kdr, np.eye(4, dtype=np.float32), run)
            if ctx is not ctx20:
                ctx.close()
    ctx20.close()


@pytest.mark.parametrize("H,W", [(128, 4096), (33, 500)])
def test_first_iteration_from_a_perturbed_pose(lib, pref, kdr, H, W):
    """T0 = the ground truth perturbed by 0.3 m / 1 degree: the transform is inexact, queries leave pixel centres."""
    from pylidar_slam_b200 import synthetic as syn
    ctx = _filled(lib, H, W, 20, 20)
    mv, mn = _model(lib, ctx, H, W)
    q = _queries(H, W, 20)
    T0 = _perturbed(syn.gt_relative_pose(20), 0.3, 1.0, 0)
    run = _register(lib, ctx, q, T0, 1)
    out = _check_sums(pref, mv, mn, q, T0, run["sums"], tag=(H, W), min_count=0.3 * H * W)
    assert out["count_tol"] < 0.05 * run["sums"][29]
    _check_pose(kdr, T0, run)
    ctx.close()


@pytest.mark.parametrize("scheme", SCHEMES)
def test_every_scheme(lib, pref, kdr, scheme):
    from pylidar_slam_b200 import synthetic as syn
    sigma = 0.5 if scheme == "default" else 0.3
    H, W = 16, 512
    ctx = _filled(lib, H, W, 20, 20, 1, scheme, sigma)
    mv, mn = _model(lib, ctx, H, W)
    q = _queries(H, W, 20)
    for T0 in (np.eye(4, dtype=np.float32), _perturbed(syn.gt_relative_pose(20), 0.3, 1.0, 0)):
        run = _register(lib, ctx, q, T0, 1)
        _check_sums(pref, mv, mn, q, T0, run["sums"], scheme, sigma, tag=scheme, min_count=0.3 * H * W)
        _check_pose(kdr, T0, run)
    ctx.close()


@pytest.mark.parametrize("H,W", [(64, 2048), (64, 2047)])
def test_last_of_several_iterations_is_a_fresh_first(lib, pref, H, W):
    """Iteration J of one frame (threshold_delta_pose = 0) gives the bits of a one-iteration frame from the pose
    iteration J - 1 returned: later iterations start from the z-buffer the previous resolve left clean."""
    from pylidar_slam_b200 import synthetic as syn
    J = 4
    q = _queries(H, W, 20)
    T0 = _perturbed(syn.gt_relative_pose(20), 0.3, 1.0, 0)
    runs = {}
    for iters in (J, J - 1):
        ctx = _filled(lib, H, W, 20, 20, iters)
        runs[iters] = _register(lib, ctx, q, T0, iters)
        ctx.close()
    assert runs[J]["losses"][:J - 1].tobytes() == runs[J - 1]["losses"].tobytes()
    ctx = _filled(lib, H, W, 20, 20, 1)
    mv, mn = _model(lib, ctx, H, W)
    one = _register(lib, ctx, q, runs[J - 1]["T"], 1)
    ctx.close()
    assert one["sums"].tobytes() == runs[J]["sums"].tobytes()
    _check_sums(pref, mv, mn, q, runs[J - 1]["T"], runs[J]["sums"], tag="iteration J", min_count=0.3 * H * W)


@pytest.mark.parametrize("H,W", [(64, 2048), (33, 500)])
def test_process_frame_vertex_map_queries(lib, pref, H, W):
    """pls_process_frame with the vertex-map layout: the queries are the frame's non-null pixels.  The model the frame
    searches is the one after the previous frame's (deferred) map update: exported before the frame."""
    vms, _ = _frames(H, W)
    ctx = _context(lib, H, W, 20)
    pose, params, has, info = np.zeros(16, np.float32), np.zeros(6, np.float32), C.c_int(0), np.zeros(12)
    with pytest.raises(RuntimeError, match="no ICP frame"):
        _last_sums(lib, ctx)
    checked = 0
    for k in range(6):
        vm = np.ascontiguousarray(vms[k])
        if k > 0:
            mv, mn = _model(lib, ctx, H, W)
        ctx.call("pls_process_frame", lib.ptr(vm), lib.INPUT_VERTEX_MAP, 0, None, lib.ptr(pose), lib.ptr(params),
                 C.byref(has), lib.ptr(info))
        if k == 0:
            with pytest.raises(RuntimeError, match="no ICP frame"):
                _last_sums(lib, ctx)
            continue
        sums, it = _last_sums(lib, ctx)
        assert it == 1 and info[0] == 1
        pts = vm.reshape(3, -1).T
        q = np.ascontiguousarray(pts[np.linalg.norm(pts, axis=1) > 0])
        assert info[2] == q.shape[0]
        _check_sums(pref, mv, mn, q, np.eye(4, dtype=np.float32), sums, tag=("frame", k), min_count=0.3 * H * W)
        checked += 1
    assert checked == 5
    ctx.close()


# ------------------------------------------------------------------------------------------- d. constructed probes
def _direction(H, W, row, col):
    theta = (2.0 * col / W - 1.0) * np.pi
    up, down = abs(UP) / 180 * np.pi, abs(DOWN) / 180 * np.pi
    phi = (1.0 - row / H) * (up + down) - down
    return np.array([np.cos(phi) * np.cos(-theta), np.cos(phi) * np.sin(-theta), np.sin(phi)])


def _grid(x):
    return np.round(np.asarray(x, np.float64) / Q) * Q


def _root32(n2):
    """float32 root of the (exact) squared length n2 Q^2."""
    return np.float32(np.sqrt(float(n2)) * Q)


def _band_pair(m0, equal_roots):
    """Integer vectors a, b near m0 (units of Q) with |b|^2 < |a|^2 inside the kernel's 2^-21 band of the squares, and
    equal (or, otherwise, different) float32 roots."""
    r = np.arange(-20, 21)
    cand = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3) + m0
    n2 = (cand.astype(np.int64) ** 2).sum(1)
    assert n2.max() < 2 ** 24
    order = np.argsort(n2, kind="stable")
    lo, hi = order[:-1], order[1:]                      # neighbours in squared length: b = lo, a = hi
    best2 = (n2[hi] * Q * Q).astype(np.float32)
    d2 = (n2[lo] * Q * Q).astype(np.float32)
    thr = best2 * np.float32(0.99999952)
    band = (d2 < best2) & ~(d2 < thr)
    same = np.array([_root32(x) == _root32(y) for x, y in zip(n2[lo], n2[hi])])
    hit = np.nonzero(band & (same == equal_roots))[0]
    assert hit.shape[0] > 0, "no band pair"
    return cand[hi[hit[0]]], cand[lo[hit[0]]]


def _tie_pair(m0):
    """Two different integer vectors near m0 (units of Q) with the same squared length."""
    r = np.arange(-20, 21)
    cand = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3) + m0
    n2 = (cand.astype(np.int64) ** 2).sum(1)
    assert n2.max() < 2 ** 24
    order = np.argsort(n2, kind="stable")
    hit = np.nonzero(n2[order[1:]] == n2[order[:-1]])[0]
    assert hit.shape[0] > 0, "no tie"
    return cand[order[hit[0]]], cand[order[hit[0] + 1]]


def _zbuffer_tie(H, W, avoid=()):
    """Two queries on the 1/16 m grid with equal (exact) squared range that project to one pixel."""
    import torch
    from oracle import icp_oracle as orc
    pj = orc.Projector(H, W, UP, DOWN)
    for x in range(150, 200):
        for y in range(-40, 40):
            z = y + 1
            a = np.array([[x, y, z], [x, z, y]], np.float64) / 16
            row, col = pj.pixels(torch.from_numpy(a)[None])
            row, col = row[0].numpy(), col[0].numpy()
            pr, pc = np.rint(row), np.rint(col)
            if pr[0] != pr[1] or pc[0] != pc[1] or not (0 <= pr[0] <= H - 1 and 1 <= pc[0] <= W - 2):
                continue
            if (np.abs(row - pr) > 0.45).any() or (np.abs(col - pc) > 0.45).any():
                continue
            if any(abs(pr[0] - c // W) <= 2 and abs(pc[0] - c % W) <= 2 for c in avoid):
                continue
            return a.astype(np.float32), int(pr[0] * W + pc[0])
    raise AssertionError("no z-buffer tie")


def probe_scene(H, W, K=PROBE_K, kdirect=4):
    """Vertex maps [K,3,H,W] (identity poses), queries [M,3] and the probes: (name, pixel, expected k or -1, wrong k or
    None).  Each frame is a smooth surface of its own.  At a probe pixel only the listed candidates are live, each the
    centre of a 5x5 window on a plane of its own: the expected one faces the sensor, the others are tilted by 60
    degrees, so that the wrong choice changes the residual by about half the candidate's distance."""
    ktma = K - min(kdirect, K - 1)
    rows, cols = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    theta = (2.0 * cols / W - 1.0) * np.pi
    up, down = abs(UP) / 180 * np.pi, abs(DOWN) / 180 * np.pi
    phi = (1.0 - rows / H) * (up + down) - down
    d = np.stack([np.cos(phi) * np.cos(-theta), np.cos(phi) * np.sin(-theta), np.sin(phi)])
    vms = np.empty((K, 3, H, W), np.float32)
    for k in range(K):
        rng = 9.0 + 0.25 * k + 1.5 * np.sin(theta * (1 + k % 4) + 0.7 * k) + 0.08 * (k % 5) * rows
        vms[k] = (d * rng).astype(np.float32)
    probes, queries, centres = [], [], set()
    hw = H * W
    r0 = 6.0

    def window(k, i, centre, n):
        row, col = divmod(i, W)
        for rr in range(max(0, row - 2), min(H, row + 3)):
            for cc in range(max(0, col - 2), min(W, col + 3)):
                j = rr * W + cc
                if j in centres and j != i:
                    continue
                ray = _direction(H, W, rr, cc)
                vms[k, :, rr, cc] = (ray * (n @ centre) / (n @ ray)).astype(np.float32)
        vms[k, :, row, col] = centre.astype(np.float32)

    def cell(i, live, name, want, wrong):
        row, col = divmod(i, W)
        ray = _direction(H, W, row, col)
        p = _grid(r0 * ray)
        side = np.cross(ray, [0.0, 0.0, 1.0])
        side /= np.linalg.norm(side)
        tilted = 0.5 * ray + np.sqrt(0.75) * side
        centres.add(i)
        vms[:, :, row, col] = 0
        for k, off in live.items():
            window(k, i, p + off, ray if k == want else tilted)
        probes.append((name, i, want, wrong))
        queries.append(p.astype(np.float32))

    def radial(i, metres):
        return _grid(metres * _direction(H, W, *divmod(i, W)))

    def near_radial(i, metres):
        return np.round(metres * _direction(H, W, *divmod(i, W)) / Q).astype(np.int64)

    mid, c0 = H // 2, W // 2

    def pick(row):
        return row * W + c0 - 60 + 9 * len(probes)

    # exact ties: |a| = |b| on the dyadic grid, the first candidate wins (inside the TMA range, inside the direct range,
    # straddling ktma)
    for name, (ka, kb) in (("tie_tma", (1, ktma - 2)), ("tie_direct", (ktma, K - 1)), ("tie_straddle", (ktma - 1, ktma))):
        if ka >= kb or kb >= K or ka < 0:
            continue
        i = pick(mid)
        ta, tb = _tie_pair(near_radial(i, 0.15))
        cell(i, {ka: ta * Q, kb: tb * Q}, name, ka, kb)
    # the 2^-21 band: squares within 2^-21 relative, with equal roots (the first wins) and different roots (the later
    # wins: only the redo with the roots finds it, for a direct candidate too)
    for name, ka, kb, equal in (("band_equal_roots", 2, min(7, K - 1), True), ("band_diff_roots", 2, min(7, K - 1), False),
                                ("band_direct_redo", 3, K - 1, False)):
        if ka >= kb:
            continue
        i = pick(mid - 1)
        va, vb = _band_pair(near_radial(i, 0.2), equal)
        cell(i, {ka: va * Q, kb: vb * Q}, name, ka if equal else kb, kb if equal else ka)
    # where the winner sits: only in the direct range; null candidates between live ones; no live candidate at all
    i = pick(mid + 1)
    cell(i, {0: radial(i, 0.6), K - 1: np.array([40, -70, 90]) * Q}, "nearest_direct", K - 1, 0)
    if K >= 3:
        i = pick(mid + 1)
        cell(i, {0: radial(i, 0.7), K // 2: np.array([-60, 30, 80]) * Q}, "nulls_between", K // 2, 0)
    i = pick(mid + 1)
    cell(i, {}, "all_null", -1, None)
    # positions: the last / first pixel of adjacent tiles, the last tile, the last pixel
    for name, i in (("tile_end", PT_TILE - 1), ("tile_start", PT_TILE), ("tile_end_2", 2 * PT_TILE - 1),
                    ("last_tile_start", (hw // PT_TILE - 1) * PT_TILE if hw % PT_TILE == 0 else hw - 100),
                    ("last_pixel", hw - 1)):
        if i % W == 0:
            i += 1
        if i in centres:
            continue
        kn = K - 1 if len(probes) % 2 else 0
        live = {kn: np.array([70, 20, -50]) * Q}
        kf = 0 if kn == K - 1 else K - 1
        if kf != kn:
            live[kf] = radial(i, 0.5)
        cell(i, live, name, kn, kf if kf != kn else None)
    # two queries in one pixel at equal range: the lower index wins
    pair, i = _zbuffer_tie(H, W, centres)
    row, col = divmod(i, W)
    centres.add(i)
    vms[:, :, row, col] = 0
    # the candidate is the first query itself, on a plane whose normal leans towards the second query
    a, b = pair.astype(np.float64)
    ray = _direction(H, W, *divmod(i, W))
    nrm = ray + 3 * (b - a) / np.linalg.norm(b - a)
    window(K // 3, i, a, nrm / np.linalg.norm(nrm))
    n = len(queries)
    queries += [pair[0], pair[1]]
    probes.append(("zbuffer_tie", i, K // 3, None))
    probes.append(("zbuffer_tie_query", n, None, n + 1))
    return np.ascontiguousarray(vms), np.ascontiguousarray(np.stack(queries).astype(np.float32)), probes


def _check_probes(pref, kdr, mv, mn, q, probes, sums, tag):
    """The reference picks what each probe expects, nothing in a probe is ambiguous, the GPU meets it, and the wrong
    choice would move sum r^2 far beyond the tolerance."""
    I = np.eye(4, dtype=np.float32)
    out = _check_sums(pref, mv, mn, q, I, sums, "geman_mcclure", 0.3, tag=tag)
    assert out["count_tol"] == 0 and not out["amb_pixel"].any(), tag
    K = mv.shape[0]
    flat_v, flat_n = mv.reshape(K, 3, -1), mn.reshape(K, 3, -1)
    for name, i, want, wrong in probes:
        if name == "zbuffer_tie_query":
            continue
        assert out["k"][i] == want, (tag, name, out["k"][i], want)
        if wrong is None:
            continue
        p = out["p"][out["win"][i]][None]
        t = [kdr.terms(p, flat_v[k, :, i][None].astype(np.float64), flat_n[k, :, i][None].astype(np.float64),
                       "geman_mcclure", 0.3)[0][28] for k in (want, wrong)]
        assert abs(t[0] - t[1]) >= 100 * out["tol"][28], (tag, name, t, out["tol"][28])
    # the z-buffer tie: the lower query index wins, and the other query's residual differs
    for name, i, want, wrong in probes:
        if name == "zbuffer_tie_query":
            pix = [pi for nm, pi, _, _ in probes if nm == "zbuffer_tie"][0]
            assert out["win"][pix] == i, (tag, out["win"][pix], i)
            k = out["k"][pix]
            t = [kdr.terms(q[j][None].astype(np.float64), flat_v[k, :, pix][None].astype(np.float64),
                           flat_n[k, :, pix][None].astype(np.float64), "geman_mcclure", 0.3)[0][28] for j in (i, wrong)]
            assert abs(t[0] - t[1]) >= 100 * out["tol"][28], (tag, "zbuffer_tie", t, out["tol"][28])
    return out


def _probe_run(lib, H, W, kcap=PROBE_K):
    vms, q, probes = probe_scene(H, W)
    ctx = _context(lib, H, W, kcap)
    for k in range(PROBE_K):
        _update(lib, ctx, np.eye(4, dtype=np.float32), vms[k])
    mv, mn = _model(lib, ctx, H, W)
    # identity poses: at the probe pixels the model holds the vertex maps' candidates themselves
    pix = [i for name, i, _, _ in probes if name != "zbuffer_tie_query"]
    assert np.array_equal(mv.reshape(PROBE_K, 3, -1)[:, :, pix], vms.reshape(PROBE_K, 3, -1)[:, :, pix])
    run = _register(lib, ctx, q, np.eye(4, dtype=np.float32), 1)
    ctx.close()
    return mv, mn, q, probes, run


@pytest.mark.parametrize("H,W", [(16, 512), (33, 500)])
def test_constructed_probes(lib, pref, kdr, H, W):
    mv, mn, q, probes, run = _probe_run(lib, H, W)
    names = {p[0] for p in probes}
    assert {"tie_tma", "tie_direct", "tie_straddle", "band_equal_roots", "band_diff_roots", "band_direct_redo",
            "nearest_direct", "nulls_between", "all_null", "tile_end", "tile_start", "last_pixel", "zbuffer_tie"} <= names
    _check_probes(pref, kdr, mv, mn, q, probes, run["sums"], (H, W))
    assert run["sums"][29] == len([p for p in probes if p[2] is not None and p[2] >= 0])
    _check_pose(kdr, np.eye(4, dtype=np.float32), run)


def test_accessor_refuses_before_the_first_icp_frame(lib):
    ctx = _context(lib, 16, 512, 4)
    with pytest.raises(RuntimeError, match="no ICP frame"):
        _last_sums(lib, ctx)
    ctx.close()


# ---------------------------------------------------------------------------------------------- e. launch knobs
KNOBS = [("PLS_PROJ_STAGES", "1"), ("PLS_PROJ_STAGES", "2"), ("PLS_PROJ_STAGES", "3"), ("PLS_PROJ_KDIRECT", "0"),
         ("PLS_PROJ_KDIRECT", "4"), ("PLS_PROJ_KDIRECT", "10"), ("PLS_PROJ_RESIDENT_MB", "0"),
         ("PLS_PROJ_RESIDENT_MB", "16"), ("PLS_PROJ_RESIDENT_MB", "4096"), ("PLS_PROJ_NO_TMA", "1")]
KNOB_SHAPE = (128, 4096)
PROBE_SHAPE = (16, 512)


def variant_main(out_path):
    """Runs in a subprocess with one launch knob set: the 128x4096 K = 20 first iteration and the 16x512 probes; writes
    their sums."""
    lib = _lib()
    H, W = KNOB_SHAPE
    ctx = _filled(lib, H, W, 20, 20)
    big = _register(lib, ctx, _queries(H, W, 20), np.eye(4, dtype=np.float32), 1)["sums"]
    ctx.close()
    probe = _probe_run(lib, *PROBE_SHAPE)[4]["sums"]
    np.savez(out_path, big=big, probe=probe)


def _geometry(env, H, W, K):
    g = dict(kdirect=4, stages=2, no_tma=False)
    for name, value in env:
        if name == "PLS_PROJ_KDIRECT":
            g["kdirect"] = int(value)
        elif name == "PLS_PROJ_STAGES":
            g["stages"] = int(value)
        elif name == "PLS_PROJ_NO_TMA":
            g["no_tma"] = True
    return _blocks(H, W, K, **g)


@pytest.fixture(scope="module")
def knob_reference(lib, tmp_path_factory):
    """The default launch (no knob) in a subprocess of its own, and the float64 references of both cases."""
    path = str(tmp_path_factory.mktemp("knobs") / "default.npz")
    _run_variant({}, path)
    H, W = KNOB_SHAPE
    ctx = _filled(lib, H, W, 20, 20)
    mv, mn = _model(lib, ctx, H, W)
    ctx.close()
    pv, pn, pq, probes, _ = _probe_run(lib, *PROBE_SHAPE)
    return dict(default=dict(np.load(path)), big=(mv, mn), probe=(pv, pn, pq, probes), dir=os.path.dirname(path))


def _run_variant(env, path):
    e = {k: v for k, v in os.environ.items() if not k.startswith("PLS_PROJ_")}
    e.update(env)
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_proj_icp_iterations_gpu as t; "
            f"t.variant_main({path!r})")
    r = subprocess.run([sys.executable, "-c", code], env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (env, r.stdout[-2000:], r.stderr[-4000:])


@pytest.mark.parametrize("name,value", KNOBS)
def test_launch_knob(pref, kdr, knob_reference, name, value):
    path = os.path.join(knob_reference["dir"], f"{name}_{value}.npz")
    _run_variant({name: value}, path)
    got = np.load(path)
    H, W = KNOB_SHAPE
    mv, mn = knob_reference["big"]
    _check_sums(pref, mv, mn, _queries(H, W, 20), np.eye(4, dtype=np.float32), got["big"], tag=(name, value),
                min_count=0.3 * H * W)
    pv, pn, pq, probes = knob_reference["probe"]
    _check_probes(pref, kdr, pv, pn, pq, probes, got["probe"], (name, value))
    ref = knob_reference["default"]
    for key, (h, w) in (("big", KNOB_SHAPE), ("probe", PROBE_SHAPE)):
        if _geometry([(name, value)], h, w, 20)[::2] == _geometry([], h, w, 20)[::2]:
            assert got[key].tobytes() == ref[key].tobytes(), (name, value, key)

