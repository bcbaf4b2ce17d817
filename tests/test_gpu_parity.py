"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the reference goldens.
Everything here needs a GPU (`-m gpu`).  Tolerances are stated per test:
  * integer / index work (a1): bit-exact
  * float32 image ops: pixel assignment exact up to points within an ulp of a rounding boundary
  * poses: 1e-4 relative translation, 1e-5 rad rotation (BASELINE.json north_star)
"""
import os

import numpy as np
import pytest
import torch

from conftest import check_pose_sequence, pose_errors

pytestmark = pytest.mark.gpu

SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


@pytest.fixture(scope="module")
def b200():
    import pylidar_slam_b200 as p
    return p


@pytest.fixture(scope="module")
def orc():
    from oracle import icp_oracle
    return icp_oracle


@pytest.fixture(scope="module")
def syn():
    from pylidar_slam_b200 import synthetic
    return synthetic


# ------------------------------------------------------------------------------------------------ a1
def test_a1_voxel_hash_golden(b200, golden_helpers):
    g = golden_helpers
    np.testing.assert_array_equal(b200.voxelise(g["a1_points"], 0.3), g["a1_coords"])
    np.testing.assert_array_equal(b200.voxel_hashing(g["a1_points"], 0.3), g["a1_hashes"])
    s, i = b200.grid_sample(g["a1_points"], 0.3)
    np.testing.assert_array_equal(i, g["a1_indices"])
    np.testing.assert_array_equal(s, g["a1_sample"])
    s, i = b200.grid_sample(g["a1_points64"], 0.1)
    np.testing.assert_array_equal(i, g["a1_indices64"])
    np.testing.assert_array_equal(s, g["a1_sample64"])


@pytest.mark.parametrize("n,voxel", [(1, 0.3), (2, 0.3), (2049, 0.05), (131072, 0.3), (524288, 0.4), (300000, 5.0)])
def test_a1_grid_sample_vs_oracle_sizes(b200, orc, syn, n, voxel):
    """Ragged sizes around the sort tile (2048), the BASELINE scan sizes and a heavy-collision case; bit-exact."""
    if n in (131072, 524288):
        pts = syn.scan(3, 64 if n == 131072 else 128, 2048 if n == 131072 else 4096)
    else:
        pts = (np.random.RandomState(n).randn(n, 3) * np.array([30.0, 30.0, 3.0])).astype(np.float32)
    s_ref, i_ref = orc.grid_sample(pts, voxel)
    s, i = b200.grid_sample(pts, voxel)
    np.testing.assert_array_equal(i, i_ref)
    np.testing.assert_array_equal(s, s_ref)
    # size-independent properties: indices unique, hashes strictly increasing, first occurrence
    h = orc.voxel_hashes(orc.voxel_coords(pts, voxel))
    assert np.all(np.diff(h[i]) > 0)
    first = {}
    for k, hv in enumerate(h[:20000]):
        first.setdefault(int(hv), k)
    sel = {int(h[k]): int(k) for k in i}
    assert all(sel[hv] == k for hv, k in first.items())


def test_a1_device_tensor_roundtrip(b200, orc):
    pts = (np.random.RandomState(5).randn(10000, 3) * 10).astype(np.float32)
    s_ref, i_ref = orc.grid_sample(pts, 0.5)
    s, i = b200.grid_sample(torch.from_numpy(pts).cuda(), 0.5)
    assert s.is_cuda and i.is_cuda
    np.testing.assert_array_equal(i.cpu().numpy(), i_ref)
    np.testing.assert_array_equal(s.cpu().numpy(), s_ref)


def test_cuda_tensor_inputs_wait_for_the_torch_stream_that_produces_them(b200, orc):
    """A CUDA tensor handed to the library may still be in the making on PyTorch's current stream (a slice copy, a
    dtype conversion, a network's forward pass).  The library runs on its own non-blocking stream, so it has to order
    itself after that stream (pls_wait_stream, issued by _lib.Context.call): here the input buffer is filled by a copy
    queued BEHIND ~30 ms of matrix products; read too early it is still all zeros."""
    rs = np.random.RandomState(11)
    pts = (rs.randn(120000, 3) * 12).astype(np.float32)
    wide = np.concatenate([pts, rs.randn(120000, 2).astype(np.float32)], axis=1)        # [n,5]: the cloud is a strided slice
    src = torch.from_numpy(wide).cuda()
    busy = torch.randn(4096, 4096, device="cuda")
    s_ref, i_ref = orc.grid_sample(pts, 0.4)
    for attempt in range(3):
        buf = torch.zeros(120000, 3, device="cuda")
        torch.cuda.synchronize()
        for _ in range(24):
            busy = (busy @ busy).clamp_(-1.0, 1.0)                                       # keeps PyTorch's stream busy
        buf.copy_(src[:, :3])                                                            # ... and only then fills the input
        s, i = b200.grid_sample(buf, 0.4)                                                # no synchronisation in between
        np.testing.assert_array_equal(i.cpu().numpy(), i_ref)
        np.testing.assert_array_equal(s.cpu().numpy(), s_ref)
        # the same through a conversion the mirror itself enqueues (float64 -> float32 .contiguous() of a strided view)
        for _ in range(24):
            busy = (busy @ busy).clamp_(-1.0, 1.0)
        view64 = src.double()[:, :3]
        s2, i2 = b200.grid_sample(view64.float(), 0.4)
        np.testing.assert_array_equal(i2.cpu().numpy(), i_ref)


def test_a1_voxelise_with_one_voxel_length_per_axis(b200, golden_misc):
    """voxelise(pointcloud, voxel_x, voxel_y, voxel_z) (pointcloud.py:55-79): bit-exact against the reference."""
    g = golden_misc
    vx, vy, vz = (float(v) for v in g["vox_sizes"])
    np.testing.assert_array_equal(b200.voxelise(g["vox_points"], vx, vy, vz), g["vox_coords"])
    np.testing.assert_array_equal(b200.voxelise(torch.from_numpy(g["vox_points"]).cuda(), vx, vy, vz).cpu().numpy(), g["vox_coords"])
    np.testing.assert_array_equal(b200.voxelise(g["vox_points"], vx), b200.voxelise(g["vox_points"], vx, vx, vx))


# --------------------------------------------------------------------------------------------- a2/a3
def _pixel_mismatch(a, b):
    return float(np.mean(np.any(a != b, axis=0)))


def test_a3_projection_golden(b200, golden_helpers):
    g = golden_helpers
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    pts = g["a3_points"][None]
    pix = proj.project_pointcloud(pts)[0]
    ok = ~np.isnan(g["a3_pixels"][:, 0])
    # float pixel coordinates: libm atan2/asin differ by <= 2 ulp between CUDA and the CPU -> 1e-3 px
    np.testing.assert_allclose(pix[ok], g["a3_pixels"][ok], atol=2e-3)
    vmap = proj.build_projection_map(pts)[0]
    assert _pixel_mismatch(vmap, g["a3_vmap"]) <= 2e-3   # points within an ulp of a .5 boundary


def test_a3_projection_default_value_and_default_channels(b200, golden_misc):
    """Projector.build_projection_map(default_value=...) (projection.py:333,378-391): pixels no point lands on hold the
    value; with no `transform` a [B,N,4] cloud yields the three xyz channels (the projector's xyz_conversion)."""
    g = golden_misc
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    out = proj.build_projection_map(g["proj_cloud"][None], default_value=float(g["proj_default"]))[0]
    assert out.shape == g["proj_map"].shape == (3, 16, 256)
    empty = np.all(g["proj_map"] == g["proj_default"], axis=0)
    assert empty.any() and not empty.all()
    assert _pixel_mismatch(out, g["proj_map"]) <= 2e-3          # points within an ulp of a .5 pixel boundary, as in a3
    np.testing.assert_array_equal(np.all(out == g["proj_default"], axis=0)[empty], True)
    four = proj.build_projection_map(g["proj_cloud"][None], default_value=2.0, transform=lambda x: x)[0]
    assert four.shape == (4, 16, 256) and np.all(four[:, empty] == 2.0)


@pytest.mark.parametrize("H,W", [(64, 2048), (128, 4096)])
def test_a3_projection_full_size_vs_oracle(b200, orc, syn, H, W):
    pts = syn.scan(2, H, W)
    T = syn.gt_relative_pose(2).astype(np.float32)
    moved = pts @ T[:3, :3].T + T[:3, 3]          # off-centre: collisions and empty pixels
    both = np.concatenate([moved, pts * 1.003], 0)[None]
    ref = orc.Projector(H, W).build_projection_map(torch.from_numpy(both))[0].numpy()
    out = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0).build_projection_map(both)[0]
    assert _pixel_mismatch(out, ref) <= 1e-3
    # ... and EVERY differing pixel is accounted for: the z-buffer itself is exact integer work; the only float step
    # before it is the pixel coordinate (atan2 / asin: CUDA's libm and the host's differ by a couple of ulp), so a
    # pixel may differ only if some input point has a coordinate within 2e-3 px of a rounding boundary there
    row, col = orc.Projector(H, W).pixels(torch.from_numpy(both))
    rc = np.stack([row[0].numpy(), col[0].numpy()], axis=1).astype(np.float64)             # float (row, col) per point
    near = (np.abs(rc - np.floor(rc) - 0.5) < 2e-3).any(axis=1) & np.isfinite(rc).all(axis=1)
    touched = np.zeros((H, W), bool)
    for r, c in rc[near]:
        for rr in (int(np.floor(r)), int(np.ceil(r))):
            for cc in (int(np.floor(c)), int(np.ceil(c))):
                if 0 <= rr < H and 0 <= cc < W:
                    touched[rr, cc] = True
    differing = np.any(out != ref, axis=0)
    # ... or the two winners are range ties to the last bits (the range itself is a float32 sqrt on either side)
    r_gpu, r_ref = np.linalg.norm(out.astype(np.float64), axis=0), np.linalg.norm(ref.astype(np.float64), axis=0)
    unexplained = differing & ~touched & (np.abs(r_gpu - r_ref) > 2e-6 * np.maximum(r_ref, 1e-9))
    assert not unexplained.any(), int(unexplained.sum())
    # closest-wins property, independent of the oracle: every written pixel holds an input point
    r_out = np.linalg.norm(out, axis=0)
    assert np.all(r_out[r_out > 0] > 0.5)


def test_a3_projection_with_channels_and_batch(b200, orc, syn):
    H, W = 16, 256
    B = 3
    xyz = np.stack([syn.scan(k, H, W) for k in range(B)], 0)
    ch = np.concatenate([xyz, np.random.RandomState(0).randn(B, H * W, 3).astype(np.float32)], -1)
    ref = orc.Projector(H, W).build_projection_map(torch.from_numpy(xyz), channels=torch.from_numpy(ch)).numpy()
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    out = proj.build_projection_map(ch, transform=lambda x: x)
    assert out.shape == (B, 6, H, W)
    for b in range(B):
        assert _pixel_mismatch(out[b], ref[b]) <= 2e-3


# ------------------------------------------------------------------------------------------------ a16
def test_a16_pose_golden(b200, golden_helpers):
    g = golden_helpers
    pose = b200.Pose("euler")
    np.testing.assert_allclose(pose.build_pose_matrix(g["a16_params"]), g["a16_mats"], atol=1e-6)
    np.testing.assert_allclose(pose.from_pose_matrix(g["a16_mats"]), g["a16_back"], atol=1e-5)


# ------------------------------------------------------------------------------------------ a11-a15
@pytest.mark.parametrize("scheme", SCHEMES)
def test_gn_step_golden(b200, golden_helpers, scheme):
    g = golden_helpers
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme=scheme, sigma=0.3, max_iters=1)))
    dT, x, loss = al.align(g["gn_ref"][None], g["gn_tgt"][None], g["gn_nrm"][None])
    # the reference solves in float32 (sgemm + float32 inverse); ours accumulates and solves in float64
    np.testing.assert_allclose(x[0], g[f"gn_{scheme}_delta"], rtol=2e-4, atol=2e-7)
    np.testing.assert_allclose(dT[0], g[f"gn_{scheme}_dT"], atol=2e-6)
    np.testing.assert_allclose(loss[0], g[f"gn_{scheme}_loss"], rtol=1e-3, atol=1e-9)


def test_gn_multi_iter_and_known_answer(b200, golden_helpers):
    g = golden_helpers
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=5, norm_stop_criterion=1e-9)))
    _, x, _ = al.align(g["gn_ref"][None], g["gn_tgt"][None], g["gn_nrm"][None])
    np.testing.assert_allclose(x[0], g["gn_multi_x"], rtol=1e-3, atol=1e-6)
    # reference tests/test_optimization.py (float64, scheme default): known answer to 1e-7
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="default", max_iters=100, norm_stop_criterion=1e-10)))
    for b in range(2):
        _, x, loss = al.align(g["ka_ref"][b][None], g["ka_tgt"][b][None], g["ka_nrm"][b][None])
        assert x.dtype == np.float64
        assert np.abs(x[0] - g["ka_params"][b]).max() <= 1e-7
        assert np.abs(x[0] - g["ka_est"][b]).max() <= 1e-9
        assert float(np.abs(loss).sum()) <= 1e-7


def test_gn_cfg1_10k_vs_oracle(b200, orc):
    """BASELINE config 1: single point-to-plane GN step, 10k points, known pose, vs the CPU path."""
    torch.manual_seed(0)
    N = 10000
    tgt = torch.randn(1, N, 3) * 10
    nrm = torch.randn(1, N, 3)
    nrm /= nrm.norm(dim=-1, keepdim=True)
    xs = torch.randn(1, 6) * torch.tensor([[.01, .01, .01, .001, .001, .001]])
    ref = orc.apply_transformation(tgt, orc.build_pose_matrix(xs)) + 0.01 * torch.randn(1, N, 3)
    for scheme in ("default", "geman_mcclure"):
        dT_o, x_o, loss_o = orc.align_p2plane(ref, tgt, nrm, scheme, 0.3, 1)
        al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
            gauss_newton_config=dict(scheme=scheme, sigma=0.3, max_iters=1)))
        dT, x, loss = al.align(ref.cuda(), tgt.cuda(), nrm.cuda())
        assert x.is_cuda
        np.testing.assert_allclose(x.cpu().numpy(), x_o.numpy(), rtol=2e-4, atol=2e-7)
        dt, ang = pose_errors(dT[0].cpu().numpy(), dT_o[0].numpy())
        assert ang <= 1e-5 and dt <= 1e-4


def test_gn_singular_raises_and_tiny_residual_warns(b200, orc, caplog):
    torch.manual_seed(0)
    tgt = torch.randn(1, 100, 3, dtype=torch.float64)
    nrm = torch.randn(1, 100, 3, dtype=torch.float64)
    nrm /= nrm.norm(dim=-1, keepdim=True)
    x = torch.tensor([[0.01, 0.01, 0.01, 0.001, 0.001, 0.001]], dtype=torch.float64)
    ref = orc.apply_transformation(tgt, orc.build_pose_matrix(x))
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="huber", sigma=1e-4, max_iters=100, norm_stop_criterion=1e-10)))
    with pytest.raises(RuntimeError, match="Invalid Jacobian"):
        al.align(ref.numpy(), tgt.numpy(), nrm.numpy())
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="default", max_iters=3)))
    dT, xx, loss = al.align(tgt.numpy(), tgt.numpy(), nrm.numpy())   # zero residual -> warning, x = 0
    assert np.all(xx == 0) and np.allclose(dT[0], np.eye(4))


def test_align_bad_shape_is_assertion(b200):
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig())
    with pytest.raises(AssertionError):
        al.align(np.zeros((1, 5, 3), np.float32), np.zeros((1, 4, 3), np.float32), np.zeros((1, 4, 3), np.float32))


# ----------------------------------------------------------------------------------------- a7-a9
def _brute_nn(q, m):
    d = ((q[:, None, :].astype(np.float64) - m[None, :, :].astype(np.float64)) ** 2).sum(-1)
    return d.argmin(1), d.min(1)


def test_kd_local_map_golden(b200, golden_helpers):
    g = golden_helpers
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=2))
    lm.init()
    lm.update(np.eye(4, dtype=np.float32)[None], new_vertex_map=g["kd_v0"][None])
    lm.update(g["kd_rel"][None], new_pc_data=g["kd_pc1"])
    np.testing.assert_allclose(lm.points(), g["kd_map"], atol=2e-5)
    res = lm.nearest_neighbor_search(g["kd_queries"])
    np.testing.assert_allclose(res.neighbor_points, g["kd_nb"], atol=2e-5)
    dots = np.abs((res.neighbor_normals * g["kd_normals"]).sum(-1))
    assert np.mean(dots > 1 - 1e-4) > 0.99


@pytest.mark.parametrize("M,N", [(1, 7), (3, 50), (11, 100), (2047, 3000), (2048, 3000), (2049, 3000), (5000, 3000),
                                 (4 * 2048 + 1, 3000), (330000, 20000)])
def test_kd_exact_nn_vs_bruteforce(b200, M, N):
    """Exactness independent of the oracle (the reference never tests KdTreeLocalMap): brute force,
    ragged/tiny maps, heavy duplicates, maps on the edges of the index build's 2048-key sort tiles."""
    rng = np.random.RandomState(M)
    m = (rng.randn(M, 3) * np.array([40, 40, 3])).astype(np.float32)
    if M >= 5000:
        m[::7] = m[1::7][: len(m[::7])]          # exact duplicates
    q = (rng.randn(N, 3) * np.array([45, 45, 4])).astype(np.float32)
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=3))
    lm.init()
    lm.update(np.eye(4, dtype=np.float32)[None], new_pc_data=m)
    res = lm.nearest_neighbor_search(q, with_normals=M >= 11)
    if M <= 5000:
        idx, dmin = _brute_nn(q, m)
    else:
        from scipy.spatial import cKDTree
        dmin, idx = cKDTree(m.astype(np.float64)).query(q.astype(np.float64))
        dmin = dmin ** 2
    d_mine = ((q.astype(np.float64) - res.neighbor_points.astype(np.float64)) ** 2).sum(-1)
    np.testing.assert_allclose(d_mine, dmin, rtol=1e-5, atol=1e-9)
    # the runner-up bound each search stored (what later ICP iterations verify against): every map point other than
    # the match is at least sqrt(second) from the query position it stored
    from pylidar_slam_b200 import _lib
    from scipy.spatial import cKDTree
    idx, state = np.empty(N, np.int64), np.empty((N, 4), np.float32)
    lm.ctx.call("pls_kdmap_last_correspondences", N, _lib.ptr(idx), None, None, _lib.ptr(state), None)
    assert np.array_equal(state[:, :3], q) and np.array_equal(m[idx], res.neighbor_points)
    dd, ii = cKDTree(m.astype(np.float64)).query(q.astype(np.float64), k=2)
    d_other = np.where(ii[:, 0] == idx, dd[:, 1], dd[:, 0])      # inf when the map has one point
    assert (np.sqrt(state[:, 3].astype(np.float64)) <= d_other * 1.00001 + 1e-6).all()


def test_a9_normals_per_point_bound(b200, syn):
    """Every returned normal against an independent float64 computation from the exact 10 nearest map neighbours of
    the matched point (scipy cKDTree on the same float32 map): |sin angle| <= 2e-5 * lambda_max / gap, gap =
    lambda_mid - lambda_min of the point's second-moment matrix -- the perturbation bound of an eigenvector for the
    float32 rounding of the moments (~1e-6 lambda_max, as in the reference).  Only points whose plane direction is
    provably ill-defined (gap < 1e-3 lambda_max: the reference's own SVD is arbitrary there) are excluded, and they
    must be rare."""
    from scipy.spatial import cKDTree
    H, W = 32, 1024
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=4))
    lm.init()
    for k in range(4):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        s, _ = b200.grid_sample(syn.scan(k, H, W), 0.3)
        lm.update(rel[None], new_pc_data=s)
    m = lm.points()
    q, _ = b200.grid_sample(syn.scan(4, H, W), 0.3)
    res = lm.nearest_neighbor_search(q)
    tree = cKDTree(m.astype(np.float64))
    _, i1 = tree.query(res.neighbor_points.astype(np.float64))
    assert np.abs(m[i1] - res.neighbor_points).max() == 0.0              # the matches are map points
    d11, i11 = tree.query(m[i1].astype(np.float64), k=12)
    unique_set = d11[:, 11] > d11[:, 10] * (1 + 1e-6)                     # no tie at the 10th neighbour
    diff = (m[i11[:, 1:11]] - m[i1][:, None, :]).astype(np.float64)
    C = (diff[:, :, :, None] * diff[:, :, None, :]).mean(axis=1)
    w, v = np.linalg.eigh(C)
    gap = (w[:, 1] - w[:, 0]) / np.maximum(w[:, 2], 1e-300)
    sin = np.linalg.norm(np.cross(res.neighbor_normals.astype(np.float64), v[:, :, 0]), axis=1)
    ok = unique_set & (gap > 1e-3)
    assert ok.mean() > 0.9, ok.mean()   # 6 % of this scene's matches sit on pillar edges / scan-line rows
    assert (sin[ok] <= 2e-5 / gap[ok] + 2e-7).all(), float((sin[ok] * gap[ok]).max())
    assert np.abs(np.linalg.norm(res.neighbor_normals, axis=1) - 1).max() <= 1e-6


def test_kd_map_lifecycle_vs_oracle(b200, orc, syn):
    """Move / append / evict over several frames; normals against the oracle (sign-free)."""
    H, W = 16, 256
    mine = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=3))
    theirs = orc.KdTreeLocalMap(local_map_size=3)
    mine.init()
    for k in range(6):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        pts = syn.scan(k, H, W)
        if k == 4:
            mine.update(rel[None])                    # move only
            theirs.update(rel)
        else:
            mine.update(rel[None], new_pc_data=pts)
            theirs.update(rel, new_points=pts)
        assert mine.num_points() == theirs.points.shape[0]
        np.testing.assert_allclose(mine.points(), theirs.points, atol=5e-5)
    q = syn.scan(6, H, W)[::2]
    res = mine.nearest_neighbor_search(q)
    nb, nrm, _ = theirs.nearest_neighbor_search(q)
    assert np.mean(np.linalg.norm(res.neighbor_points - nb, axis=1) < 1e-4) > 0.999
    dots = np.abs((res.neighbor_normals * nrm).sum(-1))
    assert np.mean(dots > 1 - 1e-4) > 0.99


# ---------------------------------------------------------------------------------------- a17/a18
def _drive(algo, frame_fn, n, iters=None):
    prev, poses = None, []
    for k in range(n):
        dd = frame_fn(k)
        dd["init_rpose"] = prev
        algo.process_next_frame(dd)
        if "odometry_pose" in dd:
            poses.append(dd["odometry_pose"].copy())
            prev = dd["odometry_pose"].astype(np.float64)
            if iters is not None:
                iters.append(int(algo.last_info[0]))
        else:
            assert k == 0
    return np.stack(poses)


def _frames(syn, grid_sample, layout, H, W, voxel, device="cpu"):
    def fn(k):
        pc = syn.scan(k, H, W)
        if layout == "vertex_map":
            return {"vertex_map": torch.from_numpy(syn.vertex_map_from_scan(pc, H, W)).to(device)}
        if voxel:
            pc, _ = grid_sample(pc, voxel)
        return {"numpy_pc": pc} if layout == "ndarray" else {"input_data": torch.from_numpy(pc).to(device)}
    return fn


def _make(b200, lm, H, W, key, iters, scheme="geman_mcclure", sigma=0.3, lm_size=20, thr=1e-4):
    lmc = (b200.KdTreeLocalMapConfig(local_map_size=lm_size) if lm == "kdtree"
           else b200.ProjectiveLocalMapConfig(local_map_size=lm_size))
    cfg = b200.ICPFrameToModelConfig(
        local_map=lmc, alignment=b200.GaussNewtonPointToPlaneConfig(
            gauss_newton_config=dict(scheme=scheme, sigma=sigma, max_iters=1)),
        max_num_alignments=iters, data_key=key, threshold_delta_pose=thr)
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0),
                                pose=b200.Pose("euler"), device="cuda:0")
    algo.init()
    return algo


KD_SMALL = [("kd_ndarray", "ndarray", "numpy_pc", 0.4, 7, "geman_mcclure", 0.3, 8),
            ("kd_tensor", "tensor", "input_data", 0.4, 7, "geman_mcclure", 0.3, 8),
            ("kd_vmap", "vertex_map", "vertex_map", None, 4, "geman_mcclure", 0.3, 8),
            ("kd_default", "ndarray", "numpy_pc", 0.4, 5, "default", 0.5, 6)]


@pytest.mark.parametrize("case", KD_SMALL, ids=[c[0] for c in KD_SMALL])
def test_icp_kd_small_vs_reference_golden(b200, syn, golden_icp_small, case):
    name, layout, key, voxel, nf, scheme, sigma, iters = case
    algo = _make(b200, "kdtree", 32, 512, key, iters, scheme, sigma, lm_size=4)
    poses = _drive(algo, _frames(syn, b200.grid_sample, layout, 32, 512, voxel), nf)
    ref = golden_icp_small[f"{name}_poses"]
    assert poses.shape == ref.shape
    for T, Tr in zip(poses, ref):
        dt, ang = pose_errors(T, Tr)
        assert dt <= 1e-4 and ang <= 1e-5, (name, dt, ang)
    assert algo.get_relative_poses().shape == (nf, 4, 4)
    assert len(algo.elapsed) == nf


@pytest.mark.parametrize("name,layout,key", [("cfg2_tensor", "tensor", "input_data"), ("cfg2_ndarray", "ndarray", "numpy_pc")])
def test_icp_cfg2_full_size_vs_reference_golden(b200, syn, golden_icp_full, name, layout, key):
    """BASELINE config 2 (64x2048, grid_sample 0.3, kd map K=20, geman_mcclure 0.3, 10 alignments):
    per-frame poses of the UNMODIFIED reference, 1e-4 relative translation / 1e-5 rad on every frame
    with the reference's iteration count (see conftest.check_pose_sequence for the stop-rule slack)."""
    ref = golden_icp_full[f"{name}_poses"]
    algo = _make(b200, "kdtree", 64, 2048, key, 10)
    iters = []
    poses = _drive(algo, _frames(syn, b200.grid_sample, layout, 64, 2048, 0.3), len(ref) + 1, iters)
    flips, worst = check_pose_sequence(poses, iters, ref, golden_icp_full[f"{name}_losses"], name=name)
    print(name, "flips", flips, "worst (rel t, rad) on matching frames", worst)


@pytest.mark.parametrize("name,layout,key", [("cfg2_tensor_fixed6", "tensor", "input_data"),
                                             ("cfg2_ndarray_fixed6", "ndarray", "numpy_pc")])
def test_icp_cfg2_fixed_iterations_strict(b200, syn, golden_icp_full, name, layout, key):
    """Same stream with threshold_delta_pose = 0 and exactly 6 alignments per frame: no stop-rule
    knife edge, so the strict north-star tolerance applies to every frame, and the per-iteration
    losses are compared too."""
    ref = golden_icp_full[f"{name}_poses"]
    algo = _make(b200, "kdtree", 64, 2048, key, 6, thr=0.0)
    iters = []
    poses = _drive(algo, _frames(syn, b200.grid_sample, layout, 64, 2048, 0.3), len(ref) + 1, iters)
    assert all(i == 6 for i in iters)
    for k, (T, Tr) in enumerate(zip(poses, ref)):
        dt, ang = pose_errors(T, Tr)
        assert dt <= 1e-4 and ang <= 1e-5, (name, k, dt, ang)


def test_icp_device_tensor_input_and_outputs(b200, syn):
    algo = _make(b200, "kdtree", 32, 512, "input_data", 8, lm_size=4)
    frames = _frames(syn, b200.grid_sample, "tensor", 32, 512, 0.4, device="cuda")
    dd0 = frames(0)
    algo.process_next_frame(dd0)
    assert "odometry_pose" not in dd0          # frame 0 writes nothing (icp_odometry.py:171-181)
    dd1 = frames(1)
    algo.process_next_frame(dd1)
    assert dd1["odometry_pose"].shape == (4, 4) and dd1["odometry_pose"].dtype == np.float32
    assert isinstance(dd1["odometry_pc"], np.ndarray) and dd1["odometry_pc"].shape[1] == 3
    gt = syn.gt_relative_pose(1)
    assert np.abs(dd1["odometry_pose"][:3, 3] - gt[:3, 3]).max() < 0.1


def test_icp_missing_key_and_bad_shape(b200):
    algo = _make(b200, "kdtree", 16, 256, "numpy_pc", 4)
    with pytest.raises(AssertionError):
        algo.process_next_frame({"other": 1})
    with pytest.raises(AssertionError):
        algo.process_next_frame({"numpy_pc": np.zeros((10, 4), np.float32)})


def test_preprocessing_chain_matches_reference_layout(b200, orc, syn):
    """grid_sample.yaml without the distortion filter: GridSample -> ToTensor keys."""
    pre = b200.Preprocessing(b200.PreprocessingConfig(filters={
        "2": dict(filter_name="grid_sample", voxel_size=0.3, pointcloud_key="numpy_pc"),
        "3": dict(filter_name="to_tensor", keys=dict(sample_points="input_data"))}))
    dd = {"numpy_pc": syn.scan(0, 32, 512)}
    pre.forward(dd)
    s_ref, i_ref = orc.grid_sample(dd["numpy_pc"], 0.3)
    np.testing.assert_array_equal(dd["sample_indices"], i_ref)
    np.testing.assert_array_equal(dd["input_data"].numpy(), s_ref)


# ------------------------------------------------------------------------------------- a4 / a5 / a6
def _normal_agreement(a, b, vmap):
    """Fraction of non-null pixels whose unit normals agree (sign-free) to 1e-2 rad, and to 0.1 rad."""
    valid = (np.abs(vmap).max(0) > 0) & (np.linalg.norm(b, axis=0) > 0.5)
    dots = np.abs((a * b).sum(0))[valid]
    return float(np.mean(dots > np.cos(1e-2))), float(np.mean(dots > np.cos(0.1)))


def test_a4_normal_map_golden_and_oracle(b200, orc, syn, golden_helpers):
    """The reference's normals are float32-rounding dominated (it inverts the uncentred second-moment
    matrix), so the kernel reproduces its exact operation order; the goldens are matched BIT-EXACTLY."""
    g = golden_helpers
    for k, vkey, key in ((5, "a4_vmap", "a4_nmap"), (3, "a4_vmap", "a4_nmap_k3"), (5, "a4b_vmap", "a4b_nmap")):
        n = b200.compute_normal_map(g[vkey][None], kernel_size=k)[0]
        assert n.shape == g[key].shape
        assert np.mean(n == g[key]) > 0.9999, (key, np.mean(n == g[key]))
        norms = np.linalg.norm(n, axis=0)
        assert np.all((np.abs(norms - 1) < 1e-4) | (norms == 0))
    H, W = 64, 2048
    vm = syn.vertex_map_from_scan(syn.scan(5, H, W), H, W)
    ref = orc.normal_map(torch.from_numpy(vm), 5)[0].numpy()
    out = b200.compute_normal_map(torch.from_numpy(vm).cuda(), 5)[0].cpu().numpy()
    tight, loose = _normal_agreement(out, ref, vm[0])
    assert tight > 0.995 and loose > 0.999, (tight, loose)
    B = 2                                                    # batched call
    both = np.concatenate([vm, syn.vertex_map_from_scan(syn.scan(6, H, W), H, W)], 0)
    outb = b200.compute_normal_map(both, 5)
    assert outb.shape == (B, 3, H, W) and np.array_equal(outb[0], out)


def test_a6_compute_neighbors_golden(b200, golden_helpers):
    g = golden_helpers
    nb, nf = b200.compute_neighbors(g["a6_tgt"][None], g["a6_ref"], g["a6_fields"])
    np.testing.assert_array_equal(nb[0], g["a6_nb"])
    np.testing.assert_array_equal(nf[0], g["a6_nf"])


def test_a6_reference_geometry_property(b200):
    """tests/test_geometry.py:6-24 of the reference on the CUDA path."""
    torch.manual_seed(0)
    tgt, ref = torch.randn(1, 3, 10, 10), torch.randn(10, 3, 10, 10)
    tgt[0, :, 0, 0] = 0.0
    nb, _ = b200.compute_neighbors(tgt.cuda(), ref.cuda())
    nb = nb.cpu()
    assert nb[0, :, 0, 0].norm() == 0.0
    d_nb = (nb - tgt).norm(dim=1)[0]
    d_all = (ref - tgt).norm(dim=1)
    mask = torch.ones(10, 10, dtype=torch.bool)
    mask[0, 0] = False
    assert bool(((d_nb.unsqueeze(0) <= d_all)[:, mask]).all())


def test_a5_projective_map_lifecycle_vs_oracle(b200, orc, syn):
    """update / evict / move-only, the re-projected model maps and the pixel association vs the oracle."""
    H, W = 32, 512
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    mine = b200.ProjectiveLocalMap(b200.ProjectiveLocalMapConfig(local_map_size=3), projector=proj)
    theirs = orc.ProjectiveLocalMap(orc.Projector(H, W), local_map_size=3)
    mine.init()
    for k in range(6):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        vm = syn.vertex_map_from_scan(syn.scan(k, H, W), H, W)
        if k == 4:
            mine.update(rel[None])
            theirs.update(torch.from_numpy(rel)[None])
        else:
            mine.update(rel[None], new_vertex_map=vm)
            theirs.update(torch.from_numpy(rel)[None], new_vertex_map=torch.from_numpy(vm))
        mv, mn = mine.model()
        assert mv.shape == tuple(theirs.model_vmap.shape)
        tv = theirs.model_vmap.numpy()
        for j in range(mv.shape[0]):
            # same z-buffer winners up to the ~1e-7 difference between the rigid and the LU pose inverse
            occupied = np.abs(tv[j]).max(0) > 0
            same = np.all(np.abs(mv[j] - tv[j]) < 1e-3, axis=0)
            assert np.mean(same[occupied]) > 0.995, (k, j, np.mean(same[occupied]))
            assert np.mean((np.abs(mv[j]).max(0) > 0) == occupied) > 0.999
    q = syn.scan(6, H, W)
    T = syn.gt_relative_pose(6).astype(np.float32)
    q = q @ T[:3, :3].T + T[:3, 3]
    res = mine.nearest_neighbor_search(q)
    tq, tn, tp = theirs.nearest_neighbor_search(torch.from_numpy(q))
    assert abs(res.neighbor_points.shape[1] - tq.shape[1]) <= 0.01 * tq.shape[1]
    # compare through a per-pixel dictionary keyed on the (exactly preserved) target point
    key = {tuple(p): (a, b) for p, a, b in zip(tp[0].numpy().round(5).tolist(), tq[0].numpy(), tn[0].numpy())}
    hits = close = 0
    for p, a in zip(res.new_target_points[0].round(5).tolist(), res.neighbor_points[0]):
        if tuple(p) in key:
            hits += 1
            close += np.linalg.norm(a - key[tuple(p)][0]) < 1e-3
    assert hits > 0.95 * tq.shape[1] and close > 0.97 * hits


PROJ_SMALL = [("proj_vmap", "vertex_map", "vertex_map"), ("proj_ndarray", "ndarray", "numpy_pc")]


def measured_sensitivity(case):
    """Largest pose deviation of the UNMODIFIED reference from itself when the last bit of its input coordinates is
    perturbed (tests/golden/sensitivity.json, written by tests/golden/sensitivity.py in the build container)."""
    import json
    d = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sensitivity.json")))["cases"][case]
    return d["max_rel_translation"], d["max_rotation_rad"]


def relaxed_tolerance(case, wanted):
    """A translation tolerance above the north star's 1e-4 is admissible only up to 1.5 x what the reference itself
    moves under 1-ulp input noise in that configuration."""
    sens_t, _ = measured_sensitivity(case)
    assert wanted <= max(1e-4, 1.5 * sens_t), (case, wanted, sens_t)
    return wanted


@pytest.mark.parametrize("name,layout,key", PROJ_SMALL)
def test_icp_projective_small_vs_reference_golden(b200, syn, golden_icp_small, name, layout, key):
    """32x512 projective ICP is numerically ill-conditioned in the REFERENCE itself: its normals come from
    a float32 inverse of the uncentred second-moment matrix and 8 iterations do not converge.  Measured on
    the unmodified reference (tests/golden/sensitivity.py -> sensitivity.json): 1-ulp noise on the input scans
    moves its own poses by up to 2.8e-3 relative translation / 2.6e-5 rad within 6 frames (3 seeds).  The translation
    tolerance here is 6e-4 -- a fifth of that -- and the rotation stays at 1e-5; the full-size config-3 test below
    keeps the strict 1e-4."""
    algo = _make(b200, "projective", 32, 512, key, 8, lm_size=4)
    iters = []
    poses = _drive(algo, _frames(syn, b200.grid_sample, layout, 32, 512, None), 7, iters)
    flips, worst = check_pose_sequence(poses, iters, golden_icp_small[f"{name}_poses"], golden_icp_small[f"{name}_losses"],
                                       name=name, tol_t=relaxed_tolerance(f"{name}_32x512", 6e-4))
    print(name, "flips", flips, "worst", worst)


@pytest.mark.parametrize("name,lm,key", [("kd_gn3", "kdtree", "numpy_pc"), ("proj_gn2", "projective", "vertex_map")])
def test_icp_with_several_gauss_newton_steps_vs_reference_golden(b200, syn, name, lm, key):
    """gauss_newton_config.max_iters > 1 (alignment.py:69-77,110-127: several re-linearised Gauss-Newton steps on the same
    correspondences per ICP iteration) takes the reference-shaped loop over the fine-grained GPU plug-ins; poses against the
    unmodified reference (tests/golden/make_golden_gn.py), 5 alignments per frame, no stop rule."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_gn.npz"))
    H, W = 32, 512
    lmc = b200.KdTreeLocalMapConfig(local_map_size=4) if lm == "kdtree" else b200.ProjectiveLocalMapConfig(local_map_size=4)
    cfg = b200.ICPFrameToModelConfig(
        local_map=lmc, alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(
            scheme="geman_mcclure", sigma=0.3, max_iters=int(g[f"{name}_gn_iters"]), norm_stop_criterion=1e-9)),
        max_num_alignments=5, data_key=key, threshold_delta_pose=0.0)
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0),
                                pose=b200.Pose("euler"), device="cuda:0")
    algo.init()
    layout = "ndarray" if key == "numpy_pc" else "vertex_map"
    poses = _drive(algo, _frames(syn, b200.grid_sample, layout, H, W, 0.4 if layout == "ndarray" else None), 6)
    ref = g[f"{name}_poses"]
    assert len(poses) == len(ref)
    tol_t = 1e-4 if lm == "kdtree" else relaxed_tolerance("proj_vmap_32x512", 6e-4)
    for k, (T, Tr) in enumerate(zip(poses, ref)):
        dt, ang = pose_errors(T, Tr)
        assert dt <= tol_t and ang <= 1e-5, (name, k, dt, ang)


def test_icp_cfg3_projective_full_size_vs_reference_golden(b200, syn, golden_icp_full):
    """BASELINE config 3 (128x2048 vertex-map input, projective map K<=20, normals kernel 5)."""
    ref = golden_icp_full["cfg3_proj_poses"]
    algo = _make(b200, "projective", 128, 2048, "vertex_map", 10)
    iters = []
    poses = _drive(algo, _frames(syn, b200.grid_sample, "vertex_map", 128, 2048, None, device="cuda"), len(ref) + 1, iters)
    flips, worst = check_pose_sequence(poses, iters, ref, golden_icp_full["cfg3_proj_losses"], name="cfg3_proj")
    print("cfg3", "flips", flips, "worst", worst)


# ------------------------------------------------------------------------------ BASELINE configs 4 / 5, edge cases
def test_cfg4_5M_point_map_exact_search(b200):
    """BASELINE config 4: a 5M-point accumulated local map, one 64x2048 scan (131072 queries): exact 1-NN
    against scipy's cKDTree (float64) and, sign-free, the 10-NN normals on a sample."""
    from scipy.spatial import cKDTree
    rng = np.random.RandomState(4)
    M = 5_000_000
    # surfaces (ground + walls) with noise, LiDAR-like density falling with range
    r = rng.gamma(2.0, 12.0, M).astype(np.float32)
    a = rng.uniform(-np.pi, np.pi, M).astype(np.float32)
    ground = rng.rand(M) < 0.7
    pts = np.stack([r * np.cos(a), r * np.sin(a), np.where(ground, -1.8 + 0.01 * rng.randn(M), rng.uniform(-1.8, 6, M))], 1).astype(np.float32)
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=2))
    lm.init()
    lm.update(np.eye(4, dtype=np.float32)[None], new_pc_data=pts)
    assert lm.num_points() == M
    q = pts[rng.choice(M, 131072, replace=False)] + (0.05 * rng.randn(131072, 3)).astype(np.float32)
    res = lm.nearest_neighbor_search(q)
    tree = cKDTree(pts.astype(np.float64))
    d_ref, _ = tree.query(q.astype(np.float64), workers=-1)
    d_mine = np.linalg.norm(q.astype(np.float64) - res.neighbor_points.astype(np.float64), axis=1)
    np.testing.assert_allclose(d_mine, d_ref, rtol=1e-5, atol=1e-7)
    # normals: compare 2000 of them with the numpy restatement
    sel = rng.choice(131072, 2000, replace=False)
    _, nb = tree.query(res.neighbor_points[sel].astype(np.float64), k=11, workers=-1)
    d = pts[nb[:, 1:].reshape(-1)].reshape(-1, 10, 3) - res.neighbor_points[sel][:, None, :]
    cov = (d[:, :, :, None] * d[:, :, None, :]).mean(axis=1)
    _, _, vh = np.linalg.svd(cov)
    dots = np.abs((vh[:, 2, :] * res.neighbor_normals[sel]).sum(-1))
    assert np.mean(dots > 1 - 1e-3) > 0.98


def test_cfg5_projective_128x4096_20_iterations(b200, orc, syn):
    """BASELINE config 5 shape: 128x4096 vertex-map input, projective map, 20 alignments forced
    (threshold_delta_pose = 0).  GPU vs the CPU oracle on identical frames.  Tolerance: strict on the first
    registered frame; 3e-4 relative translation on the second -- the unmodified reference moves by 3.2e-4 on the
    first and 1.05e-3 on the second frame under 1-ulp input noise (tests/golden/sensitivity.json,
    cfg5_proj_128x4096_20it: its float32 normal maps amplify the last bit)."""
    H, W = 128, 4096
    algo = _make(b200, "projective", H, W, "vertex_map", 20, thr=0.0)
    ocfg = orc.ICPConfig(max_num_alignments=20, data_key="vertex_map", local_map="projective", local_map_size=20,
                         scheme="geman_mcclure", sigma=0.3, threshold_delta_pose=0.0)
    torch.set_num_threads(1)   # deterministic closest-wins scatter in the oracle's index_put_
    ref = orc.ICPFrameToModelOracle(ocfg, orc.Projector(H, W))
    pa = pb = None
    for k in range(3):
        vm = torch.from_numpy(syn.vertex_map_from_scan(syn.scan(k, H, W), H, W))
        da, db = {"vertex_map": vm.cuda(), "init_rpose": pa}, {"vertex_map": vm, "init_rpose": pb}
        algo.process_next_frame(da)
        ref.process_next_frame(db)
        if k == 0:
            continue
        assert int(algo.last_info[0]) == 20
        dt, ang = pose_errors(da["odometry_pose"], db["odometry_pose"])
        assert dt <= (1e-4 if k == 1 else relaxed_tolerance("cfg5_proj_128x4096_20it", 3e-4)) and ang <= 1e-5, (k, dt, ang)
        pa, pb = da["odometry_pose"].astype(np.float64), db["odometry_pose"].astype(np.float64)


def test_nan_rows_and_nan_pixels_match_oracle(b200, orc, syn):
    """remove_nan / modify_nan_pmap (utils.py:169-196): NaN rows are dropped from the point layouts, NaN pixels
    are zeroed in the vertex-map layout; poses follow the oracle fed with the same corrupted inputs.  Tolerances from the
    reference's own sensitivity to the last input bit (tests/golden/sensitivity.json): the small kd case (voxel 0.4
    subsample of a 32x512 scan, 8 fixed iterations) moves by 1.45e-3, the projective one by 1.9e-5 -- 6e-4 and the
    north star's 1e-4 respectively."""
    H, W = 32, 512
    tol = {"ndarray": relaxed_tolerance("nan_kd_ndarray_32x512", 6e-4), "vertex_map": 1e-4}
    for layout, key in (("ndarray", "numpy_pc"), ("vertex_map", "vertex_map")):
        lm = "kdtree" if layout == "ndarray" else "projective"
        algo = _make(b200, lm, H, W, key, 8, lm_size=4, thr=0.0)
        ref = orc.ICPFrameToModelOracle(orc.ICPConfig(max_num_alignments=8, data_key=key, local_map=lm, local_map_size=4,
                                                      scheme="geman_mcclure", sigma=0.3, threshold_delta_pose=0.0), orc.Projector(H, W))
        pa = pb = None
        for k in range(3):
            pc = syn.scan(k, H, W).copy()
            pc[5::97] = np.nan
            if layout == "ndarray":
                pc, _ = orc.grid_sample(pc[~np.isnan(pc).any(1)], 0.4)
                pc = pc.copy()
                pc[3::41, 1] = np.nan
                da, db = {"numpy_pc": pc.copy()}, {"numpy_pc": pc.copy()}
            else:
                vm = torch.from_numpy(syn.vertex_map_from_scan(pc, H, W))
                da, db = {"vertex_map": vm.clone()}, {"vertex_map": vm.clone()}
            da["init_rpose"], db["init_rpose"] = pa, pb
            algo.process_next_frame(da)
            ref.process_next_frame(db)
            if k == 0:
                continue
            dt, ang = pose_errors(da["odometry_pose"], db["odometry_pose"])
            assert dt <= tol[layout] and ang <= 1e-5, (layout, k, dt, ang)
            if layout == "ndarray":
                assert not np.isnan(da["odometry_pc"]).any()
                assert da["odometry_pc"].shape == db["odometry_pc"].shape
            pa, pb = da["odometry_pose"].astype(np.float64), db["odometry_pose"].astype(np.float64)


def test_empty_and_degenerate_inputs(b200):
    with pytest.raises(AssertionError):
        b200.grid_sample(np.zeros((0, 3), np.float32), 0.3)
    with pytest.raises(AssertionError):
        b200.grid_sample(np.zeros((10, 2), np.float32), 0.3)
    # all points in one voxel -> exactly one sample, index 0
    s, i = b200.grid_sample(np.full((1000, 3), 0.01, np.float32), 0.3)
    assert s.shape == (1, 3) and i.tolist() == [0]
    # projection of points that all fall outside the image / are null -> all-zero map
    proj = b200.SphericalProjector(height=8, width=64, up_fov=3.0, down_fov=-24.0)
    up = np.tile(np.array([[0.0, 0.0, 5.0]], np.float32), (100, 1))      # straight up: outside the vertical FOV
    assert np.all(proj.build_projection_map(np.concatenate([up, np.zeros((10, 3), np.float32)])[None]) == 0)
    # a kd map searched before any update is a state error, not a crash
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig())
    lm.init()
    with pytest.raises(RuntimeError):
        lm.nearest_neighbor_search(np.zeros((4, 3), np.float32))
    # first frame with an empty point cloud
    algo = _make(b200, "kdtree", 16, 256, "numpy_pc", 4)
    with pytest.raises(AssertionError):
        algo.process_next_frame({"numpy_pc": np.zeros((0, 3), np.float32)})


def test_odometry_reinit_is_clean(b200, syn):
    """init() between sequences (slam.py:106) resets map, poses and frame counter."""
    algo = _make(b200, "kdtree", 32, 512, "numpy_pc", 8, lm_size=4)
    fr = _frames(syn, b200.grid_sample, "ndarray", 32, 512, 0.4)
    a = _drive(algo, fr, 4)
    algo.init()
    b = _drive(algo, fr, 4)
    np.testing.assert_array_equal(a, b)
    assert algo.get_relative_poses().shape == (4, 4, 4)


def test_a1_grid_sample_hashes_beyond_the_compact_sort_keys(b200, orc, syn):
    """The subsample sorts on 40-bit biased keys (5 radix passes); hashes outside [-2^39, 2^39) -- voxel coordinates
    beyond ~3e6 -- are detected on the device and the call is repeated on the raw 64-bit keys.  Bit-exact either way,
    through pls_grid_sample and through the fused pls_process_frame_grid_sample."""
    import ctypes as C
    from pylidar_slam_b200 import _lib
    rng = np.random.RandomState(12)
    base = (rng.randn(50000, 3) * np.array([30.0, 30.0, 3.0])).astype(np.float32)
    for offset, voxel in ((0.0, 0.3), (4.0e5, 0.3), (-2.5e6, 0.5), (3.0e4, 0.001)):
        pts = (base + np.float32(offset)).astype(np.float32)
        h = orc.voxel_hashes(orc.voxel_coords(pts, voxel))
        if offset != 0.0:
            assert np.abs(h).max() >= 2 ** 39, "this case is meant to overflow the compact keys"
        s_ref, i_ref = orc.grid_sample(pts, voxel)
        s, i = b200.grid_sample(pts, voxel)
        np.testing.assert_array_equal(i, i_ref)
        np.testing.assert_array_equal(s, s_ref)
    # mixed: a frame whose hashes straddle the 40-bit range, then a regular one on the same context
    pts = np.concatenate([base[:1000], base[1000:2000] + np.float32(1e6)]).astype(np.float32)
    for cloud in (pts, base):
        s_ref, i_ref = orc.grid_sample(cloud, 0.3)
        s, i = b200.grid_sample(cloud, 0.3)
        np.testing.assert_array_equal(i, i_ref)
    # fused path: frame 0 only initialises the map; info[4] = number of samples
    far = (syn.scan(0, 32, 512) + np.float32(5.0e5)).astype(np.float32)
    algo = _make(b200, "kdtree", 32, 512, "input_data", 4, lm_size=4)
    pose, params, info, has = np.zeros((4, 4), np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    algo.ctx.call("pls_process_frame_grid_sample", _lib.ptr(far), far.shape[0], 0.3, _lib.INPUT_TENSOR, None, _lib.ptr(pose),
                  _lib.ptr(params), C.byref(has), _lib.ptr(info))
    assert has.value == 0 and int(info[4]) == orc.grid_sample(far, 0.3)[1].shape[0]
