"""The kernels beside the odometry hot path at their launch edges, through the C ABI, against the float64 references of
oracle/next_rows_reference.py (pinned on the CPU by test_next_rows_reference_cpu.py):

  * training loss (training.cu): blocks per batch element = min(ceil(HW / 256), ceil(528 / B)); the finalize kernel's
    warp w serves elements w, w + 8, ...; B <= 64.  HW at 256 k +- 1 and at that cap +- 1 for B in 1 .. 64;
  * normal map (projmap.cu): 32 x 8 tiles with a halo of ksize / 2, bit for bit against the float32 emulation;
  * stand-alone Gauss-Newton alignments (gn.cu): at most 264 blocks of 256, so the grid stride loops from n = 67 585;
  * Procrustes (registration.cu): at most 528 blocks, so the grid stride loops from n = 135 169.

Each test prints `WORST <kernel> <deviation / bound>` (pytest -s) so that the margins can be reported."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import next_rows_reference as nrr

pytestmark = pytest.mark.gpu
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
U64 = 2.0 ** -53


@pytest.fixture(scope="module")
def ctx():
    from pylidar_slam_b200 import _lib
    c = _lib.Context()
    yield c
    c.close()


def _ptr(a):
    from pylidar_slam_b200 import _lib
    return _lib.ptr(a)


# ------------------------------------------------------------------------------------------ training loss
def _loss_shapes(B):
    """(H, W) with ceil(HW / 256) at the cap - 1 (even W: the tie probe), above the cap (1 row, odd W: the grid
    stride loops) and at the cap with a partial last block (odd W)."""
    cap = -(-528 // B)
    out = [(8, 32 * (cap - 1))] if cap > 1 else []
    out.append((1, 256 * cap + 1))
    hw = 256 * cap - 1
    d = next((d for d in range(3, 64, 2) if hw % d == 0 and hw // d >= 8), 1)
    out.append((d, hw // d))
    return out


LOSS_CASES = [(B, H, W) for B in (1, 2, 7, 8, 9, 17, 63, 64) for H, W in _loss_shapes(B)] + \
             [(2, 1, 255), (2, 3, 85), (7, 1, 257), (8, 16, 16)]


def _run_loss(ctx, s, B, H, W, scheme, use_params):
    out_loss = np.full(1, np.nan, np.float32)
    pb = np.full(B, np.nan, np.float32)
    gm = np.full((B, 4, 4), np.nan, np.float32)
    gp = np.full((B, 6), np.nan, np.float32)
    ctx.call("pls_p2plane_loss", _ptr(s["vt"]), _ptr(s["vr"]), _ptr(s["nr"]), None if use_params else _ptr(s["mats"]),
             _ptr(s["params"]) if use_params else None, B, H, W, 3.0, -24.0, nrr.SCHEMES[scheme], 0.5,
             _ptr(out_loss), _ptr(pb), _ptr(gm), _ptr(gp) if use_params else None)
    return float(out_loss[0]), pb, gm, gp


@pytest.mark.parametrize("B,H,W", LOSS_CASES, ids=[f"B{b}-{h}x{w}" for b, h, w in LOSS_CASES])
def test_training_loss_at_block_and_batch_edges(ctx, B, H, W):
    """Loss, per-element losses and both gradients against p2plane_loss_f64 within the float32-transform bound, with
    pose matrices and with pose parameters.  Elements differ by far more than 100 times their tolerance, so a finalize
    loop that mixes them up fails; outputs start as NaN, so one it leaves unwritten fails too."""
    s = nrr.loss_scene(B, H, W, seed=1000 * B + H + W)
    k = LOSS_CASES.index((B, H, W))
    worst = 0.0
    for scheme in (SCHEMES[k % 7], SCHEMES[(k + 3) % 7]):
        for use_params in (False, True):
            mats = np.stack([nrr.build_pose(s["params"][b]) for b in range(B)]) if use_params else s["mats"].astype(np.float64)
            r = nrr.p2plane_loss_f64(s["vt"], s["vr"], s["nr"], mats, H, W, 3.0, -24.0, scheme, 0.5,
                                     params=s["params"] if use_params else None, transform_ulps=8.0 if use_params else 4.0)
            loss, pb, gm, gp = _run_loss(ctx, s, B, H, W, scheme, use_params)
            lb = r["loss_per_batch"]
            tol_b = r["loss_bound"] + 1e-12 * np.abs(lb) + 2 * nrr.U * np.abs(lb)
            tol_g = r["grad_mats_bound"] + nrr.U * np.abs(r["grad_mats"]) + 1e-30
            assert np.all(np.abs(pb - lb) <= tol_b), (scheme, use_params, np.abs(pb - lb) / tol_b)
            assert np.all(np.abs(gm - r["grad_mats"]) <= tol_g), (scheme, use_params, float((np.abs(gm - r["grad_mats"]) / tol_g).max()))
            assert abs(loss - r["loss"]) <= tol_b.mean() + 2 * nrr.U * abs(r["loss"]), (scheme, loss, r["loss"])
            worst = max(worst, float((np.abs(pb - lb) / tol_b).max()), float((np.abs(gm - r["grad_mats"]) / tol_g).max()))
            if use_params:
                tol_p = r["grad_params_bound"] + nrr.U * np.abs(r["grad_params"]) + 1e-30
                assert np.all(np.abs(gp - r["grad_params"]) <= tol_p), (scheme, np.abs(gp - r["grad_params"]) / tol_p)
                worst = max(worst, float((np.abs(gp - r["grad_params"]) / tol_p).max()))
            if B > 1:  # every pair of elements is told apart by > 100x its tolerance
                v = np.concatenate([lb[:, None], r["grad_mats"][:, :3].reshape(B, -1)], 1)
                t = np.concatenate([tol_b[:, None], tol_g[:, :3].reshape(B, -1)], 1)
                sep = (np.abs(v[:, None] - v[None]) / t[:, None]).max(2)
                assert (sep + np.eye(B) * 1e9).min() > 100, scheme
            if s["tie"] is not None:  # the lower index won the bit-identical range tie
                assert r["winner"][0][r["pixel"][0][s["tie"][0]]] == s["tie"][0]
    print(f"WORST loss {B}x{H}x{W} {worst:.3g}")


def test_training_loss_tie_probe_decides_the_loss(ctx):
    """The tie probe on its own: swapping the two points (so that the other one has the lower index) changes the
    kernel's loss by more than 100 times the tolerance, the way the reference says."""
    B, H, W = 3, 8, 64
    s = nrr.loss_scene(B, H, W, seed=77)
    i1, i2 = s["tie"]
    sw = dict(s, vt=s["vt"].copy())
    v = sw["vt"].reshape(B, 3, H * W)
    v[0][:, [i1, i2]] = v[0][:, [i2, i1]]
    for scheme in SCHEMES:
        r = nrr.p2plane_loss_f64(s["vt"], s["vr"], s["nr"], s["mats"], H, W, 3.0, -24.0, scheme, 0.5)
        r2 = nrr.p2plane_loss_f64(sw["vt"], s["vr"], s["nr"], s["mats"], H, W, 3.0, -24.0, scheme, 0.5)
        _, pb, _, _ = _run_loss(ctx, s, B, H, W, scheme, False)
        _, pb2, _, _ = _run_loss(ctx, sw, B, H, W, scheme, False)
        tol = r["loss_bound"][0] + 2 * nrr.U * abs(r["loss_per_batch"][0])
        assert abs(pb[0] - r["loss_per_batch"][0]) <= tol and abs(pb2[0] - r2["loss_per_batch"][0]) <= tol, scheme
        assert abs(r["loss_per_batch"][0] - r2["loss_per_batch"][0]) > 100 * tol, scheme


def test_training_loss_rejects_65_elements(ctx):
    s = nrr.loss_scene(2, 4, 32, seed=5)
    big = {k: np.ascontiguousarray(np.concatenate([s[k]] * 33)[:65]) for k in ("vt", "vr", "nr", "params", "mats")}
    with pytest.raises(AssertionError, match="batch"):
        _run_loss(ctx, big, 65, 4, 32, "default", False)
    _run_loss(ctx, {k: v[:64] for k, v in big.items()}, 64, 4, 32, "default", False)


def test_training_loss_module_computes_missing_normal_maps(ctx):
    """_PointToPlaneLossModule without a normal map: the loss of the K3 normals (ksize 5) of the reference maps."""
    import pylidar_slam_b200 as b200
    B, H, W = 3, 16, 96
    s = nrr.loss_scene(B, H, W, seed=11)
    nm = nrr.normal_map_f32_emulated(s["vr"], 5)
    for scheme in ("geman_mcclure", "neighborhood"):
        mod = b200._PointToPlaneLossModule(b200.PointToPlaneLossConfig(least_square_scheme=dict(scheme=scheme, sigma=0.5)),
                                           b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0), b200.Pose("euler"))
        vm = torch.from_numpy(np.stack([s["vr"], s["vt"]], 1)).cuda()
        x = torch.from_numpy(s["params"]).cuda().requires_grad_(True)
        dd = {"vertex_map": vm, "pose_params": x}
        loss, dd = mod(dd)
        loss.backward()
        assert np.array_equal(dd["normal_map"][:, 0].cpu().numpy().view(np.uint32), nm.view(np.uint32))
        mats = np.stack([nrr.build_pose(s["params"][b]) for b in range(B)])
        r = nrr.p2plane_loss_f64(s["vt"], s["vr"], nm, mats, H, W, 3.0, -24.0, scheme, 0.5, params=s["params"], transform_ulps=8.0)
        tol = r["loss_bound"].mean() + 2 * nrr.U * abs(r["loss"])
        assert abs(float(loss.detach()) - r["loss"]) <= tol, (scheme, float(loss.detach()), r["loss"])
        tol_p = r["grad_params_bound"] + nrr.U * np.abs(r["grad_params"])
        assert np.all(np.abs(x.grad.cpu().numpy() - r["grad_params"]) <= tol_p), scheme


# ------------------------------------------------------------------------------------------ normal map
def _normal_vmap(B, H, W, seed):
    """Smooth surfaces seen from the sensor, column scales from 1e-4 to 1 (so that |det| crosses 1e-6), null pixels at
    random, on tile halo columns / rows and on the image border."""
    rs = np.random.RandomState(seed)
    pc = nrr.proj_consts(H, W, 3.0, -24.0)
    row, col = np.meshgrid(np.arange(H) + 0.1, np.arange(W) + 0.1, indexing="ij")
    out = np.zeros((B, 3, H, W), np.float32)
    for b in range(B):
        rg = 10 + 3 * np.sin(col / 37.0 + b) + 2 * np.cos(row / 5.0) + rs.normal(0, 0.02, (H, W))
        p = nrr._inverse_projection(row, col, rg, pc) * np.logspace(-4, 0, W)[None, :, None]
        p[rs.rand(H, W) < 0.08] = 0.0
        halo = ((np.arange(W) % 32 == 31) | (np.arange(W) % 32 == 0))[None, :] & (rs.rand(H, W) < 0.5)
        halo |= ((np.arange(H) % 8 == 7) | (np.arange(H) % 8 == 0))[:, None] & (rs.rand(H, W) < 0.3)
        p[halo] = 0.0
        p[0, rs.rand(W) < 0.5] = 0.0
        p[:, -1][rs.rand(H) < 0.5] = 0.0
        out[b] = np.moveaxis(p, -1, 0)
    return out


@pytest.mark.parametrize("ksize", [1, 3, 5, 7, 9])
def test_normal_map_bit_exact_at_tile_edges(ctx, ksize):
    n_bits = 0
    for H in (1, 7, 8, 9, 64):
        for W in (1, 31, 32, 33, 2047, 2048):
            B = 3 if (H * W <= 64 * 33 or (H + W + ksize) % 2 == 0) else 1
            vm = _normal_vmap(B, H, W, seed=H * 7919 + W + ksize)
            out = np.full_like(vm, np.nan)
            ctx.call("pls_normal_map", _ptr(vm), B, H, W, ksize, _ptr(out))
            emu, det = nrr.normal_map_f32_emulated(vm, ksize, return_det=True)
            same = out.view(np.uint32) == emu.view(np.uint32)
            assert same.all(), (H, W, B, int((~same).sum()), np.argwhere(~same)[:5])
            n_bits += out.size
            if H == 64 and W == 2048 and ksize >= 3:  # windows on both sides of the |det| > 1e-6 test
                live = (vm[:, None] != 0).any(2)[:, 0]
                a = np.abs(det)[live]
                assert ((a > 1e-7) & (a <= 1e-6)).any() and ((a > 1e-6) & (a < 1e-5)).any()
    print(f"WORST normal_map k={ksize} 0 (bit-exact on {n_bits} values)")


@pytest.mark.parametrize("ksize", [0, 2, 4, 10, 11])
def test_normal_map_rejects_kernel_size(ctx, ksize):
    vm = np.ones((1, 3, 8, 32), np.float32)
    out = np.zeros_like(vm)
    with pytest.raises(AssertionError, match="kernel size"):
        ctx.call("pls_normal_map", _ptr(vm), 1, 8, 32, ksize, _ptr(out))


# ------------------------------------------------------------------------------------------ Gauss-Newton alignments
GN_SIZES = [1, 2, 255, 256, 257, 67583, 67584, 67585, 300007]


@functools.lru_cache(maxsize=2)
def _gn_data(n):
    rs = np.random.RandomState(n % 100003)
    tgt = rs.uniform(-20, 20, (n, 3))
    T = nrr.build_pose([0.05, -0.03, 0.02, 0.004, -0.003, 0.005])
    ref = tgt @ T[:3, :3].T + T[:3, 3] + rs.normal(0, 0.05, (n, 3))
    nrm = rs.normal(0, 1, (n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return ref, tgt, nrm


def _align(ctx, cost, ref, tgt, nrm, n, dt, scheme, sigma, max_iters=1, norm_stop=1e-3):
    x, dT, loss = np.zeros(6, dt), np.zeros(16, dt), np.full(n, np.nan, dt)
    if cost == "plane":
        ctx.call("pls_align_p2plane", _ptr(ref), _ptr(tgt), _ptr(nrm), n, int(dt == np.float64), nrr.SCHEMES[scheme],
                 sigma, max_iters, norm_stop, None, _ptr(dT), _ptr(x), _ptr(loss))
    else:
        ctx.call("pls_align_p2point", _ptr(ref), _ptr(tgt), n, int(dt == np.float64), nrr.SCHEMES[scheme], sigma,
                 max_iters, norm_stop, None, _ptr(dT), _ptr(x), _ptr(loss))
    return x.astype(np.float64), loss.astype(np.float64)


@pytest.mark.parametrize("n", GN_SIZES)
def test_gn_alignments_at_grid_stride_edges(ctx, n):
    """float64: x within 1e-10 relative of gn_step_f64; float32: x within gn_f32_step_bound (the conditioning of the
    normal equations times the float32 error of their terms).  Every per-element (w r)^2 within gn_loss_bound.
    At n = 1 and 2 the normal equations are rank-deficient: the reference's RuntimeError."""
    ref64, tgt64, nrm64 = _gn_data(n)
    worst = {}
    for cost in ("plane", "point"):
        for dt in (np.float64, np.float32):
            ref, tgt = np.ascontiguousarray(ref64, dt), np.ascontiguousarray(tgt64, dt)
            nrm = np.ascontiguousarray(nrm64, dt) if cost == "plane" else None
            args = (ref.astype(np.float64), tgt.astype(np.float64), None if nrm is None else nrm.astype(np.float64))
            for scheme in SCHEMES:
                sig = float(dt(0.3))
                if n <= 2:
                    with pytest.raises(RuntimeError, match="Invalid Jacobian"):
                        _align(ctx, cost, ref, tgt, nrm, n, dt, scheme, sig)
                    continue
                x, loss = _align(ctx, cost, ref, tgt, nrm, n, dt, scheme, sig)
                st, xr, _, lr = nrr.gn_align_f64(*args, scheme, sig)
                assert st == "ok"
                lb = nrr.gn_loss_bound(*args, np.zeros(6), scheme, sig, U64 if dt == np.float64 else nrr.U)
                e_l = float((np.abs(loss - lr) / lb).max())
                assert e_l <= 1.0, (cost, dt, scheme, e_l)
                if dt == np.float64:
                    e_x = float(np.abs(x - xr).max() / (1e-10 * np.abs(xr).max()))
                else:
                    e_x = float((np.abs(x - xr) / nrr.gn_f32_step_bound(*args, scheme, sig)).max())
                assert e_x <= 1.0, (cost, dt, scheme, np.abs(x - xr))
                key = f"{cost}-{np.dtype(dt).name}"
                worst[key] = max(worst.get(key, 0.0), e_x, e_l)
    print(f"WORST gn n={n} {worst}")


def test_gn_multi_iteration_ends_on_norm_stop(ctx):
    n = 67585
    _, tgt, nrm = _gn_data(n)
    T = nrr.build_pose([0.6, -0.4, 0.2, 0.03, -0.02, 0.05])
    ref = np.ascontiguousarray(tgt @ T[:3, :3].T + T[:3, 3] + np.random.RandomState(9).normal(0, 0.05, (n, 3)))
    # point-to-plane only: the point-to-point step (the reference's r dr/dx Jacobian) converges too slowly to reach a stop
    for cost in ("plane",):
        nn = nrm if cost == "plane" else None
        st, xr, iters, _ = nrr.gn_align_f64(ref, tgt, nn, "geman_mcclure", 0.3, max_iters=30, norm_stop=1e-7)
        assert st == "ok" and 2 < iters < 30, iters
        x, _ = _align(ctx, cost, ref, tgt, nn, n, np.float64, "geman_mcclure", 0.3, 30, 1e-7)
        assert np.abs(x - xr).max() <= 1e-10 * np.abs(xr).max(), (cost, np.abs(x - xr).max())
        x_at, _ = _align(ctx, cost, ref, tgt, nn, n, np.float64, "geman_mcclure", 0.3, iters, 1e-7)
        x_before, _ = _align(ctx, cost, ref, tgt, nn, n, np.float64, "geman_mcclure", 0.3, iters - 1, 1e-7)
        assert np.array_equal(x, x_at) and not np.array_equal(x, x_before), cost


# ------------------------------------------------------------------------------------------ Procrustes
def _procrustes(ctx, tgt, ref, w, dt):
    tgt, ref = np.ascontiguousarray(tgt, dt), np.ascontiguousarray(ref, dt)
    w = None if w is None else np.ascontiguousarray(w, dt)
    out = np.full(16, np.nan)
    ctx.call("pls_weighted_procrustes", _ptr(tgt), _ptr(ref), _ptr(w), len(tgt), int(dt == np.float64), _ptr(out))
    return out.reshape(4, 4), tgt, ref, w


@pytest.mark.parametrize("n", [135167, 135168, 135169, 1000003])
def test_procrustes_at_grid_stride_edges(ctx, n):
    """Well-conditioned clouds with noise, float64 and float32 data, with and without weights (a tenth of them zero):
    within 1e-12 of procrustes_f64 on the same (float32-rounded) data."""
    rs = np.random.RandomState(n % 1009)
    tgt = rs.normal(0, [12.0, 8.0, 3.0], (n, 3)) + [3.0, -2.0, 1.0]
    T = nrr.build_pose([1.5, -0.7, 0.3, 0.1, -0.2, 0.4])
    ref = tgt @ T[:3, :3].T + T[:3, 3] + rs.normal(0, 0.01, (n, 3))
    w = rs.uniform(0.1, 2.0, n)
    w[rs.rand(n) < 0.1] = 0.0
    worst = 0.0
    for dt in (np.float64, np.float32):
        for ww in (None, w):
            got, t32, r32, w32 = _procrustes(ctx, tgt, ref, ww, dt)
            exp = nrr.procrustes_f64(t32, r32, w32)
            e = float(np.abs(got - exp).max())
            assert e <= 1e-12, (dt, ww is None, e)
            worst = max(worst, e / 1e-12)
    print(f"WORST procrustes n={n} {worst:.3g}")


def test_procrustes_elongated_and_planar_clouds(ctx):
    """Exact motions of elongated clouds (sigma_2 / sigma_1 from 1e-2 to 1e-5) and planar clouds, n = 135 169: the
    kernel's error against the true motion is at most 4x LAPACK's on the same data + 1e-11.  The rotation about the
    long axis is conditioned by sigma_1 / (sigma_2 + sigma_3).  Measured on an H100 (line clouds): 9e-10 at 1e-3, 1.4e-7
    at 1e-4 and 5.9e-6 at 1e-5, against LAPACK's 7e-10, 3.9e-8 and 1.9e-6 on the same data; planar clouds stay below
    1e-14.  The former eigen-decomposition of C^T C gave 4e-4 at 1e-3 and a wrong rotation from 1e-4 on (host code)."""
    from scipy.spatial.transform import Rotation
    rs = np.random.RandomState(3)
    n = 135169
    worst = 0.0
    for ratio in (1e-2, 1e-3, 1e-4, 1e-5):
        for shape in ("line", "planar"):
            s = np.array([10.0, 10 * ratio, 5 * ratio]) if shape == "line" else np.array([10.0, 7.0, 10 * ratio])
            tgt = (rs.randn(n, 3) * s) @ Rotation.random(random_state=rs).as_matrix().T + rs.randn(3) * 5
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = Rotation.random(random_state=rs).as_matrix(), rs.randn(3)
            ref = tgt @ T[:3, :3].T + T[:3, 3]
            got, *_ = _procrustes(ctx, tgt, ref, None, np.float64)
            e_k = float(np.abs(got - T).max())
            e_l = float(np.abs(nrr.procrustes_f64(tgt, ref) - T).max())
            assert e_k <= 4 * e_l + 1e-11, (ratio, shape, e_k, e_l)
            print(f"procrustes {shape} {ratio:g}: kernel {e_k:.2e} LAPACK {e_l:.2e}")
            worst = max(worst, e_k / (4 * e_l + 1e-11))
    print(f"WORST procrustes_elongated {worst:.3g}")
