"""oracle/next_rows_reference.py pinned to what already exists, on the CPU: the goldens of the unmodified reference
(p2plane_loss.npz, the a4 normal maps and gn_* of helpers.npz, p2p_* and proc_* of next_rows.npz) and the host
restatements of the kernels' per-element code in tests/host_harness.cu.  The GPU edge tests
(test_next_rows_edges_gpu.py) then compare the kernels with these functions."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle import next_rows_reference as nrr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


@pytest.fixture(scope="module")
def hh(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    so = str(tmp_path_factory.mktemp("hh") / "host_harness.so")
    subprocess.check_call([NVCC, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
                           "-o", so, os.path.join(ROOT, "tests", "host_harness.cu")])
    lib = C.CDLL(so)
    lib.hh_align.restype = C.c_int
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------ training loss
@pytest.mark.parametrize("scheme", SCHEMES)
def test_loss_reference_matches_reference_autograd(golden_loss, scheme):
    """The reference sums 4096 float32 pixels; measured agreement is 1.4e-6 on the loss and 1e-5 on the gradients."""
    g = golden_loss
    vm, nm, x = g["vertex_map"], g["normal_map"], g["pose_params"]
    B, _, _, H, W = vm.shape
    mats = np.stack([nrr.build_pose(x[b]) for b in range(B)])
    r = nrr.p2plane_loss_f64(vm[:, 1], vm[:, 0], nm[:, 0], mats, H, W, 3.0, -24.0, scheme, 0.5, params=x)
    ref = float(g[f"{scheme}_loss"])
    assert abs(r["loss"] - ref) <= 1e-5 * abs(ref), (r["loss"], ref)
    assert abs(r["loss"] - float(g[f"{scheme}_loss_matrix"])) <= 1e-5 * abs(ref)
    gp, gm = g[f"{scheme}_grad_params"], g[f"{scheme}_grad_matrix"]
    assert np.abs(r["grad_params"] - gp).max() <= 5e-5 * np.abs(gp).max()
    assert np.abs(r["grad_mats"] - gm).max() <= 5e-5 * np.abs(gm).max()
    assert r["ambiguous"].mean() < 0.01  # 65 of 12 288 golden points sit within the float32 bands


def test_loss_pixel_terms_match_host_code(hh):
    rs = np.random.RandomState(4)
    pw, q = rs.normal(0, 5, (500, 3)).astype(np.float32), rs.normal(0, 5, (500, 3)).astype(np.float32)
    n = rs.normal(0, 1, (500, 3)).astype(np.float32)
    q[::7] = 0
    n[::11] = 0
    for scheme in SCHEMES:
        mask, c2, g = nrr.loss_pixel_terms(scheme, 0.5, pw.astype(np.float64), q.astype(np.float64), n.astype(np.float64))
        for i in range(0, 500, 3):
            out = np.zeros(5)
            hh.hh_loss_pixel(nrr.SCHEMES[scheme], C.c_double(0.5), _p(pw[i]), _p(q[i]), _p(n[i]), _p(out))
            exp = np.concatenate([[mask[i], c2[i]], g[i]])
            assert np.allclose(out, exp, rtol=1e-12, atol=1e-300), (scheme, i, out, exp)


@pytest.mark.parametrize("B,H,W", [(1, 8, 64), (2, 1, 257), (3, 16, 33), (9, 8, 64)])
def test_loss_scene_and_bounds_hold_for_the_host_kernel(hh, B, H, W):
    """The kernels' per-point code run sequentially on the CPU (hh_p2plane_loss) stays inside the reference's bounds,
    with pose matrices and with pose parameters; the tie probe moves the loss by more than 100 times its bound."""
    s = nrr.loss_scene(B, H, W, seed=B * 100 + H)
    for scheme in SCHEMES:
        for use_params in (False, True):
            mats = np.stack([nrr.build_pose(s["params"][b]) for b in range(B)]) if use_params else s["mats"].astype(np.float64)
            r = nrr.p2plane_loss_f64(s["vt"], s["vr"], s["nr"], mats, H, W, 3.0, -24.0, scheme, 0.5,
                                     params=s["params"] if use_params else None, transform_ulps=8.0 if use_params else 4.0)
            ol, pb = np.zeros(1, np.float32), np.zeros(B, np.float32)
            gm, gp = np.zeros((B, 4, 4), np.float32), np.zeros((B, 6), np.float32)
            hh.hh_p2plane_loss(_p(s["vt"]), _p(s["vr"]), _p(s["nr"]), None if use_params else _p(s["mats"]), _p(s["params"]),
                               B, H, W, C.c_float(3.0), C.c_float(-24.0), nrr.SCHEMES[scheme], C.c_float(0.5),
                               _p(ol), _p(pb), _p(gm), _p(gp))
            lb = r["loss_per_batch"]
            assert (np.abs(pb - lb) <= r["loss_bound"] + 2 * nrr.U * np.abs(lb)).all(), (scheme, pb, lb)
            assert (np.abs(gm - r["grad_mats"]) <= r["grad_mats_bound"] + nrr.U * np.abs(r["grad_mats"])).all(), scheme
            if use_params:
                assert (np.abs(gp - r["grad_params"]) <= r["grad_params_bound"] + nrr.U * np.abs(r["grad_params"])).all()
    if s["tie"] is not None:
        i1, i2 = s["tie"]
        swapped = s["vt"].copy().reshape(B, 3, H * W)
        swapped[0][:, [i1, i2]] = swapped[0][:, [i2, i1]]
        for scheme in SCHEMES:
            a = nrr.p2plane_loss_f64(s["vt"], s["vr"], s["nr"], s["mats"], H, W, 3.0, -24.0, scheme, 0.5)
            b = nrr.p2plane_loss_f64(swapped.reshape(s["vt"].shape), s["vr"], s["nr"], s["mats"], H, W, 3.0, -24.0, scheme, 0.5)
            assert a["winner"][0][a["pixel"][0][i1]] == i1
            assert abs(a["loss_per_batch"][0] - b["loss_per_batch"][0]) > 100 * a["loss_bound"][0], scheme


# ------------------------------------------------------------------------------------------ normal map
def test_fma32_is_correctly_rounded():
    rs = np.random.RandomState(1)
    a = rs.normal(0, 1, 20000).astype(np.float32)
    b = rs.normal(0, 1, 20000).astype(np.float32)
    c = rs.normal(0, 1e-7, 20000).astype(np.float32)
    # constructed midpoints: a * b = 1 + 2^-24 exactly, c = tiny -> the float64 sum rounds onto a float32 midpoint
    a[:4] = np.float32(1 + 2 ** -12)
    b[:4] = np.float32(1 + 2 ** -12)
    c[:4] = np.array([2.0 ** -80, -(2.0 ** -80), 0.0, 2.0 ** -60], np.float32)
    got = nrr.fma32(a, b, c)
    for i in list(range(8)) + list(range(8, 20000, 97)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        assert got[i] == nrr._round_fraction_to_f32(exact), i
    assert nrr._is_f32_midpoint(a[:3].astype(np.float64) * b[:3].astype(np.float64)).all() and got[0] > got[1]


def test_normal_map_emulation_reproduces_the_a4_goldens_bit_for_bit(golden_helpers):
    """The kernel matches these goldens on more than 99.99 % of the values; the emulation matches all of them."""
    g = golden_helpers
    for k, vkey, key in ((5, "a4_vmap", "a4_nmap"), (3, "a4_vmap", "a4_nmap_k3"), (5, "a4b_vmap", "a4b_nmap")):
        n = nrr.normal_map_f32_emulated(g[vkey][None], k)[0]
        assert n.dtype == np.float32 and n.shape == g[key].shape
        assert np.array_equal(n.view(np.uint32), g[key].view(np.uint32)), (key, np.mean(n == g[key]))


# ------------------------------------------------------------------------------------------ Gauss-Newton
@pytest.mark.parametrize("scheme", SCHEMES)
def test_gn_reference_matches_goldens(golden_helpers, golden_next, scheme):
    """Point-to-plane (helpers gn_*) and point-to-point (next_rows p2p_*) single steps of the reference, which solves in
    float32: 2e-4 relative on x, 1e-3 on the per-element loss, as the GPU parity tests allow."""
    g = golden_helpers
    st, x, it, loss = nrr.gn_align_f64(g["gn_ref"], g["gn_tgt"], g["gn_nrm"], scheme, float(np.float32(0.3)))
    assert st == "ok" and it == 1
    np.testing.assert_allclose(x, g[f"gn_{scheme}_delta"], rtol=2e-4, atol=2e-7)
    np.testing.assert_allclose(loss, g[f"gn_{scheme}_loss"], rtol=1e-3, atol=1e-7)
    n = golden_next
    st, x, it, loss = nrr.gn_align_f64(n["p2p_ref"], n["p2p_tgt"], None, scheme, float(np.float32(0.3)))
    rx = n[f"p2p_{scheme}_x"]
    assert np.abs(x - rx).max() <= 2e-5 * max(1.0, np.abs(rx).max())
    rl = n[f"p2p_{scheme}_loss"]
    assert np.abs(loss - rl).max() <= 1e-5 * max(1.0, np.abs(rl).max())


def test_gn_reference_multi_iteration_goldens(golden_helpers, golden_next):
    g = golden_helpers
    _, x, _, _ = nrr.gn_align_f64(g["gn_ref"], g["gn_tgt"], g["gn_nrm"], "geman_mcclure", float(np.float32(0.3)),
                                  max_iters=5, norm_stop=1e-9)
    np.testing.assert_allclose(x, g["gn_multi_x"], rtol=1e-3, atol=1e-6)
    n = golden_next
    _, x, _, loss = nrr.gn_align_f64(n["p2p_ref"].astype(np.float64), n["p2p_tgt"].astype(np.float64), None, "default", 0.5,
                                     max_iters=6, norm_stop=1e-12)
    assert np.abs(x - n["p2p_f64_x"]).max() <= 1e-9 and np.abs(loss - n["p2p_f64_loss"]).max() <= 1e-9
    assert np.abs(nrr.build_pose(x) - n["p2p_f64_dT"]).max() <= 1e-9


@pytest.mark.parametrize("cost", ["plane", "point"])
def test_gn_reference_matches_host_code_and_float32_bound(hh, cost):
    """hh_align runs gn_accumulate_kernel's per-element code sequentially: float64 x within 1e-10 relative, float32
    x within gn_f32_step_bound, every per-element loss within gn_loss_bound."""
    rs = np.random.RandomState(7)
    n = 3000
    tgt = rs.uniform(-20, 20, (n, 3))
    T = nrr.build_pose([0.05, -0.03, 0.02, 0.004, -0.003, 0.005])
    ref = tgt @ T[:3, :3].T + T[:3, 3] + rs.normal(0, 0.05, (n, 3))
    nrm = rs.normal(0, 1, (n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm = nrm if cost == "plane" else None
    for scheme in SCHEMES:
        for dt, u in ((np.float64, 2.0 ** -53), (np.float32, nrr.U)):
            a, b = np.ascontiguousarray(ref, dt), np.ascontiguousarray(tgt, dt)
            c = None if nrm is None else np.ascontiguousarray(nrm, dt)
            sig = float(dt(0.3))
            x, dT, loss = np.zeros(6, dt), np.zeros(16, dt), np.zeros(n, dt)
            st = hh.hh_align(0 if nrm is not None else 1, int(dt == np.float64), _p(a), _p(b), _p(c), C.c_int64(n),
                             nrr.SCHEMES[scheme], C.c_double(sig), 1, C.c_double(1e-3), None, _p(x), _p(dT), _p(loss))
            assert st == 0
            args = (a.astype(np.float64), b.astype(np.float64), None if c is None else c.astype(np.float64))
            _, xr, _, lr = nrr.gn_align_f64(*args, scheme, sig)
            lb = nrr.gn_loss_bound(*args, np.zeros(6), scheme, sig, u)
            assert (np.abs(loss - lr) <= lb).all(), (scheme, dt, float((np.abs(loss - lr) / lb).max()))
            if dt == np.float64:
                assert np.abs(x - xr).max() <= 1e-10 * np.abs(xr).max(), (scheme, np.abs(x - xr).max())
            else:
                bound = nrr.gn_f32_step_bound(*args, scheme, sig)
                assert (np.abs(x - xr) <= bound).all(), (scheme, np.abs(x - xr) / bound)


# ------------------------------------------------------------------------------------------ Procrustes
def test_procrustes_reference_matches_goldens(golden_next):
    g = golden_next
    pt, pr = g["proc_tgt"], g["proc_ref"]
    assert np.abs(nrr.procrustes_f64(pt, pr) - g["proc_T"]).max() <= 1e-12
    assert np.abs(nrr.procrustes_f64(pt, pr, g["proc_w"]) - g["proc_T_w"]).max() <= 1e-12
    assert np.abs(nrr.procrustes_f64(pt, g["proc_ref_mirror"]) - g["proc_T_mirror"]).max() <= 1e-12
    assert np.abs(nrr.procrustes_f64(g["proc_planar_tgt"], g["proc_planar_ref"]) - g["proc_T_planar"]).max() <= 1e-9


def test_procrustes_solve_tail_is_as_accurate_as_lapack_on_elongated_clouds(hh):
    """kabsch_from_cross (the solve kernel's code) against the exact motion, next to LAPACK on the same cross-covariance.
    Elongated clouds with sigma_2 / sigma_1 from 1e-2 to 1e-5: the rotation about the long axis is conditioned by
    sigma_1 / (sigma_2 + sigma_3), so both lose accuracy in step.  The former eigen-decomposition of C^T C squared that
    condition number: 2e-8 at 1e-2, 4e-4 at 1e-3 and a wrong rotation from 1e-4 on, against LAPACK's 2e-11 .. 6e-5."""
    from scipy.spatial.transform import Rotation
    rs = np.random.RandomState(1)
    for ratio in (1e-1, 1e-2, 1e-3, 1e-4, 1e-5):
        for shape in ("line", "planar"):
            for _ in range(10):
                s = np.array([10.0, 10 * ratio, 5 * ratio]) if shape == "line" else np.array([10.0, 7.0, 10 * ratio])
                pt = (rs.randn(2000, 3) * s) @ Rotation.random(random_state=rs).as_matrix().T + rs.randn(3) * 5
                T = np.eye(4)
                T[:3, :3], T[:3, 3] = Rotation.random(random_state=rs).as_matrix(), rs.randn(3)
                pr = pt @ T[:3, :3].T + T[:3, 3]
                mu_t, mu_r = pt.mean(0), pr.mean(0)
                Cm = np.ascontiguousarray((pr - mu_r).T @ (pt - mu_t))
                out = np.zeros(16)
                hh.hh_kabsch(_p(Cm), _p(np.ascontiguousarray(np.concatenate([mu_t, mu_r]))), _p(out))
                e_k = np.abs(out.reshape(4, 4) - T).max()
                e_l = np.abs(nrr.procrustes_f64(pt, pr) - T).max()
                assert e_k <= 4 * e_l + 1e-11, (ratio, shape, e_k, e_l)
