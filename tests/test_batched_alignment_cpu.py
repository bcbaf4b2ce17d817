"""The batched alignments without a GPU: the CPU oracles and the float64 batched reference against the goldens of the
unmodified reference (tests/golden/batch_align.npz), the joint rules the solve kernel applies (gn_device.cuh, compiled
for the host through tests/batch_harness.cu) against the same goldens, and the mirrors' [B,N,3] host logic through a
stand-in of the C ABI."""
import ctypes as C
import logging
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import batch_align_reference as bar
from oracle import icp_oracle as orc
from oracle import next_rows_oracle as nxt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
SCHEME_IDS = {"default": 0, "least_square": 1, "huber": 2, "exp": 3, "neighborhood": 4, "geman_mcclure": 5,
              "square_geman_mcclure": 6, "cauchy": 7}
STATUS = {0: "ok", 3: "singular", 4: "tiny"}


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(ROOT, "tests", "golden", "batch_align.npz"))


@pytest.fixture(scope="module")
def bh():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    out_dir = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "batch_harness.so")
    deps = [os.path.join(ROOT, "tests", "batch_harness.cu")] + \
        [os.path.join(ROOT, "pylidar_slam_b200", "csrc", f) for f in ("gn_device.cuh", "pose_device.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([NVCC, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
                               "-o", so, deps[0]])
    lib = C.CDLL(so)
    lib.bh_align_batch.restype = C.c_int
    return lib


def _data(g, prefix, dt, B=None):
    return [np.ascontiguousarray(g[f"{prefix}_{k}"][:B], dt) for k in ("ref", "tgt", "nrm")]


def harness(bh, cost, ref, tgt, nrm, scheme, sigma, max_iters=1, norm_stop=1e-3, x0=None):
    B, n, dt = tgt.shape[0], tgt.shape[1], tgt.dtype
    x, dT, loss, it = np.zeros((B, 6), dt), np.zeros((B, 16), dt), np.zeros((B, n), dt), C.c_int(0)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    x0 = None if x0 is None else np.ascontiguousarray(x0, dt)
    st = bh.bh_align_batch(0 if cost == "plane" else 1, int(dt == np.float64), p(ref), p(tgt),
                           p(nrm) if cost == "plane" else None, C.c_int64(B), C.c_int64(n), SCHEME_IDS[scheme],
                           C.c_double(sigma), max_iters, C.c_double(norm_stop), p(x0), p(x), p(dT), p(loss), C.byref(it))
    return STATUS[st], x, dT.reshape(B, 4, 4), loss, it.value


def _close32(x, gx, gx64):
    """float32 reference values: its own float32 error (against float64 on the same data) twice, plus 2e-4 relative."""
    return (np.abs(x - gx) <= 2e-7 + 2e-4 * np.abs(gx) + 2 * np.abs(gx - gx64)).all()


# ------------------------------------------------------------------------------------------ oracles vs goldens
@pytest.mark.parametrize("cost", ["plane", "point"])
def test_cpu_oracles_match_the_batch_goldens(g, cost):
    """icp_oracle.gauss_newton_p2plane / next_rows_oracle.align_p2point restate GaussNewton.compute for any B."""
    def run(ref, tgt, nrm, sch, iters, stop, x0=None):
        r, t = torch.from_numpy(ref), torch.from_numpy(tgt)
        if cost == "plane":
            x, loss, st = orc.gauss_newton_p2plane(r, t, torch.from_numpy(nrm), sch, 0.3, iters, stop,
                                                   None if x0 is None else torch.from_numpy(x0))
        else:
            _, x, loss, st = nxt.align_p2point(r, t, sch, 0.3, iters, stop, None if x0 is None else torch.from_numpy(x0))
        return x.numpy(), loss.numpy(), st
    for dn, dt in (("f32", np.float32), ("f64", np.float64)):
        tol = dict(rtol=1e-4, atol=1e-6) if dt == np.float32 else dict(rtol=1e-8, atol=1e-12)
        for i, sch in enumerate(SCHEMES):
            ref, tgt, nrm = _data(g, "ba_sch", dt, 3 + i % 3)
            x, loss, st = run(ref, tgt, nrm, sch, 1, 1e-3)
            np.testing.assert_allclose(x, g[f"ba_sch_{cost}_{sch}_{dn}_x"], **tol)
        ref, tgt, nrm = _data(g, f"ba_multi_{cost}", dt)
        for k in ((1,) if (cost, dn) == ("point", "f32") else (1, 3, 8)):   # float32 point-to-point drifts (GPU test)
            x, _, _ = run(ref, tgt, nrm, "geman_mcclure", k, 1e-6)
            np.testing.assert_allclose(x, g[f"ba_multi_{cost}_{dn}_x"][k - 1], **tol)
    ref, tgt, nrm = _data(g, "ba_degen", np.float64)
    with pytest.raises(RuntimeError, match="Invalid Jacobian"):
        run(ref, tgt, nrm, "default", 1, 1e-3)


def test_float64_batched_reference_matches_the_goldens(g):
    for cost in ("plane", "point"):
        for i, sch in enumerate(SCHEMES):
            ref, tgt, nrm = _data(g, "ba_sch", np.float64, 3 + i % 3)
            st, x, it, loss = bar.gn_align_batch_f64(ref, tgt, nrm if cost == "plane" else None, sch, 0.3)
            assert st == "ok" and it == 1
            np.testing.assert_allclose(x, g[f"ba_sch_{cost}_{sch}_f64_x"], rtol=1e-9, atol=1e-13)
            np.testing.assert_allclose(loss, g[f"ba_sch_{cost}_{sch}_f64_loss"], rtol=1e-9, atol=1e-16)
        ref, tgt, nrm = _data(g, f"ba_multi_{cost}", np.float64)
        for k in range(1, 9):
            st, x, _, _ = bar.gn_align_batch_f64(ref, tgt, nrm if cost == "plane" else None, "geman_mcclure", 0.3, k, 1e-6)
            assert st == "ok"
            np.testing.assert_allclose(x, g[f"ba_multi_{cost}_f64_x"][k - 1], rtol=1e-9, atol=1e-13)
        ref, tgt, nrm = _data(g, "ba_degen", np.float64)
        assert bar.gn_align_batch_f64(ref, tgt, nrm if cost == "plane" else None, "default", 0.5)[0] == "singular"
        t = g["ba_allzero_tgt"]
        st, x, it, _ = bar.gn_align_batch_f64(t, t, g["ba_zero_nrm"] if cost == "plane" else None, "huber", 0.3, 3)
        assert st == "tiny" and it == 1 and not x.any()
    ref, tgt, nrm = _data(g, "ba_zero", np.float64)
    st, x, _, _ = bar.gn_align_batch_f64(ref, tgt, nrm, "default", 0.3, 2, 1e-9)
    assert st == "ok"
    np.testing.assert_allclose(x, g["ba_zero_plane_default_f64_x"], rtol=1e-9, atol=1e-13)
    assert bar.gn_align_batch_f64(ref, tgt, nrm, "geman_mcclure", 0.3, 2, 1e-9)[0] == "singular"
    assert bar.gn_align_batch_f64(ref, tgt, None, "default", 0.5, 2)[0] == "singular"


# ------------------------------------------------------------------------------------------ the joint rules on the host
@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_joint_rules_compiled_for_the_host_match_the_goldens(bh, g, dn):
    dt = np.float32 if dn == "f32" else np.float64
    for cost in ("plane", "point"):
        for i, sch in enumerate(SCHEMES):
            ref, tgt, nrm = _data(g, "ba_sch", dt, 3 + i % 3)
            st, x, dT, loss, it = harness(bh, cost, ref, tgt, nrm, sch, dt(0.3))
            key = f"ba_sch_{cost}_{sch}"
            assert st == "ok" and it == 1
            if dt == np.float64:
                np.testing.assert_allclose(x, g[f"{key}_f64_x"], rtol=1e-9, atol=1e-13)
                np.testing.assert_allclose(dT, g[f"{key}_f64_dT"], atol=1e-12)
            else:
                assert _close32(x, g[f"{key}_f32_x"], g[f"{key}_f64_x"]), key
        ref, tgt, nrm = _data(g, f"ba_multi_{cost}", dt)
        for k in ((1,) if (cost, dn) == ("point", "f32") else (1, 2, 5, 8)):
            st, x, _, _, it = harness(bh, cost, ref, tgt, nrm, "geman_mcclure", dt(0.3), k, 1e-6)
            gx, gx64 = g[f"ba_multi_{cost}_{dn}_x"][k - 1], g[f"ba_multi_{cost}_f64_x"][k - 1]
            assert st == "ok"
            assert (_close32(x, gx, gx64) if dt == np.float32 else np.allclose(x, gx, rtol=1e-8, atol=1e-12)), (cost, k)
        # the joint stop: all elements run until |dx| over the batch is small -- the same count as the reference
        xs = g[f"ba_multi_plane_{dn}_x"]
        ref_iters = 1 + next(k for k in range(7) if np.array_equal(xs[k], xs[7]))
        ref, tgt, nrm = _data(g, "ba_multi_plane", dt)
        assert abs(harness(bh, "plane", ref, tgt, nrm, "geman_mcclure", dt(0.3), 8, 1e-6)[4] - ref_iters) <= 1
    # guards
    ref, tgt, nrm = _data(g, "ba_degen", dt)
    for cost in ("plane", "point"):
        assert harness(bh, cost, ref, tgt, nrm, "default", 0.5)[0] == "singular"
        t = np.ascontiguousarray(g["ba_allzero_tgt"], dt)
        st, x, dT, loss, it = harness(bh, cost, t, t, _data(g, "ba_zero", dt)[2], "huber", dt(0.3), 3)
        assert st == "tiny" and it == 1 and not x.any() and not loss.any()
        assert np.array_equal(dT, g[f"ba_allzero_{cost}_{dn}_dT"])
    ref, tgt, nrm = _data(g, "ba_zero", dt)
    st, x, _, _, _ = harness(bh, "plane", ref, tgt, nrm, "default", dt(0.3), 2, 1e-9)
    assert st == "ok" and (np.allclose(x, g[f"ba_zero_plane_default_{dn}_x"], rtol=1e-9, atol=1e-13) if dt == np.float64
                           else _close32(x, g["ba_zero_plane_default_f32_x"], g["ba_zero_plane_default_f64_x"]))
    assert harness(bh, "plane", ref, tgt, nrm, "geman_mcclure", dt(0.3), 2, 1e-9)[0] == "singular"


def test_joint_rules_at_one_element_are_the_single_alignment(bh, g):
    """B = 1 through the joint rules equals the single path's host replica (tests/host_harness.cu's align_host
    restates gn_solve_kernel of one element) bit for bit: the joint sums of one element are its own."""
    ref, tgt, nrm = _data(g, "ba_sch", np.float32, 1)
    for sch in SCHEMES:
        a = harness(bh, "plane", ref, tgt, nrm, sch, np.float32(0.3), 4, 1e-9)
        b = bar.gn_align_batch_f64(ref, tgt, nrm, sch, float(np.float32(0.3)), 4, 1e-9, f32=True)
        assert a[0] == b[0] == "ok" and a[4] == b[2]
        assert _close32(a[1], b[1].astype(np.float32), b[1])


# ------------------------------------------------------------------------------------------ the mirrors' host logic
@pytest.fixture
def stand_in(monkeypatch):
    """FakeContext (tests/dryrun_next_rows.py) plus the two batch entry points, answered from the CPU oracles."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class BatchFakeContext(dry.FakeContext):
        def call(self, name, *a):
            calls.append(name)
            return getattr(self, name)(*a)

        def _batch(self, cost, ref, tgt, nrm, B, n, is64, scheme, sigma, max_iters, norm_stop, x0, dT, x, loss, iters):
            dt = np.float64 if is64 else np.float32
            r, t = (torch.from_numpy(dry.arr(p, (B, n, 3), dt).copy()) for p in (ref, tgt))
            x0t = None if not x0 else torch.from_numpy(dry.arr(x0, (B, 6), dt).copy())
            try:
                if cost == "plane":
                    m = torch.from_numpy(dry.arr(nrm, (B, n, 3), dt).copy())
                    xo, lo, status = orc.gauss_newton_p2plane(r, t, m, dry.SCHEME_NAMES[scheme], sigma, max_iters,
                                                              norm_stop, x0t)
                else:
                    _, xo, lo, status = nxt.align_p2point(r, t, dry.SCHEME_NAMES[scheme], sigma, max_iters, norm_stop, x0t)
            except orc.SingularHessian:
                return _lib.check(None, _lib.PLS_E_SINGULAR)
            dry.arr(dT, (B, 4, 4), dt)[:] = orc.build_pose_matrix(xo).numpy()
            dry.arr(x, (B, 6), dt)[:] = xo.numpy()
            dry.arr(loss, (B, n), dt)[:] = lo.numpy()
            if status == "tiny_residual":
                return _lib.check(None, _lib.PLS_W_TINY_RESIDUAL)

        def pls_align_p2plane_batch(self, ref, tgt, nrm, B, n, *rest):
            return self._batch("plane", ref, tgt, nrm, B, n, *rest)

        def pls_align_p2point_batch(self, ref, tgt, B, n, *rest):
            return self._batch("point", ref, tgt, None, B, n, *rest)

    monkeypatch.setattr(_lib, "Context", BatchFakeContext)
    monkeypatch.setattr(common, "_default_ctx", BatchFakeContext())
    import pylidar_slam_b200 as b200
    return b200, calls


def test_mirrors_batch_host_logic(stand_in, g, caplog):
    b200, calls = stand_in
    ref, tgt, nrm = _data(g, "ba_x0", np.float32)
    gn = dict(scheme="huber", sigma=0.3, max_iters=3, norm_stop_criterion=1e-9)
    plane = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=gn))
    point = b200.GaussNewtonPointToPointAlignment(b200.GNPointToPointConfig(gauss_newton_config=gn))
    for cost, run in (("plane", lambda **k: plane.align(ref, tgt, nrm, **k)), ("point", lambda **k: point.align(ref, tgt, **k))):
        for form, init in (("vec", g["ba_x0_x0"]), ("mat", g["ba_x0_mats"])):
            dT, x, loss = run(initial_estimate=init)
            assert dT.shape == (3, 4, 4) and x.shape == (3, 6) and loss.shape == (3, 300) and x.dtype == np.float32
            if cost == "plane":   # three float32 point-to-point steps amplify rounding differences (GPU test)
                np.testing.assert_allclose(x, g[f"ba_x0_{cost}_{form}_x"], rtol=1e-4, atol=1e-6)
        assert calls[-1] == f"pls_align_p2{cost}_batch"
        dT, x, loss = run(initial_estimate=torch.from_numpy(g["ba_x0_x0"]))
        assert isinstance(x, np.ndarray)
    # torch inputs come back as torch tensors; float64 stays float64
    dT, x, loss = plane.align(*(torch.from_numpy(a.astype(np.float64)) for a in (ref, tgt, nrm)))
    assert isinstance(x, torch.Tensor) and x.dtype == torch.float64 and tuple(loss.shape) == (3, 300)
    # B = 1 keeps the single entry point
    plane.align(ref[:1], tgt[:1], nrm[:1])
    assert calls[-1] == "pls_align_p2plane"
    # shapes, masks, initial estimates of the wrong batch
    with pytest.raises(AssertionError):
        plane.align(ref[:2], tgt, nrm)
    with pytest.raises(AssertionError):
        point.align(ref, tgt, initial_estimate=np.zeros((2, 6), np.float32))
    with pytest.raises(RuntimeError, match="broadcast shape \\[3, 3, 300, 6\\]"):
        plane.align(ref, tgt, nrm, mask=np.ones((3, 300, 1), np.float32))
    with pytest.raises(AssertionError):
        point.align(ref, tgt, mask=np.ones((1, 300, 1), np.float32))
    # the warning and the error
    t = np.ascontiguousarray(g["ba_allzero_tgt"], np.float32)
    with caplog.at_level(logging.WARNING):
        _, x, _ = plane.align(t, t, nrm)
    assert "residual norm is lower" in caplog.text and not x.any()
    ref, tgt, nrm = _data(g, "ba_degen", np.float32)
    with pytest.raises(RuntimeError, match="Invalid Jacobian in Gauss Newton minimization"):
        point.align(ref, tgt)
