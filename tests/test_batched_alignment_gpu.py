"""The two Gauss-Newton alignments on a batch of B correspondence sets in one call (pls_align_p2plane_batch,
pls_align_p2point_batch and the mirrors' [B,N,3] path), on the GPU:

  * the reference's own unit test (tests/test_optimization.py: B = 2 in one call) and the batch goldens of the
    unmodified reference (tests/golden/batch_align.npz), including its warning, its RuntimeError and a zero-residual
    element beside live ones;
  * per element, bit for bit, the element's own single alignment: at max_iters = 1, and with more iterations against
    single calls of max_iters = the batch's iteration count and norm_stop = 0; an element whose own call stops earlier
    shows the coupling of the joint stop test;
  * batch edges up to 65 537 elements and point counts up to the block cap, against oracle/batch_align_reference within
    gn_f32_step_bound / gn_loss_bound; rank-deficient elements raise; results are deterministic;
  * the input forms of the mirrors."""
import ctypes as C
import logging

import numpy as np
import pytest
import torch

from oracle import batch_align_reference as bar
from oracle import next_rows_reference as nrr

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
DT = {"f32": np.float32, "f64": np.float64}


@pytest.fixture(scope="module")
def ctx():
    from pylidar_slam_b200 import _lib
    c = _lib.Context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def g():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "batch_align.npz"))


@pytest.fixture(scope="module")
def b200():
    import pylidar_slam_b200
    return pylidar_slam_b200


def _ptr(a):
    return None if a is None else a.ctypes.data


def align_batch(ctx, cost, ref, tgt, nrm, scheme, sigma, max_iters=1, norm_stop=1e-3, x0=None):
    """One pls_align_*_batch call on [B,N,3] numpy arrays -> (dT [B,16], x [B,6], loss [B,N], iterations)."""
    B, n = tgt.shape[0], tgt.shape[1]
    dt = tgt.dtype
    dT, x, loss, it = np.full((B, 16), np.nan, dt), np.full((B, 6), np.nan, dt), np.full((B, n), np.nan, dt), C.c_int(0)
    x0 = None if x0 is None else np.ascontiguousarray(x0, dt)
    args = (int(dt == np.float64), nrr.SCHEMES[scheme], float(sigma), max_iters, float(norm_stop), _ptr(x0), _ptr(dT),
            _ptr(x), _ptr(loss), C.byref(it))
    if cost == "plane":
        ctx.call("pls_align_p2plane_batch", _ptr(ref), _ptr(tgt), _ptr(nrm), B, n, *args)
    else:
        ctx.call("pls_align_p2point_batch", _ptr(ref), _ptr(tgt), B, n, *args)
    return dT, x, loss, it.value


def align_single(ctx, cost, ref, tgt, nrm, scheme, sigma, max_iters=1, norm_stop=1e-3, x0=None):
    """The single entry point on one element [N,3] -> (dT [16], x [6], loss [N])."""
    n, dt = tgt.shape[0], tgt.dtype
    dT, x, loss = np.full(16, np.nan, dt), np.full(6, np.nan, dt), np.full(n, np.nan, dt)
    x0 = None if x0 is None else np.ascontiguousarray(x0, dt)
    args = (int(dt == np.float64), nrr.SCHEMES[scheme], float(sigma), max_iters, float(norm_stop), _ptr(x0), _ptr(dT),
            _ptr(x), _ptr(loss))
    if cost == "plane":
        ctx.call("pls_align_p2plane", _ptr(np.ascontiguousarray(ref)), _ptr(np.ascontiguousarray(tgt)),
                 _ptr(np.ascontiguousarray(nrm)), n, *args)
    else:
        ctx.call("pls_align_p2point", _ptr(np.ascontiguousarray(ref)), _ptr(np.ascontiguousarray(tgt)), n, *args)
    return dT, x, loss


def _cast(g, prefix, dt, B=None):
    a = [np.ascontiguousarray(g[f"{prefix}_{k}"][:B], dt) for k in ("ref", "tgt", "nrm")]
    return a


def _check_close(dT, x, loss, g, key, dt, ref64=None, gold=None):
    """float32: the tolerances of the single path's golden tests, widened by twice the reference's own float32 error
    (its distance from the float64 result ref64 = (x, loss) on the same data) -- the reference solves in float32, this
    library in float64, and the point-to-point normal equations (Jacobian r dr/dx) amplify that difference.  A loss
    (w r)^2 may further move by what the measured pose difference moves r: |dr| <= 40 |dx| (points within 30 m).
    float64: float64 rounding.  gold overrides the golden (x, dT, loss) of `key`."""
    gx, gd, gl = gold if gold is not None else (g[f"{key}_x"], g[f"{key}_dT"], g[f"{key}_loss"])
    if dt == np.float32:
        ex = el = 0.0
        if ref64 is not None:
            ex, el = 2 * np.abs(gx - ref64[0]), 2 * np.abs(gl - ref64[1])
        ed = np.max(ex, axis=-1)[:, None, None] if ref64 is not None else 0.0
        assert (np.abs(x - gx) <= 2e-7 + 2e-4 * np.abs(gx) + ex).all(), (key, np.abs(x - gx).max())
        assert (np.abs(dT.reshape(-1, 4, 4) - gd) <= 2e-6 + ed).all(), (key, np.abs(dT.reshape(-1, 4, 4) - gd).max())
        e_r = 40 * np.abs(x - gx).max(axis=-1, keepdims=True) + 1e-6
        tol_l = 1e-9 + 1e-3 * np.abs(gl) + el + 2 * np.sqrt(np.abs(gl)) * e_r + e_r * e_r
        assert (np.abs(loss - gl) <= tol_l).all(), (key, np.abs(loss - gl).max())
    else:
        np.testing.assert_allclose(x, gx, rtol=1e-9, atol=1e-12, err_msg=key)
        np.testing.assert_allclose(dT.reshape(-1, 4, 4), gd, atol=1e-12, err_msg=key)
        np.testing.assert_allclose(loss, gl, rtol=1e-8, atol=1e-15, err_msg=key)


def _f64(g, key):
    return g[f"{key}_x"], g[f"{key}_loss"]


# ------------------------------------------------------------------------------------------ the reference's own test
def test_reference_unit_test_in_one_call(b200, golden_helpers):
    """tests/test_optimization.py of the reference: two float64 problems, scheme default, max_iters 100, norm_stop
    1e-10, solved as ONE batch of two; its bounds 1e-7 on the parameters and the loss, 1e-9 against its own estimate."""
    gh = golden_helpers
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="default", max_iters=100, norm_stop_criterion=1e-10)))
    dT, x, loss = al.align(gh["ka_ref"], gh["ka_tgt"], gh["ka_nrm"])
    assert x.dtype == np.float64 and x.shape == (2, 6) and dT.shape == (2, 4, 4) and loss.shape == (2, 100)
    assert np.abs(x - gh["ka_params"]).max() <= 1e-7
    assert np.abs(x - gh["ka_est"]).max() <= 1e-9
    assert float(np.abs(loss).sum()) <= 1e-7


# ------------------------------------------------------------------------------------------ goldens of the reference
@pytest.mark.parametrize("cost", ["plane", "point"])
@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_batch_goldens_every_scheme(ctx, g, cost, dn):
    dt = DT[dn]
    for i, sch in enumerate(SCHEMES):
        B = 3 + i % 3
        ref, tgt, nrm = _cast(g, "ba_sch", dt, B)
        dT, x, loss, it = align_batch(ctx, cost, ref, tgt, nrm, sch, dt(0.3), 1)
        assert it == 1
        _check_close(dT, x, loss, g, f"ba_sch_{cost}_{sch}_{dn}", dt, _f64(g, f"ba_sch_{cost}_{sch}_f64"))


@pytest.mark.parametrize("cost,dn", [("plane", "f32"), ("plane", "f64"), ("point", "f32"), ("point", "f64")])
def test_batch_goldens_iterations(ctx, g, cost, dn):
    """max_iters = k for k = 1..8 against the reference's x after k joint iterations.  Point-to-point in float32 is
    compared at k = 1 only: the reference's own float32 iteration of that cost (Jacobian r dr/dx) drifts by 1e-2 from
    its float64 one within a few steps, so later iterates of two float32 implementations need not agree."""
    dt = DT[dn]
    ref, tgt, nrm = _cast(g, f"ba_multi_{cost}", dt)
    xs, xs64 = g[f"ba_multi_{cost}_{dn}_x"], g[f"ba_multi_{cost}_f64_x"]
    for k in range(1, 2 if (cost, dn) == ("point", "f32") else 9):
        _, x, loss, it = align_batch(ctx, cost, ref, tgt, nrm, "geman_mcclure", dt(0.3), k, 1e-6)
        if dt == np.float32:
            tol = 2e-6 + 2e-4 * np.abs(xs[k - 1]) + 2 * np.abs(xs[k - 1] - xs64[k - 1])
            assert (np.abs(x - xs[k - 1]) <= tol).all(), (cost, dn, k, np.abs(x - xs[k - 1]).max())
        else:
            np.testing.assert_allclose(x, xs[k - 1], rtol=1e-8, atol=1e-12, err_msg=f"{cost} {dn} k={k}")
    if (cost, dn) != ("point", "f32"):
        dT, x, loss, _ = align_batch(ctx, cost, ref, tgt, nrm, "geman_mcclure", dt(0.3), 8, 1e-6)
        key = f"ba_multi_{cost}_{dn}"
        _check_close(dT, x, loss, g, key, dt, (xs64[-1], g[f"ba_multi_{cost}_f64_loss"]),
                     gold=(xs[-1], g[f"{key}_dT"], g[f"{key}_loss"]))


@pytest.mark.parametrize("cost", ["plane", "point"])
def test_batch_goldens_initial_estimates(b200, g, cost):
    """initial_estimate as [B,6] parameters and as [B,4,4] float32 pose matrices, through the mirrors."""
    ref, tgt, nrm = _cast(g, "ba_x0", np.float32)
    gn = dict(scheme="huber", sigma=0.3, max_iters=3, norm_stop_criterion=1e-9)
    if cost == "plane":
        al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=gn))
        run = lambda x0: al.align(ref, tgt, nrm, initial_estimate=x0)  # noqa: E731
    else:
        al = b200.GaussNewtonPointToPointAlignment(b200.GNPointToPointConfig(gauss_newton_config=gn))
        run = lambda x0: al.align(ref, tgt, initial_estimate=x0)  # noqa: E731
    _, x64, _, l64 = bar.gn_align_batch_f64(ref, tgt, nrm if cost == "plane" else None, "huber", 0.3, 3, 1e-9,
                                            x0=g["ba_x0_x0"])
    for form, init in (("vec", g["ba_x0_x0"]), ("mat", g["ba_x0_mats"])):
        dT, x, loss = run(init)
        _check_close(dT, x, loss, g, f"ba_x0_{cost}_{form}", np.float32, (x64, l64))


@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_batch_goldens_zero_residual_element_warning_and_errors(ctx, g, dn, caplog):
    dt = DT[dn]
    ref, tgt, nrm = _cast(g, "ba_zero", dt)
    for sch in ("default", "geman_mcclure"):
        key = f"ba_zero_plane_{sch}_{dn}"
        with caplog.at_level(logging.WARNING):
            caplog.clear()
            if bool(g[f"{key}_raises"]):
                with pytest.raises(RuntimeError, match="Invalid Jacobian in Gauss Newton minimization"):
                    align_batch(ctx, "plane", ref, tgt, nrm, sch, dt(0.3), 2, 1e-9)
            else:
                dT, x, loss, _ = align_batch(ctx, "plane", ref, tgt, nrm, sch, dt(0.3), 2, 1e-9)
                _check_close(dT, x, loss, g, key, dt, _f64(g, f"ba_zero_plane_{sch}_f64"))
            assert "residual norm is lower" not in caplog.text
    assert bool(g[f"ba_zero_point_{dn}_raises"])
    with pytest.raises(RuntimeError, match="Invalid Jacobian in Gauss Newton minimization"):
        align_batch(ctx, "point", ref, tgt, None, "default", 0.5, 2)
    # every residual zero: the reference warns and returns x unchanged with loss r^2 = 0
    t = np.ascontiguousarray(g["ba_allzero_tgt"], dt)
    for cost in ("plane", "point"):
        assert bool(g[f"ba_allzero_{cost}_{dn}_warned"])
        caplog.clear()
        with caplog.at_level(logging.WARNING):
            dT, x, loss, it = align_batch(ctx, cost, t, t, nrm, "huber", dt(0.3), 3)
        assert "residual norm is lower than threshold 1e-7" in caplog.text and it == 1
        assert np.array_equal(x, g[f"ba_allzero_{cost}_{dn}_x"]) and np.array_equal(loss, g[f"ba_allzero_{cost}_{dn}_loss"])
        assert np.array_equal(dT.reshape(-1, 4, 4), g[f"ba_allzero_{cost}_{dn}_dT"])
    # one degenerate element fails the whole call
    ref, tgt, nrm = _cast(g, "ba_degen", dt)
    for cost in ("plane", "point"):
        assert bool(g[f"ba_degen_{cost}_{dn}_raises"])
        with pytest.raises(RuntimeError, match="Invalid Jacobian in Gauss Newton minimization"):
            align_batch(ctx, cost, ref, tgt, nrm if cost == "plane" else None, "default", 0.5, 1)


def test_golden_raise_through_the_mirror(b200, g):
    ref, tgt, nrm = _cast(g, "ba_degen", np.float32)
    al = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig())
    with pytest.raises(RuntimeError, match="Invalid Jacobian in Gauss Newton minimization"):
        al.align(ref, tgt, nrm)


# ------------------------------------------------------------------------------------------ bit for bit, per element
@pytest.mark.parametrize("cost", ["plane", "point"])
@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_each_element_equals_its_own_single_call_at_one_iteration(ctx, g, cost, dn):
    dt = DT[dn]
    ref, tgt, nrm = _cast(g, "ba_sch", dt)
    x0 = np.ascontiguousarray(np.random.RandomState(3).normal(0, 0.01, (5, 6)), dt)
    for sch in SCHEMES:
        for init in (None, x0):
            dT, x, loss, it = align_batch(ctx, cost, ref, tgt, nrm, sch, dt(0.3), 1, x0=init)
            assert it == 1
            for b in range(5):
                sdT, sx, sloss = align_single(ctx, cost, ref[b], tgt[b], nrm[b] if cost == "plane" else None, sch,
                                              dt(0.3), 1, x0=None if init is None else init[b])
                assert np.array_equal(dT[b], sdT) and np.array_equal(x[b], sx) and np.array_equal(loss[b], sloss), (sch, b)


@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_each_element_equals_single_calls_of_the_batch_iteration_count(ctx, g, dn):
    """The batch stops when |dx| over all elements is small; each element's result is then its own alignment run for
    exactly that many iterations (norm_stop = 0).  Element 0's own call, with the batch's norm_stop, stops earlier:
    the batch kept iterating it, as the reference does."""
    dt = DT[dn]
    ref, tgt, nrm = _cast(g, "ba_multi_plane", dt)
    dT, x, loss, K = align_batch(ctx, "plane", ref, tgt, nrm, "geman_mcclure", dt(0.3), 30, 1e-6)
    assert 2 < K <= 30, K
    for b in range(4):
        sdT, sx, sloss = align_single(ctx, "plane", ref[b], tgt[b], nrm[b], "geman_mcclure", dt(0.3), K, 0.0)
        assert np.array_equal(dT[b], sdT) and np.array_equal(x[b], sx) and np.array_equal(loss[b], sloss), b
    _, own_x, _, own_iters = align_batch(ctx, "plane", ref[:1], tgt[:1], nrm[:1], "geman_mcclure", dt(0.3), 30, 1e-6)
    assert own_iters < K, (own_iters, K)
    own_single = align_single(ctx, "plane", ref[0], tgt[0], nrm[0], "geman_mcclure", dt(0.3), 30, 1e-6)[1]
    assert np.array_equal(own_x[0], own_single)
    # point-to-point, float64, a few iterations
    if dt == np.float64:
        ref, tgt, _ = _cast(g, "ba_multi_point", dt)
        dT, x, loss, K = align_batch(ctx, "point", ref, tgt, None, "geman_mcclure", 0.3, 5, 1e-6)
        for b in range(4):
            sdT, sx, sloss = align_single(ctx, "point", ref[b], tgt[b], None, "geman_mcclure", 0.3, K, 0.0)
            assert np.array_equal(dT[b], sdT) and np.array_equal(x[b], sx) and np.array_equal(loss[b], sloss), b


# ------------------------------------------------------------------------------------------ edges vs float64 reference
def _edge_data(B, n, seed):
    rs = np.random.RandomState(seed)
    tgt = rs.uniform(-20, 20, (B, n, 3))
    prm = rs.normal(0, 1, (B, 6)) * [0.05, 0.05, 0.05, 0.004, 0.004, 0.004]
    T = np.stack([nrr.build_pose(p) for p in prm]) if B <= 4096 else None
    if T is None:  # many elements: a few distinct poses, cycled
        Ts = np.stack([nrr.build_pose(p) for p in prm[:64]])
        T = Ts[np.arange(B) % 64]
    ref = np.einsum("bij,bnj->bni", T[:, :3, :3], tgt) + T[:, None, :3, 3] + rs.normal(0, 0.05, (B, n, 3))
    nrm = rs.normal(0, 1, (B, n, 3))
    nrm /= np.linalg.norm(nrm, axis=2, keepdims=True)
    return ref, tgt, nrm


def _sampled(B):
    return sorted({b for b in (0, 1, 2, 30, 31, 32, 33, 255, 256, 257, B // 2, 65534, 65535, 65536, B - 2, B - 1)
                   if 0 <= b < B})


def _check_edges(ctx, B, n, seed):
    ref64, tgt64, nrm64 = _edge_data(B, n, seed)
    for cost in ("plane", "point"):
        for dt in (np.float64, np.float32):
            ref, tgt = np.ascontiguousarray(ref64, dt), np.ascontiguousarray(tgt64, dt)
            nrm = np.ascontiguousarray(nrm64, dt) if cost == "plane" else None
            sig = float(dt(0.3))
            if n <= 2:
                with pytest.raises(RuntimeError, match="Invalid Jacobian"):
                    align_batch(ctx, cost, ref, tgt, nrm, "geman_mcclure", sig)
                continue
            dT, x, loss, it = align_batch(ctx, cost, ref, tgt, nrm, "geman_mcclure", sig)
            assert it == 1 and np.isfinite(x).all() and np.isfinite(loss).all()
            idx = _sampled(B)
            r, t = ref[idx].astype(np.float64), tgt[idx].astype(np.float64)
            m = None if nrm is None else nrm[idx].astype(np.float64)
            st, xr, _, lr = bar.gn_align_batch_f64(r, t, m, "geman_mcclure", sig)
            assert st == "ok"
            for j, b in enumerate(idx):
                args = (r[j], t[j], None if m is None else m[j])
                lb = nrr.gn_loss_bound(*args, np.zeros(6), "geman_mcclure", sig, U64 if dt == np.float64 else nrr.U)
                assert (np.abs(loss[b] - lr[j]) <= lb).all(), (cost, dt, B, n, b)
                if dt == np.float64:
                    assert np.abs(x[b] - xr[j]).max() <= 1e-10 * np.abs(xr[j]).max(), (cost, B, n, b)
                else:
                    assert (np.abs(x[b] - xr[j]) <= nrr.gn_f32_step_bound(*args, "geman_mcclure", sig)).all(), (cost, B, n, b)
                Tx = nrr.build_pose(x[b].astype(np.float64))
                assert (np.abs(dT[b].reshape(4, 4) - Tx) <= 16 * np.finfo(dt).eps * (1 + np.abs(Tx))).all(), (cost, B, n, b)


@pytest.mark.parametrize("B", [1, 2, 31, 32, 33, 257, 65535, 65536, 65537])
def test_batch_edges_at_n64(ctx, B):
    _check_edges(ctx, B, 64, B)


@pytest.mark.parametrize("n,B", [(1, 2), (2, 3), (255, 2), (256, 3), (257, 2), (67583, 3), (67584, 2), (67585, 3)])
def test_point_count_edges(ctx, n, B):
    _check_edges(ctx, B, n, n)


def test_deterministic_on_one_context_and_across_contexts(ctx):
    from pylidar_slam_b200 import _lib
    ref, tgt, nrm = (np.ascontiguousarray(a, np.float32) for a in _edge_data(257, 3000, 5))
    first = align_batch(ctx, "plane", ref, tgt, nrm, "cauchy", 0.3, 4, 1e-9)
    again = align_batch(ctx, "plane", ref, tgt, nrm, "cauchy", 0.3, 4, 1e-9)
    other = _lib.Context()
    try:
        third = align_batch(other, "plane", ref, tgt, nrm, "cauchy", 0.3, 4, 1e-9)
    finally:
        other.close()
    for a, b, c in zip(first[:3], again[:3], third[:3]):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    assert first[3] == again[3] == third[3]


# ------------------------------------------------------------------------------------------ input forms of the mirrors
def test_mirror_input_forms(b200, g):
    ref, tgt, nrm = _cast(g, "ba_sch", np.float32)
    plane = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=3, norm_stop_criterion=1e-9)))
    point = b200.GaussNewtonPointToPointAlignment(b200.GNPointToPointConfig(
        gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=3, norm_stop_criterion=1e-9)))
    base = plane.align(ref, tgt, nrm)
    base_pt = point.align(ref, tgt)
    for conv in (torch.from_numpy, lambda a: torch.from_numpy(a).cuda()):
        out = plane.align(conv(ref), conv(tgt), conv(nrm))
        out_pt = point.align(conv(ref), conv(tgt))
        for a, b in zip(out + out_pt, base + base_pt):
            assert isinstance(a, torch.Tensor) and a.device == conv(ref).device
            assert np.array_equal(a.cpu().numpy(), b)
    # float64 stays float64 on every form
    for conv in (lambda a: a, torch.from_numpy, lambda a: torch.from_numpy(a).cuda()):
        dT, x, loss = plane.align(conv(ref.astype(np.float64)), conv(tgt.astype(np.float64)), conv(nrm.astype(np.float64)))
        assert x.dtype in (np.float64, torch.float64) and tuple(x.shape) == (5, 6) and tuple(loss.shape) == (5, 400)
    # shapes: a mismatch is the reference's AssertionError; a mask is its RuntimeError after the [B,N,1] check
    with pytest.raises(AssertionError):
        plane.align(ref[:4], tgt, nrm)
    with pytest.raises(AssertionError):
        point.align(ref, tgt[:, :399])
    with pytest.raises(AssertionError):
        plane.align(ref, tgt, nrm, initial_estimate=np.zeros((4, 6), np.float32))
    with pytest.raises(RuntimeError):
        plane.align(ref, tgt, nrm, mask=np.ones((5, 400, 1), np.float32))
    with pytest.raises(AssertionError):
        point.align(ref, tgt, mask=np.ones((1, 400, 1), np.float32))


def test_cuda_input_written_on_a_side_stream(b200, g):
    """Tensors produced on a non-default torch stream: the call is ordered after that stream's work."""
    ref, tgt, nrm = _cast(g, "ba_sch", np.float32)
    plane = b200.GaussNewtonPointToPlaneAlignment(b200.GaussNewtonPointToPlaneConfig(
        gauss_newton_config=dict(scheme="huber", sigma=0.3, max_iters=2)))
    base = plane.align(ref, tgt, nrm)
    side = torch.cuda.Stream()
    big = torch.randn(4096, 4096, device="cuda")
    with torch.cuda.stream(side):
        for _ in range(4):
            big = big @ big * 1e-3          # keeps the side stream busy while the inputs are written behind it
        r, t, n = (torch.from_numpy(a).cuda(non_blocking=False) * 1.0 for a in (ref, tgt, nrm))
        out = plane.align(r, t, n)
    side.synchronize()
    for a, b in zip(out, base):
        assert np.array_equal(a.cpu().numpy(), b)
