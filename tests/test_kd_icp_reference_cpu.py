"""The float64 reference of one kd ICP iteration (oracle/kd_icp_reference.py), pinned on the CPU: its accumulators
give the oracle's Gauss-Newton step, its matches and normals are exact, its float32 tolerance covers float32 inputs."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import icp_oracle as orc
from oracle import kd_icp_reference as ref

SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


def _correspondences(seed, n=2000):
    rng = np.random.RandomState(seed)
    q = rng.uniform(-30, 30, (n, 3))
    nrm = rng.randn(n, 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    p = q + nrm * rng.normal(0, 0.2, (n, 1)) + rng.normal(0, 0.05, (n, 3))
    return p, q, nrm


@pytest.mark.parametrize("scheme", SCHEMES)
def test_step_from_the_sums_is_the_oracle_gauss_newton_step(scheme):
    p, q, nrm = _correspondences(SCHEMES.index(scheme))
    sigma = 0.3
    sums = ref.accumulate(p, q, nrm, scheme, sigma)
    assert sums[29] == len(p)
    x = ref.gauss_newton_step(sums)
    t = [torch.from_numpy(a)[None] for a in (q, p, nrm)]
    x_orc, loss, status = orc.gauss_newton_p2plane(*t, scheme=scheme, sigma=sigma, max_iters=1)
    assert status == "ok"
    np.testing.assert_allclose(x, x_orc[0].numpy(), rtol=0, atol=1e-10)
    np.testing.assert_allclose(sums[27], loss.sum().item(), rtol=1e-12)


def test_matches_runner_up_and_normals_are_exact():
    rng = np.random.RandomState(3)
    m = (rng.randn(3000, 3) * np.array([10, 10, 1])).astype(np.float32)
    q = (rng.randn(500, 3) * np.array([10, 10, 1])).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    T[:3, 3] = [0.3, -0.2, 0.1]
    out = ref.kd_icp_iteration(m, q, T, "geman_mcclure", 0.3, k=10)
    p = q.astype(np.float64) + T[:3, 3].astype(np.float64)
    np.testing.assert_array_equal(out["p"], p)
    d = np.linalg.norm(p[:, None, :] - m[None].astype(np.float64), axis=2)
    order = np.argsort(d, axis=1)
    np.testing.assert_array_equal(out["match"], order[:, 0])
    np.testing.assert_allclose(out["d2"], d[np.arange(len(p)), order[:, 1]], rtol=1e-15)
    # normal of one matched point by brute force: smallest eigenvector of its 10 nearest other points' moments
    i = out["match"][0]
    nb = np.argsort(np.linalg.norm(m - m[i], axis=1))[1:11]
    diff = (m[nb] - m[i]).astype(np.float64)
    v = np.linalg.eigh(diff.T @ diff / 10)[1][:, 0]
    assert abs(abs(v @ out["normals"][0]) - 1) < 1e-12
    np.testing.assert_allclose(out["sums"], ref.accumulate(p, m[out["match"]].astype(np.float64), out["normals"],
                                                           "geman_mcclure", 0.3), rtol=1e-14)


@pytest.mark.parametrize("scheme", SCHEMES)
def test_float32_tolerance_covers_a_float32_evaluation(scheme):
    """The same correspondences evaluated in float32 (residual, Jacobian, weight, products; fp64 sums, as the kernels
    do) stay within the tolerance -- and the tolerance is not so loose that a dropped robust weight would pass."""
    p, q, nrm = (a.astype(np.float32) for a in _correspondences(10 + SCHEMES.index(scheme)))
    sigma = 0.3
    p64, q64, n64 = (a.astype(np.float64) for a in (p, q, nrm))
    exact = ref.accumulate(p64, q64, n64, scheme, sigma)
    e = 8 * 2.0 ** -23 * (np.linalg.norm(p64, axis=1) + np.linalg.norm(q64, axis=1))
    tol = ref.float32_tolerance(p64, q64, n64, scheme, sigma, e)
    t32 = [torch.from_numpy(a)[None] for a in (p, q, nrm)]
    x = torch.zeros(1, 6, dtype=torch.float32)
    r = orc.p2plane_residual(x, t32[0], t32[1], t32[2])
    J = orc.p2plane_jacobian(x, t32[0], t32[2])
    w = orc.ls_weights(scheme, sigma, r, t32[0], t32[1]).expand_as(r)
    wj = (J * w.unsqueeze(-1))[0].double().numpy()
    wr = (w * r)[0].double().numpy()
    f32 = np.concatenate([np.stack([wj[:, a] * wj[:, b] for a in range(6) for b in range(a, 6)], 1),
                          wj * wr[:, None], (wr * wr)[:, None], (r[0].double().numpy() ** 2)[:, None],
                          np.ones((len(p), 1))], 1).sum(0)
    assert (np.abs(f32 - exact) <= tol).all(), np.abs(f32 - exact) / tol
    if scheme != "default":
        unweighted = ref.accumulate(p64, q64, n64, "default", sigma)
        assert (np.abs(unweighted - exact) > tol).any()
