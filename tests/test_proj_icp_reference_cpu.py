"""Pins oracle/proj_icp_reference.py (the float64 projective ICP iteration the GPU tests compare against) to the oracle's
own ProjectiveLocalMap: its nearest_neighbor_search plus the point-to-plane accumulators, and its model rebuild."""
import numpy as np
import pytest
import torch

from oracle import icp_oracle as orc
from oracle import kd_icp_reference as kdr
from oracle import proj_icp_reference as pref
from pylidar_slam_b200 import synthetic as syn

H, W = 16, 256
U = pref.U


@pytest.fixture(scope="module")
def local_map():
    lm = orc.ProjectiveLocalMap(orc.Projector(H, W), local_map_size=3)
    vmaps, rels = [], []
    for k in range(4):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        vm = syn.vertex_map_from_scan(syn.scan(k, H, W), H, W)
        lm.update(torch.from_numpy(rel)[None], new_vertex_map=torch.from_numpy(vm))
        vmaps.append(vm[0])
        rels.append(rel)
    return lm, vmaps, rels


def _oracle_sums(lm, p32, scheme, sigma):
    q, n, p = lm.nearest_neighbor_search(torch.from_numpy(p32))
    return kdr.accumulate(p[0].numpy().astype(np.float64), q[0].numpy().astype(np.float64), n[0].numpy().astype(np.float64),
                          scheme, sigma)


@pytest.mark.parametrize("perturb", [False, True])
@pytest.mark.parametrize("scheme", ["geman_mcclure", "neighborhood"])
def test_iteration_matches_the_oracle_search(local_map, perturb, scheme):
    lm = local_map[0]
    mv, mn = lm.model_vmap.numpy(), lm.model_nmap.numpy()
    q = syn.scan(4, H, W)
    T = np.eye(4, dtype=np.float32)
    if perturb:
        T = syn.gt_relative_pose(4).astype(np.float32)
    out = pref.proj_icp_iteration(mv, mn, q, T, scheme, 0.3)
    p32 = np.ascontiguousarray(kdr.transform(T, q).astype(np.float32))
    exp = _oracle_sums(lm, p32, scheme, 0.3)
    err = np.abs(out["sums"] - exp)
    assert (err <= out["tol"]).all(), (np.nonzero(err > out["tol"])[0], (err / out["tol"]).max())
    assert abs(out["sums"][29] - exp[29]) <= out["count_tol"]
    assert out["sums"][29] > 0.5 * H * W
    if not perturb:
        # at the identity the transform is exact, the scan sits on pixel centres: nothing is ambiguous
        assert out["count_tol"] == 0 and out["sums"][29] == exp[29]


def test_wrong_candidate_is_outside_the_tolerance(local_map):
    """The tolerance is tight enough to see one pixel that took its second-nearest candidate."""
    lm = local_map[0]
    mv, mn = lm.model_vmap.numpy(), lm.model_nmap.numpy()
    q = syn.scan(4, H, W)
    out = pref.proj_icp_iteration(mv, mn, q, np.eye(4, dtype=np.float32), "geman_mcclure", 0.3)
    pix = np.nonzero((out["k"] >= 0) & ~out["amb_pixel"] & ~out["amb_query"])[0]
    K = mv.shape[0]
    v = mv.reshape(K, 3, -1)[:, :, pix]
    live = (np.abs(v).max(1) > 0).sum(0)
    pix = pix[live >= 2][:1]
    assert pix.shape[0] == 1
    i = pix[0]
    p = out["p"][out["win"][i]][None]
    k_ok = out["k"][i]
    k_bad = next(k for k in range(K) if k != k_ok and np.abs(mv.reshape(K, 3, -1)[k, :, i]).max() > 0)
    t = [kdr.terms(p, mv.reshape(K, 3, -1)[k, :, i][None].astype(np.float64), mn.reshape(K, 3, -1)[k, :, i][None].astype(np.float64),
                   "geman_mcclure", 0.3)[0] for k in (k_ok, k_bad)]
    assert (np.abs(t[0] - t[1]) > out["tol"]).any()


def test_first_minimum_and_null_candidates():
    """Hand-made model: an exact distance tie goes to the first candidate, a null candidate never competes, a pixel of
    null candidates matches nothing."""
    mv = np.zeros((3, 3, H, W), np.float32)
    mn = np.zeros_like(mv)
    row, col = 8, 100
    theta = (2.0 * col / W - 1.0) * np.pi
    up, down = 3.0 / 180 * np.pi, 24.0 / 180 * np.pi
    phi = (1.0 - row / H) * (up + down) - down
    d = np.array([np.cos(phi) * np.cos(-theta), np.cos(phi) * np.sin(-theta), np.sin(phi)])
    p = np.round(10 * d * 2 ** 14) / 2 ** 14
    q = p.astype(np.float32)[None]
    mv[0, :, row, col] = p + np.array([3, 4, 0]) * 2 ** -10
    mv[2, :, row, col] = p + np.array([0, 4, 3]) * 2 ** -10
    mn[0, :, row, col] = [1, 0, 0]
    mn[2, :, row, col] = [0, 0, 1]
    out = pref.proj_icp_iteration(mv, mn, q, np.eye(4, dtype=np.float32), "default", 0.5)
    i = row * W + col
    assert out["win"][i] == 0 and out["k"][i] == 0 and not out["amb_pixel"][i]
    assert out["sums"][29] == 1 and out["sums"][28] == pytest.approx((3 * 2 ** -10) ** 2)
    mv[0, :, row, col] = 0
    out = pref.proj_icp_iteration(mv, mn, q, np.eye(4, dtype=np.float32), "default", 0.5)
    assert out["k"][i] == 2
    mv[2, :, row, col] = 0
    out = pref.proj_icp_iteration(mv, mn, q, np.eye(4, dtype=np.float32), "default", 0.5)
    assert out["k"][i] == -1 and out["sums"][29] == 0


def test_model_rebuild_matches_the_oracle(local_map):
    lm, vmaps, rels = local_map
    # the oracle holds the last 3 frames; poses frame -> newest in float64
    P = [np.eye(4)]
    for rel in reversed(rels[2:]):
        P.insert(0, P[0] @ np.linalg.inv(rel.astype(np.float64)))
    nm = orc.normal_map(torch.from_numpy(np.stack(vmaps[1:])), 5).numpy()
    V, N, occ, amb, err = pref.rebuild_model(np.stack(vmaps[1:]), nm, np.stack(P), [64 * U * (3 - k) for k in range(3)], H, W)
    mv, mn = lm.model_vmap.numpy(), lm.model_nmap.numpy()
    got = np.abs(mv).max(1) > 0
    sure = ~amb
    assert sure.mean() > 0.95
    assert np.array_equal(got[sure], occ[sure])
    both = sure & occ
    d = np.abs(mv.astype(np.float64) - V).max(1)
    assert (d[both] <= err[both] + 1e-6).all(), d[both].max()
    dn = np.abs(mn.astype(np.float64) - N).max(1)
    assert (dn[both] <= 1e-5).all(), dn[both].max()

