"""Gated registration without a GPU: the float64 oracle of one gated ICP iteration
(oracle/gated_registration_reference) against hand-computed cases and an independent per-row restatement, the float32
search bound G at its edges, the changed-map scenario the GPU test takes its tolerance from, and the Python routing of
max_distance over a stand-in backend."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import evaluate_poses_reference as er  # noqa: E402
from oracle import gated_registration_reference as gr  # noqa: E402

# the changed-map scenario: what the float64 ICP gives (test_changed_map_scenario) and the GPU test asserts
CHANGED_MAP_GATE = 1.0
CHANGED_MAP_TOL = (0.02, 0.002)      # metres, radians: the gated registration ends within this of the truth
CHANGED_MAP_UNGATED_MIN = 0.5        # metres: the ungated one ends at least this far off


def _d2_f32_variants(p, q):
    """float32 d^2 of dist2_point under every FMA contraction the compiler may choose (the plain sum, and fused
    forms), computed with exact float64 products rounded once where fused."""
    d = (p - q).astype(np.float32)
    sq = (d * d).astype(np.float32)
    plain = ((sq[:, 0] + sq[:, 1]).astype(np.float32) + sq[:, 2]).astype(np.float32)
    d64 = d.astype(np.float64)
    f1 = np.float32(d64[:, 0] * d64[:, 0] + np.float64(sq[:, 1]))                    # fma(dx, dx, dy*dy)
    f2 = np.float32(d64[:, 2] * d64[:, 2] + np.float64(f1))                           # fma(dz, dz, that)
    g1 = np.float32(d64[:, 1] * d64[:, 1] + np.float64(sq[:, 0]))
    g2 = np.float32(d64[:, 2] * d64[:, 2] + np.float64(g1))
    return [plain, f2, g2]


@pytest.mark.parametrize("scale", [1e-30, 1e-6, 1e-2, 0.3, 1.0, 7.0, 1e3, 1e15])
def test_gate_bound_covers_every_inlier(scale):
    rng = np.random.RandomState(int(abs(np.log2(scale))) + 1)
    q = rng.uniform(-50, 50, (20000, 3)).astype(np.float32)
    u = rng.normal(size=(20000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = (q + scale * u).astype(np.float32)
    d2 = er.match_d2(p, q)
    for md in (np.sqrt(d2), np.nextafter(np.sqrt(d2), np.inf)):
        # max_distance at (or an ulp above) each row's own distance: every row is an inlier at the edge of the gate
        assert np.all(d2 <= md * md) or np.all(np.sqrt(d2) <= md)
        G = np.array([gr.gate_bound(m) for m in md[:2000]], np.float32)
        for v in _d2_f32_variants(p[:2000], q[:2000]):
            assert np.all(v < G)
        # and G is tight: within 2^-19 relative (plus the FLT_MIN floor) of max_distance^2
        assert np.all(G.astype(np.float64) <= (md[:2000] ** 2) * (1 + 2.0 ** -19) + 2.0 ** -125)


def test_gate_bound_edges():
    assert gr.gate_bound(0.0) == np.float32(2.0 ** -126)
    # 1 + 2^-20 is a float32; the 2^-126 floor is below its ulp and leaves it as it is
    assert gr.gate_bound(1.0) == np.float32(1.0 + 2.0 ** -20)
    assert gr.gate_bound(2.0 ** 64) == np.float32(np.inf)   # beyond FLT_MAX: the search is never cut short
    assert gr.dmax32(0.1) >= 0.1 and np.float64(np.nextafter(gr.dmax32(0.1), np.float32(0))) < 0.1
    assert gr.dmax32(1e40) == np.float32(np.inf)


def test_gated_iteration_by_hand():
    """Three rows on the plane z = 0 with normal +z: two within 0.5 m, one at 0.6 m.  scheme 'default' (w = 1)."""
    q = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    p = np.array([[0, 0, 0.25], [1, 0, -0.5], [0, 1, 0.6]], np.float32)
    n = np.tile(np.float32([0, 0, 1]), (3, 1))
    it = gr.gated_iteration(p, q, n, np.ones(3, bool), 0.5, "default", 1.0)
    assert it["count"] == 2 and list(it["inliers"]) == [True, True, False]
    assert it["sums"][29] == 2.0
    assert it["sums"][28] == pytest.approx(0.25 ** 2 + 0.5 ** 2, rel=1e-12)   # sum r^2 over the inliers
    assert it["sums"][0] == 0.0 and it["sums"][6] == 0.0 and it["sums"][11] == 2.0   # J = [0, 0, 1, ...]: n = z
    assert it["step"] is None   # a plane constrains three of six directions: singular
    # the d^2 of the gate is float64, every operation rounded once: exactly 0.5^2 is in, one ulp more is out
    it2 = gr.gated_iteration(p, q, n, np.ones(3, bool), np.nextafter(0.5, 0), "default", 1.0)
    assert list(it2["inliers"]) == [True, False, False]


@pytest.mark.parametrize("max_distance", [0.0, 0.05, 0.2, 1.0, np.inf])
@pytest.mark.parametrize("scheme", ["default", "huber", "cauchy"])
def test_gated_iteration_against_a_per_row_restatement(max_distance, scheme):
    """The gate row by row in Python floats (IEEE doubles, one rounding per operation), the sums as kd_icp_reference's
    accumulate over the rows kept, the step by an explicit 6x6 solve."""
    from oracle import kd_icp_reference as kref
    rng = np.random.RandomState(7)
    q = rng.uniform(-5, 5, (3000, 3)).astype(np.float32)
    p = (q + rng.normal(0, 0.2, q.shape)).astype(np.float32)
    q[:40] = p[:40]                                           # d = 0 exactly
    n = rng.normal(size=q.shape)
    n = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
    matched = rng.uniform(size=3000) > 0.05
    md2 = float(max_distance) * float(max_distance)
    keep = np.zeros(3000, bool)
    for i in range(3000):
        dx, dy, dz = (float(p[i, a]) - float(q[i, a]) for a in range(3))
        keep[i] = bool(matched[i]) and (dx * dx + dy * dy) + dz * dz <= md2
    it = gr.gated_iteration(p, q, n, matched, max_distance, scheme, 0.3)
    assert np.array_equal(it["inliers"], keep) and it["count"] == keep.sum() == it["sums"][29]
    want = kref.accumulate(p[keep].astype(np.float64), q[keep].astype(np.float64), n[keep].astype(np.float64),
                           scheme, 0.3) if keep.any() else np.zeros(30)
    np.testing.assert_allclose(it["sums"], want, rtol=1e-12, atol=1e-12)
    H = np.zeros((6, 6))
    iu = np.triu_indices(6)
    H[iu] = want[:21]
    H = H + np.triu(H, 1).T
    if keep.sum() >= 6 and abs(np.linalg.det(H)) >= 1e-7:
        np.testing.assert_allclose(it["step"], -np.linalg.solve(H, want[21:27]), rtol=1e-9, atol=1e-12)
    else:
        assert it["step"] is None


def test_brute_force_gated_nn():
    m = np.array([[0, 0, 0], [1, 0, 0], [0.5, 0, 0], [10, 0, 0]], np.float32)
    positions = np.array([3, 1, 0, 2])
    p = np.array([[0.25, 0, 0], [0.75, 0, 0], [5.0, 0, 0], [9.5, 0, 0], [0.1, 0, 0]], np.float32)
    match, decided = gr.brute_force_gated_nn(m, positions, p, 1.0)
    # [0.25]: equidistant from 0 and 0.5 -> the smaller sorted position (point 2); [5.0] beyond the gate -> -1
    assert list(match) == [2, 2, -1, 3, 0]
    assert not decided[0] and not decided[1] and decided[2] and decided[3] and decided[4]
    match, decided = gr.brute_force_gated_nn(m, positions, p, 0.4)
    assert match[4] == 0 and match[2] == -1 and match[3] == -1


def test_changed_map_scenario():
    """The float64 ICP on the changed map: the gate recovers the truth, the ungated registration is pulled off by the
    object the map lacks.  The GPU test holds the kernels to these numbers."""
    prior, scan, truth, start = gr.changed_map_scene(0)
    Tg, inl = gr.icp(prior, scan, start, CHANGED_MAP_GATE)
    Tu, _ = gr.icp(prior, scan, start, np.inf)
    et, er_ = gr.pose_error(Tg, truth)
    assert et <= CHANGED_MAP_TOL[0] / 10 and er_ <= CHANGED_MAP_TOL[1] / 10
    assert gr.pose_error(Tu, truth)[0] >= 2 * CHANGED_MAP_UNGATED_MIN
    assert inl == 18000   # the room's rows; none of the object's


# ------------------------------------------------------------------------------------------------ Python routing
@pytest.fixture
def stand_in(monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dryrun_next_rows as dry
    from pylidar_slam_b200 import _lib, common
    calls = []

    class GatedFakeContext(dry.FakeContext):
        M = 4

        def call(self, name, *a):
            calls.append((name, a))
            return getattr(self, name)(*a)

        def _answer(self, S, scan_of, B, out_T, out_iters, out_status):
            dry.arr(out_T, (B, 4, 4), np.float32)[:] = np.eye(4, dtype=np.float32)
            dry.arr(out_iters, (B,), np.int32)[:] = 1
            dry.arr(out_status, (B,), np.int32)[:] = _lib.PLS_OK

        def pls_register_scans(self, scans, n, S, scan_of, T0s, B, out_T, out_params, out_losses, out_iters,
                               out_status):
            self._answer(S, scan_of, B, out_T, out_iters, out_status)

        def pls_register_scans_gated(self, scans, n, S, scan_of, T0s, B, max_distance, out_T, out_params, out_losses,
                                     out_iters, out_status, out_inliers):
            self._answer(S, scan_of, B, out_T, out_iters, out_status)
            dry.arr(out_inliers, (B,), np.int32)[:] = np.arange(B) + 100

        def pls_register_hypotheses(self, points, n, T0s, B, out_T, out_params, out_losses, out_iters, out_status):
            self._answer(1, None, B, out_T, out_iters, out_status)

    monkeypatch.setattr(_lib, "Context", GatedFakeContext)
    monkeypatch.setattr(common, "_default_ctx", GatedFakeContext())
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = GatedFakeContext()
    odo.ctx.cfg.local_map_type = _lib.MAP_KDTREE
    odo.config = ICPFrameToModelConfig(max_num_alignments=GatedFakeContext.M)
    return odo, calls, _lib


def _inputs(B=3):
    rng = np.random.RandomState(0)
    return [rng.randn(50, 3).astype(np.float32), rng.randn(40, 3).astype(np.float32)], \
        np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))


def test_inf_calls_the_ungated_entry_points(stand_in):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    odo.register_new_frames(scans, T0, [0, 1, 0])
    odo.register_new_frames(scans, T0, [0, 1, 0], max_distance=np.inf)
    odo.register_new_frame_hypotheses(scans[0], T0)
    assert [c[0] for c in calls] == ["pls_register_scans", "pls_register_scans", "pls_register_hypotheses"]
    assert odo.last_registrations_inliers is None and odo.last_hypotheses_inliers is None


def test_finite_gate_calls_the_gated_entry_point(stand_in):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    odo.register_new_frames(scans, T0, [0, 1, 0], max_distance=0.75)
    name, a = calls[-1]
    assert name == "pls_register_scans_gated" and a[2] == 2 and a[5] == 3 and a[6] == 0.75
    assert list(odo.last_registrations_inliers) == [100, 101, 102]
    calls.clear()
    odo.register_new_frame_hypotheses(scans[1], T0, max_distance=0.0)
    name, a = calls[-1]
    assert name == "pls_register_scans_gated" and a[2] == 1 and a[6] == 0.0
    import dryrun_next_rows as dry
    assert list(dry.arr(a[3], (3,), np.int32)) == [0, 0, 0]
    assert list(odo.last_hypotheses_inliers) == [100, 101, 102]
    assert list(odo.last_registrations_inliers) == [100, 101, 102] and odo.last_registrations_status is not \
        odo.last_hypotheses_status   # the hypotheses leave the registrations' attributes alone


@pytest.mark.parametrize("bad", [-1.0, float("nan"), -np.inf])
def test_refusals_raise_before_any_call(stand_in, bad):
    odo, calls, _ = stand_in
    scans, T0 = _inputs()
    with pytest.raises(Exception):
        odo.register_new_frames(scans, T0, [0, 1, 0], max_distance=bad)
    with pytest.raises(Exception):
        odo.register_new_frame_hypotheses(scans[0], T0, max_distance=bad)
    assert calls == []


def test_finite_gate_on_a_projective_map_raises_before_any_call(stand_in):
    odo, calls, lib = stand_in
    odo.ctx.cfg.local_map_type = lib.MAP_PROJECTIVE
    scans, T0 = _inputs()
    with pytest.raises(Exception):
        odo.register_new_frame_hypotheses(scans[0], T0, max_distance=1.0)
    odo.register_new_frame_hypotheses(scans[0], T0)
    assert [c[0] for c in calls] == ["pls_register_hypotheses"]


def test_localize_passes_the_gate_to_its_refinement_only(stand_in, monkeypatch):
    from pylidar_slam_b200 import odometry as od
    odo, calls, _ = stand_in
    seen = []
    T0 = np.tile(np.eye(4), (2, 1, 1))
    monkeypatch.setattr(od, "_pose_search", lambda *a, **k: (seen.append("search"), (T0, np.zeros(2), None))[1])
    monkeypatch.setattr(od, "_score_poses", lambda *a, **k: (seen.append("score"), np.zeros(2, np.int32))[1])
    monkeypatch.setattr(od, "_pose_candidates", lambda *a: list(a))
    scan = _inputs()[0][0]
    odo.localize(scan, np.eye(4), 2.0, 0.5)
    odo.localize(scan, np.eye(4), 2.0, 0.5, max_distance=0.8)
    assert seen == ["search", "score", "search", "score"]
    assert [c[0] for c in calls] == ["pls_register_hypotheses", "pls_register_scans_gated"]
    assert calls[1][1][6] == 0.8
