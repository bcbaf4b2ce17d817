"""Registration on a prior map with the eigenvalue-thresholded solve: pls_register_scans_degeneracy and the
min_eigenvalue of ICPFrameToModel.register_new_frames.

  * every iteration's 30 sums are, bit for bit, pls_kdmap_evaluate_poses's row at that iteration's pose and gate, and
    its step, pose update, degenerate count and eigenvalues are the float64 oracle's (oracle/degeneracy_reference.py)
    from those sums; on the one-kernel refine path (k = 10) and on the four launches (k = 64, and a map of 2 M points),
    gated and at +inf;
  * with a threshold below every eigenvalue, nothing is degenerate and the poses are those of pls_register_scans_gated
    to within the rounding of the two solves;
  * on a flat field the plain call is singular, the thresholded one reports three degenerate directions, recovers z,
    roll and pitch and holds x, y and yaw; in a tunnel one direction is degenerate, the position along the axis is
    held and the other five are recovered;
  * batches that mix degenerate and well-constrained registrations across the PLS_MAX_SEQUENCES chunk edges equal
    single calls on both later-iteration paths, with host and device pointers and NULL optional outputs;
  * every refusal leaves the outputs and the context unchanged;
  * the Python methods make the C call.
The maps, scans and start poses are those of tests/test_gated_registration_gpu.py.
"""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_gated_registration_gpu as gg  # noqa: E402
from test_gated_registration_gpu import lib, maps  # noqa: E402,F401  (module fixtures)
from oracle import degeneracy_reference as dr  # noqa: E402

EPS = 2.0 ** -52
EIG_C = 16   # the eigen-solver's error bound in eps ||H||_F (tests/test_degeneracy_cpu.py)
KEYS = ("T", "params", "losses", "iters", "status", "inliers", "degenerate", "eigenvalues")


def _register(lib, ctx, scans, T0, scan_of=None, max_distance=np.inf, min_eigenvalue=1e-3, M=5, dev=False,
              nulls=()):
    """pls_register_scans_degeneracy.  Returns (status, dict of outputs); the outputs named in `nulls` are NULL."""
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([s.shape[0] for s in scans], np.int64)
    B = T0.shape[0]
    o = dict(T=np.zeros((B, 4, 4), np.float32), params=np.zeros((B, 6), np.float32),
             losses=np.zeros((B, M), np.float32), iters=np.zeros(B, np.int32), status=np.zeros(B, np.int32),
             inliers=np.full(B, -7, np.int32), degenerate=np.full(B, -7, np.int32),
             eigenvalues=np.full((B, 6), -7.0))
    of = None if scan_of is None else lib.ptr(np.asarray(scan_of, np.int32))
    f = lib.load().pls_register_scans_degeneracy
    if dev:
        import torch
        keep = [torch.from_numpy(s).cuda() for s in scans]
        addr = np.array([t.data_ptr() for t in keep], np.uint64)
        Td = torch.from_numpy(np.ascontiguousarray(T0)).cuda()
        outs = {k: torch.from_numpy(v).cuda() for k, v in o.items()}
        st = f(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans), of, Td.data_ptr(), B, float(max_distance),
               float(min_eigenvalue), *[None if k in nulls else outs[k].data_ptr() for k in o])
        return st, {k: v.cpu().numpy() for k, v in outs.items()}
    st = f(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans), of, lib.ptr(T0), B, float(max_distance),
           float(min_eigenvalue), *[None if k in nulls else lib.ptr(v) for k, v in o.items()])
    return st, o


def _evaluate(lib, ctx, scan, T, max_distance):
    rows = np.zeros((1, 32))
    addr = np.array([lib.ptr(scan)], np.uint64)
    n = np.array([len(scan)], np.int64)
    assert lib.load().pls_kdmap_evaluate_poses(ctx.handle, lib.ptr(addr), lib.ptr(n), 1, None,
                                               lib.ptr(np.ascontiguousarray(T[None], np.float32)), 1,
                                               float(max_distance), lib.ptr(rows)) == lib.PLS_OK
    return rows[0, :30]


def _check_step(T_lin, got, sums, thr):
    """The pose update is the oracle's projected step from the GPU's sums, cast to float32, applied through the Euler
    round trip (the bound of test_gated_registration_gpu._check_pose_update); the degenerate count is the oracle's
    unless an eigenvalue lies within the eigen-solver's bound of the threshold, and the eigenvalues are within it."""
    import torch
    from oracle import icp_oracle as orc
    step, kept, lam = dr.projected_step(sums, thr)
    N = sums[29]
    bound = EIG_C * EPS * np.linalg.norm(dr.hessian(sums)) / N
    assert np.all(np.abs(got["eigenvalues"][0] - lam) <= bound), (got["eigenvalues"][0], lam)
    tie = np.any(np.abs(lam - thr) <= 2 * bound)
    if not tie:
        assert got["degenerate"][0] == 6 - kept.sum()
    if got["status"][0] != 0 or tie:
        return tie
    dx = step.astype(np.float32).astype(np.float64)
    if got["T"][0].tobytes() == np.asarray(T_lin, np.float32).tobytes():   # the stop test: the step is not applied
        assert np.linalg.norm(step.astype(np.float32)) < 1e-4 * (1 + 1e-6)
        return tie
    dT = orc.build_pose_matrix(torch.from_numpy(dx)[None])[0].numpy()
    prm = orc.from_pose_matrix(torch.from_numpy(dT @ np.asarray(T_lin, np.float64))[None])
    T_exp = orc.build_pose_matrix(prm)[0].numpy()
    T = got["T"][0].astype(np.float64)
    scale = 1 + np.abs(T_exp[:3, 3]).sum()
    assert np.abs(T[:3, :3] - T_exp[:3, :3]).max() <= 2e-6
    assert np.abs(T[:3, 3] - T_exp[:3, 3]).max() <= 2e-6 * scale
    return tie


def _middle_threshold(lib, ctx, scan, T, max_distance):
    """A threshold in the widest gap of the start's spectrum of H / N that keeps at least one direction: some
    directions are degenerate and the kept set is decided."""
    sums = _evaluate(lib, ctx, scan, T, max_distance)
    lam = np.maximum(dr.projected_step(sums, 1.0)[2], 1e-12)
    i = int(np.argmax(np.log(lam[1:]) - np.log(lam[:-1])))
    return float(np.sqrt(lam[i] * lam[i + 1]))


# ------------------------------------------------------------------------------------------------ every iteration
@pytest.mark.parametrize("max_distance", [0.3, np.inf])
@pytest.mark.parametrize("which,k", [("warm", 10), ("warm", 64), ("cold", 10)])
def test_every_iteration_against_evaluate_poses_and_the_oracle(lib, maps, which, k, max_distance):
    """Iteration j, read back after max_num_alignments = j at the pose it ran at (the result of j - 1 alignments)."""
    scan = gg._scans(maps["warm"], [1500], 21, noise=0.05)[0]
    start = gg._poses(2, 21, spread=0.5)[1]
    ev = gg._odometry("default", k, max_iters=1)
    gg._set_map(ev, maps[which])
    thr = _middle_threshold(lib, ev.ctx, scan, start, max_distance)
    T_lin, ran, degenerate = start, 0, 0
    for j in range(1, 7):
        odo = gg._odometry("default", k, max_iters=j)
        gg._set_map(odo, maps[which])
        st, got = _register(lib, odo.ctx, [scan], start[None], max_distance=max_distance, min_eigenvalue=thr, M=j)
        if got["iters"][0] < j:
            break
        ran = j
        sums = gg._last(lib, odo.ctx, len(scan))[3]
        assert sums.tobytes() == _evaluate(lib, ev.ctx, scan, T_lin, max_distance).tobytes(), j
        if np.isinf(max_distance):
            assert got["inliers"][0] == sums[29]
        _check_step(T_lin, got, sums, thr)
        degenerate = max(degenerate, int(got["degenerate"][0]))
        T_lin = got["T"][0]
    assert ran >= 2 and degenerate > 0, (ran, degenerate)


# ------------------------------------------------------------------------------------------------ well constrained
@pytest.mark.parametrize("max_distance", [0.5, np.inf])
def test_a_threshold_below_every_eigenvalue_is_the_plain_solve(lib, maps, max_distance):
    """Jacobi and elimination round differently: each step differs in the last bits of its float64 solve, which the
    float32 cast of the step mostly absorbs; the poses agree to 1e-5 (rotation entries, and metres per metre of
    translation), ten float32 ulps of the largest entries, after the same iterations."""
    odo = gg._odometry("geman_mcclure", 10, max_iters=10)
    gg._set_map(odo, maps["warm"])
    scans = gg._scans(maps["warm"], [6000, -4000], 31)
    T0 = gg._poses(4, 31)
    of = np.array([0, 1, 0, 1], np.int32)
    if np.isinf(max_distance):
        _, ref = gg._register(lib, odo.ctx, scans, T0, of, M=10)
    else:
        _, ref = gg._register(lib, odo.ctx, scans, T0, of, max_distance, M=10)
    st, got = _register(lib, odo.ctx, scans, T0, of, max_distance, 1e-9, M=10)
    assert np.all(got["degenerate"] == 0) and np.all(got["eigenvalues"][:, 0] > 1e-9)
    assert np.array_equal(got["status"], ref["status"])
    d = np.abs(got["T"].astype(np.float64) - ref["T"])
    assert d[:, :3, :3].max() <= 1e-5 and np.all(d[:, :3, 3] <= 1e-5 * (1 + np.abs(ref["T"][:, :3, 3])))


# ------------------------------------------------------------------------------------------------ the scenes
def _scene_odometry(m, max_iters=30):
    odo = gg._odometry("default", 10, max_iters=max_iters)
    gg._set_map(odo, m)
    return odo


def test_flat_field(lib):
    """The field constrains z, roll and pitch and nothing else.  x, y and yaw are held: no step moves them, and the
    rotation steps, composed on the left about the map origin, move x and y by at most the rotation (4.2 mrad) times
    the start's lever arm above the plane (5 cm), 2.1e-4 m, and yaw by their second order."""
    m, s, truth, start = dr.flat_field_scene()
    odo = _scene_odometry(m)
    st, plain = gg._register(lib, odo.ctx, [s], start[None], M=30)
    assert plain["status"][0] == lib.PLS_E_SINGULAR
    st, got = _register(lib, odo.ctx, [s], start[None], min_eigenvalue=dr.FLAT_MIN_EIGENVALUE, M=30)
    assert got["status"][0] == lib.PLS_OK and got["degenerate"][0] == 3
    assert list(got["eigenvalues"][0, :3]) == [0.0, 0.0, 0.0]
    e, e0, et = dr.euler(got["T"][0]), dr.euler(start), dr.euler(truth)
    assert abs(e[2] - et[2]) <= 1e-3 and np.all(np.abs(e[3:5] - et[3:5]) <= 1e-4), e - et
    assert np.all(np.abs(e[:2] - e0[:2]) <= 2.5e-4) and abs(e[5] - e0[5]) <= 2e-5, e - e0


def test_tunnel(lib):
    """Only the translation along the axis is (nearly) unconstrained: it is held within 1e-4 m of the start -- the
    rotation steps about the origin move it by at most 1.7 mrad times the 2.5 cm lateral offset -- and the other five
    are recovered.  The plain solve, by contrast, lets the axis drift on the noise (DESIGN section 22)."""
    m, s, truth, start = dr.tunnel_scene()
    odo = _scene_odometry(m)
    st, got = _register(lib, odo.ctx, [s], start[None], min_eigenvalue=dr.TUNNEL_MIN_EIGENVALUE, M=30)
    assert got["status"][0] == lib.PLS_OK and got["degenerate"][0] == 1
    e, e0, et = dr.euler(got["T"][0]), dr.euler(start), dr.euler(truth)
    assert abs(e[0] - e0[0]) <= 1e-4, e - e0
    assert np.all(np.abs(e[1:3] - et[1:3]) <= 1e-3) and np.all(np.abs(e[3:] - et[3:]) <= 1e-4), e - et


# ------------------------------------------------------------------------------------------------ batches
BATCH_CASES = [("warm", 10, B) for B in (1, 63, 64, 65, 130)] + \
    [(which, k, B) for which, k in (("cold", 10), ("warm", 64)) for B in (1, 65, 130)]


@pytest.mark.parametrize("which,k,B", BATCH_CASES)
def test_batch_equals_single_calls(lib, maps, which, k, B):
    """Scans of 1 to 5000 rows at a threshold of 0.05: the small ones have degenerate directions, the large ones none.
    A batch equals single calls; host and device pointers agree; NULL optional outputs change no other output."""
    md, thr = (0.3 if B % 2 else np.inf), 0.05
    odo = gg._odometry("cauchy", k)
    gg._set_map(odo, maps[which])
    scans = gg._scans(maps["warm"], [255, 256, 257, 2048, -5000, 1, 2, 6], B, noise=0.15)
    rng = np.random.RandomState(B)
    of = rng.randint(0, len(scans), B).astype(np.int32)
    of[: min(B, len(scans))] = np.arange(min(B, len(scans)))
    T0 = gg._poses(B, B, spread=1.5)
    st, rows = _register(lib, odo.ctx, scans, T0, of, md, thr)
    _, rows_dev = _register(lib, odo.ctx, scans, T0, of, md, thr, dev=True)
    for key in KEYS:
        assert rows[key].tobytes() == rows_dev[key].tobytes(), key
    _, bare = _register(lib, odo.ctx, scans, T0, of, md, thr, nulls=("inliers", "degenerate", "eigenvalues"))
    for key in ("T", "params", "losses", "iters", "status"):
        assert rows[key].tobytes() == bare[key].tobytes(), key
    assert np.all(bare["degenerate"] == -7) and np.all(bare["eigenvalues"] == -7.0)
    for b in range(B):
        _, one = _register(lib, odo.ctx, [scans[of[b]]], T0[b:b + 1], None, md, thr)
        for key in KEYS:
            assert one[key].tobytes() == rows[key][b:b + 1].tobytes(), (b, key)
    if B >= 8:   # every scan size is in the batch
        assert np.any(rows["degenerate"] > 0) and np.any(rows["degenerate"] == 0)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_leave_outputs_and_context_unchanged(lib, maps):
    a, b = gg._odometry(max_iters=4), gg._odometry(max_iters=4)
    lma, lmb = gg._set_map(a, maps["warm"]), gg._set_map(b, maps["warm"])
    scans = gg._scans(maps["warm"], [1000, 2000], 4)
    T0 = gg._poses(2, 4)
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([1000, 2000], np.int64)
    f = lib.load().pls_register_scans_degeneracy
    h = a.ctx.handle
    outs = [np.full((2, 16), 7.0, np.float32), np.full((2, 6), 7.0, np.float32), np.full((2, 4), 7.0, np.float32),
            np.full(2, 7, np.int32), np.full(2, 7, np.int32), np.full(2, 7, np.int32), np.full(2, 7, np.int32),
            np.full((2, 6), 7.0)]
    tail = [lib.ptr(o) for o in outs]
    bad_n, null_addr = np.array([1000, 0], np.int64), np.array([lib.ptr(scans[0]), 0], np.uint64)
    ok = (lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 2)
    cases = [
        (h, lib.ptr(addr), lib.ptr(n), 0, None, lib.ptr(T0), 2, 1.0, 1e-3),           # S = 0
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 0, 1.0, 1e-3),           # B = 0
        (h, lib.ptr(addr), lib.ptr(bad_n), 2, None, lib.ptr(T0), 2, 1.0, 1e-3),       # n[s] = 0
        (h, lib.ptr(null_addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, 1.0, 1e-3),      # NULL scan
        (h, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(np.array([0, 2], np.int32)), lib.ptr(T0), 2, 1.0, 1e-3),
        (h, lib.ptr(addr), lib.ptr(n), 1, None, lib.ptr(T0), 2, 1.0, 1e-3),           # B != S, no scan_of
        (h, None, lib.ptr(n), 2, None, lib.ptr(T0), 2, 1.0, 1e-3),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, None, 2, 1.0, 1e-3),
        (h, *ok, -1.0, 1e-3),
        (h, *ok, float("nan"), 1e-3),
        (h, *ok, 1.0, 0.0),
        (h, *ok, np.inf, -1e-3),
        (h, *ok, 1.0, float("nan")),
        (h, *ok, np.inf, np.inf),
        (h, *ok, 1.0, -np.inf),
    ]
    for i, args in enumerate(cases):
        assert f(*args, *tail) == lib.PLS_E_INVALID, i
        assert all(np.all(o == 7) for o in outs), i
    assert gg._twin_state(lma, a) == gg._twin_state(lmb, b)
    for odo in (gg._odometry(), gg._odometry(local_map="projective_local_map")):   # no map yet; a projective map
        assert f(odo.ctx.handle, *ok, 1.0, 1e-3, *tail) == lib.PLS_E_INVALID
        assert all(np.all(o == 7) for o in outs)


# ------------------------------------------------------------------------------------------------ Python
@pytest.mark.parametrize("max_distance", [0.4, np.inf])
def test_python_methods_make_the_c_call(lib, maps, max_distance):
    odo = gg._odometry("huber", 10, max_iters=6)
    gg._set_map(odo, maps["warm"])
    scans = gg._scans(maps["warm"], [3000, 40], 41)
    T0 = gg._poses(3, 41)
    of = np.array([0, 1, 1], np.int32)
    st, c = _register(lib, odo.ctx, scans, T0, of, max_distance, 0.05, M=6)
    params, T, losses, iters = odo.register_new_frames(scans, T0, of, max_distance=max_distance, min_eigenvalue=0.05)
    assert T.tobytes() == c["T"].tobytes() and params.tobytes() == c["params"].tobytes()
    assert iters.tobytes() == c["iters"].tobytes() and odo.last_registrations_status.tobytes() == c["status"].tobytes()
    assert [list(x) for x in losses] == [list(c["losses"][b, :c["iters"][b]]) for b in range(3)]
    assert odo.last_registrations_degenerate.tobytes() == c["degenerate"].tobytes()
    assert odo.last_registrations_eigenvalues.tobytes() == c["eigenvalues"].tobytes()
    if np.isinf(max_distance):
        assert odo.last_registrations_inliers is None
    else:
        assert odo.last_registrations_inliers.tobytes() == c["inliers"].tobytes()
    _, Th, _, _ = odo.register_new_frame_hypotheses(scans[1], T0, max_distance=max_distance, min_eigenvalue=0.05)
    _, ch = _register(lib, odo.ctx, [scans[1]], T0, np.zeros(3, np.int32), max_distance, 0.05, M=6)
    assert Th.tobytes() == ch["T"].tobytes()
    assert odo.last_hypotheses_degenerate.tobytes() == ch["degenerate"].tobytes()
    assert odo.last_hypotheses_eigenvalues.tobytes() == ch["eigenvalues"].tobytes()
