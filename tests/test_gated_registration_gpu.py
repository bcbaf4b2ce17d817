"""Registration on a prior map with a correspondence gate: pls_register_scans_gated and the max_distance of
ICPFrameToModel.register_new_frames.

  * at max_distance = +inf, and at a finite gate above every match distance of every iteration, the bits of
    pls_register_scans for every scheme, on a map below KD_COLD_MAP_POINTS and one above, at k = 10 and 64 (both
    later-iteration paths: the one-kernel refine and the four launches);
  * one gated iteration's matches equal the ungated search's wherever the float64 gate admits them; gates met exactly,
    one ulp below, queries far outside the grid's box and in empty space;
  * a gated one-alignment registration's sums are entries 0..29 of pls_kdmap_evaluate_poses at the same gate, bit for
    bit;
  * every iteration against the ungated search plus the float64 gate at that iteration's pose (and the brute-force
    gated 1-NN on small maps): matches, exact inlier count, sums within float32_tolerance, the pose update; on the
    one-kernel refine path, on both four-launch cases (k = 64, a map of 2 M points) and on a map with overflowed cell
    tables, with rows that cross the gate in both directions;
  * batches across the PLS_MAX_SEQUENCES chunk edges equal single calls on both later-iteration paths; host and device
    pointers; out_inliers against the ungated matches plus the float64 gate;
  * every refusal leaves the outputs and the context unchanged;
  * on the changed-map scene the gated registration recovers the truth and the ungated one does not (the scenario and
    its tolerance are the CPU oracle's, tests/test_gated_registration_cpu.py).
"""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
COLD_MAP_POINTS = 2_000_000  # kdmap.cu: KD_COLD_MAP_POINTS
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def _scene_cloud():
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    parts = []
    for k in range(0, 40, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k).astype(np.float64)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.3)[0]))
    return np.ascontiguousarray(np.concatenate(parts).astype(np.float32))


@pytest.fixture(scope="module")
def maps():
    warm = _scene_cloud()
    rng = np.random.RandomState(3)
    fill = rng.uniform([-80, -80, -2], [80, 80, 4], (COLD_MAP_POINTS, 3)).astype(np.float32)
    return dict(warm=warm, cold=np.ascontiguousarray(np.concatenate([warm, fill])))


def _odometry(scheme="geman_mcclure", k=10, max_iters=5, local_map="kdtree_local_map"):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=max_iters, threshold_delta_pose=1e-4, data_key="numpy_pc",
               local_map=dict(type=local_map, local_map_size=20, num_neighbors_normals=k),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme=scheme, sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def _set_map(odo, cloud):
    import pylidar_slam_b200 as b200
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20), ctx=odo.ctx)
    lm.set_map_pointcloud(cloud)
    return lm


def _scans(warm, sizes, seed, noise=0.05):
    """Map points with noise; size < 0: that many rows with every 97th row NaN."""
    rng = np.random.RandomState(seed)
    out = []
    for n in sizes:
        s = warm[rng.choice(len(warm), abs(n), replace=abs(n) > len(warm))]
        s = np.ascontiguousarray((s + rng.normal(0, noise, s.shape)).astype(np.float32))
        if n < 0:
            s[::97] = np.nan
        out.append(s)
    return out


def _poses(B, seed, spread=0.8):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(1, B):
        T[b, :3, :3] = Rotation.from_euler("z", rng.uniform(-4, 4), degrees=True).as_matrix()
        T[b, :3, 3] = rng.uniform(-spread, spread, 3) * [1, 1, 0.1]
    return T


def _register(lib, ctx, scans, T0, scan_of=None, max_distance=None, M=5, dev=False):
    """pls_register_scans (max_distance None) or pls_register_scans_gated.  Returns (status, dict of outputs)."""
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([s.shape[0] for s in scans], np.int64)
    B = T0.shape[0]
    o = dict(T=np.zeros((B, 4, 4), np.float32), params=np.zeros((B, 6), np.float32),
             losses=np.zeros((B, M), np.float32), iters=np.zeros(B, np.int32), status=np.zeros(B, np.int32),
             inliers=np.full(B, -7, np.int32))
    of = None if scan_of is None else lib.ptr(np.asarray(scan_of, np.int32))
    if max_distance is None:
        st = lib.load().pls_register_scans(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans), of, lib.ptr(T0), B,
                                           lib.ptr(o["T"]), lib.ptr(o["params"]), lib.ptr(o["losses"]),
                                           lib.ptr(o["iters"]), lib.ptr(o["status"]))
        del o["inliers"]
        return st, o
    if dev:
        import torch
        keep = [torch.from_numpy(s).cuda() for s in scans]
        addr = np.array([t.data_ptr() for t in keep], np.uint64)
        Td = torch.from_numpy(np.ascontiguousarray(T0)).cuda()
        outs = {k: torch.from_numpy(v).cuda() for k, v in o.items()}
        st = lib.load().pls_register_scans_gated(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans), of, Td.data_ptr(),
                                                 B, float(max_distance), *[outs[k].data_ptr() for k in o])
        return st, {k: v.cpu().numpy() for k, v in outs.items()}
    st = lib.load().pls_register_scans_gated(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans), of, lib.ptr(T0), B,
                                             float(max_distance), *[lib.ptr(v) for v in o.values()])
    return st, o


def _same(a, b, keys=("T", "params", "losses", "iters", "status")):
    for k in keys:
        assert a[k].tobytes() == b[k].tobytes(), k


def _last(lib, ctx, nq):
    idx, nb, nrm = np.empty(nq, np.int64), np.empty((nq, 3), np.float32), np.empty((nq, 3), np.float32)
    sums = np.empty(30, np.float64)
    assert lib.load().pls_kdmap_last_correspondences(ctx.handle, nq, lib.ptr(idx), lib.ptr(nb), lib.ptr(nrm), None,
                                                     lib.ptr(sums)) == lib.PLS_OK
    return idx, nb, nrm, sums


# ------------------------------------------------------------------------------------------------ the anchor
@pytest.mark.parametrize("scheme", SCHEMES)
@pytest.mark.parametrize("k", [10, 64])
@pytest.mark.parametrize("which", ["warm", "cold"])
def test_inf_and_a_wide_gate_give_the_ungated_bits(lib, maps, which, k, scheme):
    odo = _odometry(scheme, k)
    _set_map(odo, maps[which])
    scans = _scans(maps["warm"], [-6000, 3000], 1)
    T0 = _poses(4, 2)
    of = np.array([0, 1, 0, 1], np.int32)
    st, ref = _register(lib, odo.ctx, scans, T0, of)
    assert st == lib.PLS_OK
    for md in (np.inf, 50.0):   # 50 m: above every match distance of every iteration (poses within 1 m of the map)
        st, got = _register(lib, odo.ctx, scans, T0, of, md)
        assert st == lib.PLS_OK
        _same(ref, got)
        nq = np.array([np.sum(~np.isnan(scans[s]).any(1)) for s in of])
        assert np.array_equal(got["inliers"], nq)   # every valid row is an inlier


# ------------------------------------------------------------------------------------------------ one iteration
@pytest.mark.parametrize("which", ["warm", "cold"])
@pytest.mark.parametrize("max_distance", [0.03, 0.1, 0.4])
def test_one_gated_iteration_keeps_every_inlier_match(lib, maps, which, max_distance):
    from oracle import evaluate_poses_reference as er
    from oracle import projection_reference as pr
    odo = _odometry("geman_mcclure", max_iters=1)
    _set_map(odo, maps[which])
    scan = _scans(maps["warm"], [8000], 5, noise=0.1)[0]
    # rows far outside the grid's box and in empty space above the scene
    far = np.float32([[5000, 0, 0], [-3000, 2000, 100], [0, 0, 1e6], [0, 0, 60], [10, -10, 45]])
    scan = np.ascontiguousarray(np.concatenate([scan, far]))
    T0 = _poses(2, 6)[1:]
    st, _ = _register(lib, odo.ctx, [scan], T0, M=1)
    assert st == lib.PLS_OK
    ref_idx, ref_nb, _, _ = _last(lib, odo.ctx, len(scan))
    st, got = _register(lib, odo.ctx, [scan], T0, max_distance=max_distance, M=1)
    assert st in (lib.PLS_OK, lib.PLS_E_SINGULAR)
    idx, nb, _, sums = _last(lib, odo.ctx, len(scan))
    p = pr.transform32(T0[0], scan)
    inl = er.inliers(p, ref_nb, ref_idx >= 0, max_distance)
    assert 0 < inl.sum() < len(scan)
    assert np.array_equal(idx[inl], ref_idx[inl])               # every inlier: the ungated match
    assert np.all((idx[~inl] == -1) | (idx[~inl] == ref_idx[~inl]))
    assert np.all(idx[-5:] == -1)
    assert sums[29] == inl.sum() == got["inliers"][0]


def test_gates_met_exactly():
    """A dyadic map (4 m grid) and a scan 0.5 m beside it: every d is exactly 0.5."""
    from pylidar_slam_b200 import _lib as lib
    g = np.mgrid[0:40:4.0, 0:40:4.0, 0:12:4.0].reshape(3, -1).T.astype(np.float32)
    odo = _odometry("default", max_iters=1)
    _set_map(odo, g)
    scan = np.ascontiguousarray(g + np.float32([0.5, 0, 0]))
    T0 = np.eye(4, dtype=np.float32)[None]
    st, got = _register(lib, odo.ctx, [scan], T0, max_distance=0.5, M=1)
    assert got["inliers"][0] == len(g)
    assert np.all(_last(lib, odo.ctx, len(g))[0] >= 0)
    for md in (np.nextafter(0.5, 0), 0.0):
        st, got = _register(lib, odo.ctx, [scan], T0, max_distance=md, M=1)
        # no inlier: nothing to solve, the registration is singular and keeps its start
        assert got["inliers"][0] == 0 and got["status"][0] == lib.PLS_E_SINGULAR and got["iters"][0] == 1
        assert got["T"].tobytes() == T0.tobytes()
        assert np.all(_last(lib, odo.ctx, len(g))[0] == -1)


# ------------------------------------------------------------------------------------------------ evaluation anchor
@pytest.mark.parametrize("max_distance", [0.0, 0.05, 0.3, np.inf])
def test_first_iteration_is_the_evaluation_row(lib, maps, max_distance):
    odo = _odometry("huber", max_iters=1)
    _set_map(odo, maps["warm"])
    scans = _scans(maps["warm"], [-7000, 2500], 11, noise=0.08)
    T0 = _poses(3, 11)
    of = np.array([1, 0, 1], np.int32)
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([s.shape[0] for s in scans], np.int64)
    rows = np.zeros((3, 32))
    assert lib.load().pls_kdmap_evaluate_poses(odo.ctx.handle, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(of), lib.ptr(T0),
                                               3, float(max_distance), lib.ptr(rows)) == lib.PLS_OK
    for b in range(3):
        _register(lib, odo.ctx, [scans[of[b]]], T0[b:b + 1], max_distance=max_distance, M=1)
        nq = int(np.sum(~np.isnan(scans[of[b]]).any(1)))
        assert _last(lib, odo.ctx, nq)[3].tobytes() == rows[b, :30].tobytes(), b


# ------------------------------------------------------------------------------------------------ every iteration
U = 2.0 ** -24
POLE = np.array([2.0, 1.0, 4.0])   # a thin cluster in free space, 4 m above the room's floor


def _room_scene(seed):
    """The changed-map room, subsampled, with a pole cluster added to the map and two groups of scan rows that cross
    the gate: 20 on the pole at the truth (outliers at the start, 0.4 m off) and 20 on the pole at the start
    (inliers there, outliers once the pose has moved towards the truth)."""
    from oracle import gated_registration_reference as gr
    prior, scan, _, start = gr.changed_map_scene(seed)
    rng = np.random.RandomState(seed)
    pole = POLE + rng.normal(0, 0.03, (40, 3))
    prior = np.concatenate([prior[rng.choice(len(prior), 5000, replace=False)], pole])
    at_truth = POLE + rng.normal(0, 0.03, (20, 3))
    S = start.astype(np.float64)
    at_start = (POLE + rng.normal(0, 0.03, (20, 3)) - S[:3, 3]) @ S[:3, :3]   # start^-1 applied
    scan = np.concatenate([scan[rng.choice(len(scan), 1960, replace=False)], at_truth, at_start])
    return np.ascontiguousarray(prior, np.float32), np.ascontiguousarray(scan, np.float32), start, 0.25


def _overflow_scene(seed):
    """The clusters-in-a-lattice map of test_kd_overflow_gpu.py, whose coarser cell tables overflow, and a scan of
    its points and of points in the lattice's empty gaps."""
    import test_kd_overflow_gpu as ov
    m = ov._map(seed)
    levels = ov._table_cells(m, local_map_size=1)
    assert any(cells > slots for cells, slots in levels[1:]), levels
    rng = np.random.RandomState(seed)
    on = m[rng.choice(len(m), 1500, replace=False)] + rng.normal(0, 0.05, (1500, 3))
    gaps = rng.uniform(0, 26, (500, 3))
    start = np.eye(4, dtype=np.float32)
    c, s = np.cos(np.deg2rad(1.0)), np.sin(np.deg2rad(1.0))
    start[:2, :2] = [[c, -s], [s, c]]
    start[:3, 3] = [0.15, -0.1, 0.05]
    return m, np.ascontiguousarray(np.concatenate([on, gaps]), np.float32), start, 0.3


def _scene(name):
    """(map, scan, start, gate, k, local_map_size, brute force?) of an every-iteration scene."""
    if name == "overflow":
        m, scan, start, md = _overflow_scene(0)
        return m, scan, start, md, 10, 1, True
    m, scan, start, md = _room_scene(4)
    if name == "cold":   # 2 M points far from the room: the four-launch later iterations at k = 10
        fill = np.random.RandomState(5).uniform([40, -80, -2], [200, 80, 4], (COLD_MAP_POINTS, 3))
        return np.ascontiguousarray(np.concatenate([m, fill.astype(np.float32)])), scan, start, md, 10, 20, False
    return m, scan, start, md, (64 if name == "wide_k" else 10), 20, True


def _load(odo, m, lms):
    import pylidar_slam_b200 as b200
    if lms == 20:
        return _set_map(odo, m)
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=lms, num_neighbors_normals=10), ctx=odo.ctx)
    lm.init()
    lm.update(np.eye(4, dtype=np.float32)[None], new_pc_data=m)
    return lm


def _odometry_lms(scheme, k, max_iters, lms):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=max_iters, threshold_delta_pose=1e-4, data_key="numpy_pc",
               local_map=dict(type="kdtree_local_map", local_map_size=lms, num_neighbors_normals=k),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme=scheme, sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def _check_pose_update(kref, T_lin, got, sums, j):
    """losses[j-1] is sums[27] in float32; the pose is the float64 solve of the GPU's sums applied to T_lin through
    the Euler round trip, to float32 resolution (test_kd_icp_iterations_gpu.py's bound)."""
    import torch
    from oracle import icp_oracle as orc
    assert got["losses"][0, j - 1] == np.float32(sums[27])
    dx = kref.gauss_newton_step(sums).astype(np.float32).astype(np.float64)
    dT = orc.build_pose_matrix(torch.from_numpy(dx)[None])[0].numpy()
    prm = orc.from_pose_matrix(torch.from_numpy(dT @ np.asarray(T_lin, np.float64))[None])
    T_exp = orc.build_pose_matrix(prm)[0].numpy()
    T = got["T"][0].astype(np.float64)
    scale = 1 + np.abs(T_exp[:3, 3]).sum()
    assert np.abs(T[:3, :3] - T_exp[:3, :3]).max() <= 2e-6
    assert np.abs(T[:3, 3] - T_exp[:3, 3]).max() <= 2e-6 * scale


@pytest.mark.parametrize("name", ["refine", "wide_k", "cold", "overflow"])
def test_every_iteration_against_the_oracle(lib, name):
    """Iteration j of a gated registration, read back after max_num_alignments = j, at the pose it ran at (the result
    of j - 1 alignments): its matches are the ungated search's at that pose wherever the float64 gate admits them (and
    the brute-force gated 1-NN's on the small maps); its inlier count is exact; its sums are kd_icp_reference's over
    those inliers within float32_tolerance; its pose update is the solve of its sums.  "refine" takes the one-kernel
    later iterations; "wide_k" (k = 64), "cold" (2 M points) the four launches; "overflow" a map with overflowed
    cell tables."""
    from oracle import evaluate_poses_reference as er
    from oracle import kd_icp_reference as kref
    from oracle import gated_registration_reference as gr
    from oracle import projection_reference as pr
    m, scan, start, md, k, lms, brute = _scene(name)
    scheme, K = "default", 6
    positions = kref.kernel_sort_positions(m) if brute else None
    ungated = _odometry_lms(scheme, k, 1, lms)
    _load(ungated, m, lms)
    inside = []
    T_lin, ran = start, 0
    for j in range(1, K + 1):
        odo = _odometry_lms(scheme, k, j, lms)
        _load(odo, m, lms)
        st, got = _register(lib, odo.ctx, [scan], start[None], max_distance=md, M=j)
        if got["iters"][0] < j:   # stopped before iteration j
            break
        ran = j
        idx, _, _, sums = _last(lib, odo.ctx, len(scan))
        _register(lib, ungated.ctx, [scan], T_lin[None], M=1)
        idx_u, nb_u, nrm_u, _ = _last(lib, ungated.ctx, len(scan))
        p32 = pr.transform32(T_lin, scan)
        inl = er.inliers(p32, nb_u, idx_u >= 0, md)
        assert 0 < inl.sum() < len(scan), (j, int(inl.sum()))
        assert np.array_equal(idx[inl], idx_u[inl]), j
        assert np.all((idx[~inl] == -1) | (idx[~inl] == idx_u[~inl])), j
        assert sums[29] == inl.sum() == got["inliers"][0], (j, sums[29], int(inl.sum()))
        if brute:
            want, decided = gr.brute_force_gated_nn(m, positions, p32, md)
            sure = decided & (want >= 0)
            assert np.array_equal(idx[sure], want[sure]), j
            assert np.array_equal((want >= 0)[decided], inl[decided]), j
        p64 = kref.transform(np.asarray(T_lin, np.float64), scan)[inl]
        q64, n64 = nb_u[inl].astype(np.float64), nrm_u[inl].astype(np.float64)
        exact = kref.accumulate(p64, q64, n64, scheme, 0.3)
        e = 8 * 2 * U * (np.linalg.norm(p64, axis=1) + np.linalg.norm(q64, axis=1))
        tol = kref.float32_tolerance(p64, q64, n64, scheme, 0.3, e)
        err = np.abs(sums - exact)
        assert (err <= tol).all(), (j, np.nonzero(err > tol)[0], (err / tol).max())
        if got["status"][0] == lib.PLS_OK and got["T"][0].tobytes() != np.asarray(T_lin, np.float32).tobytes():
            _check_pose_update(kref, T_lin, got, sums, j)
        inside.append(inl)
        T_lin = got["T"][0]
    assert ran >= 2, ran
    if name != "overflow":   # the pole rows cross the gate in both directions between iterations
        seq = np.array(inside)[:, -40:]
        assert np.any(~seq[0, :20] & seq[-1, :20]), "no row entered the gate"
        assert np.any(seq[0, 20:] & ~seq[-1, 20:]), "no row left the gate"


# ------------------------------------------------------------------------------------------------ batches
BATCH_CASES = [("warm", 10, B) for B in (1, 2, 63, 64, 65, 130)] + \
    [(which, k, B) for which, k in (("cold", 10), ("warm", 64)) for B in (1, 65, 130)]


@pytest.mark.parametrize("which,k,B", BATCH_CASES)
def test_batch_equals_single_calls(lib, maps, which, k, B):
    """A gate (0.3 m) with outliers in every registration, on the refine path (warm, k = 10) and the four launches
    (cold, k = 64): a batch equals single calls, host and device pointers agree, and at one alignment each
    out_inliers is the count of the ungated matches within the float64 gate."""
    from oracle import evaluate_poses_reference as er
    from oracle import projection_reference as pr
    md = 0.3
    odo = _odometry("cauchy", k)
    _set_map(odo, maps[which])
    scans = _scans(maps["warm"], [255, 256, 257, 2048, -5000, 1, 2], B, noise=0.15)
    rng = np.random.RandomState(B)
    of = rng.randint(0, len(scans), B).astype(np.int32)
    of[: min(B, len(scans))] = np.arange(min(B, len(scans)))
    T0 = _poses(B, B, spread=1.5)
    st, rows = _register(lib, odo.ctx, scans, T0, of, md)
    _, rows_dev = _register(lib, odo.ctx, scans, T0, of, md, dev=True)
    _same(rows, rows_dev, ("T", "params", "losses", "iters", "status", "inliers"))
    for b in range(B):
        _, one = _register(lib, odo.ctx, [scans[of[b]]], T0[b:b + 1], None, md)
        for key in ("T", "params", "losses", "iters", "status", "inliers"):
            assert one[key].tobytes() == rows[key][b:b + 1].tobytes(), (b, key)
    nq = int(np.sum(~np.isnan(scans[of[-1]]).any(1)))
    assert _last(lib, odo.ctx, nq)[3][29] == rows["inliers"][-1]
    # one alignment: out_inliers against the ungated search plus the float64 gate at each start
    one = _odometry("cauchy", k, max_iters=1)
    _set_map(one, maps[which])
    _, first = _register(lib, one.ctx, scans, T0, of, md, M=1)
    valid = [s[~np.isnan(s).any(1)] for s in scans]
    outliers = 0
    for b in range(B):
        _register(lib, one.ctx, [scans[of[b]]], T0[b:b + 1], M=1)
        idx_u, nb_u, _, _ = _last(lib, one.ctx, len(valid[of[b]]))
        count = int(er.inliers(pr.transform32(T0[b], valid[of[b]]), nb_u, idx_u >= 0, md).sum())
        assert first["inliers"][b] == count, (b, int(first["inliers"][b]), count)
        outliers += len(valid[of[b]]) - count
    assert outliers > 0


# ------------------------------------------------------------------------------------------------ refusals
def _twin_state(lm, odo):
    from pylidar_slam_b200 import synthetic as syn
    pts, counts = lm.points().tobytes(), list(lm.frame_counts())
    scan = _scans(np.asarray(lm.points()), [2000], 13)[0]
    _, T, _ = odo.register_new_frame(scan, np.eye(4, dtype=np.float32))
    pc = np.ascontiguousarray(syn.scan(0, 16, 256), np.float32)
    odo.process_next_frame({"numpy_pc": pc})
    return pts, counts, T.tobytes(), odo.get_relative_poses().tobytes()


def test_refusals_leave_outputs_and_context_unchanged(lib, maps):
    a, b = _odometry(max_iters=4), _odometry(max_iters=4)
    lma, lmb = _set_map(a, maps["warm"]), _set_map(b, maps["warm"])
    scans = _scans(maps["warm"], [1000, 2000], 4)
    T0 = _poses(2, 4)
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([1000, 2000], np.int64)
    f = lib.load().pls_register_scans_gated
    h = a.ctx.handle
    outs = [np.full((2, 16), 7.0, np.float32), np.full((2, 6), 7.0, np.float32), np.full((2, 4), 7.0, np.float32),
            np.full(2, 7, np.int32), np.full(2, 7, np.int32), np.full(2, 7, np.int32)]
    tail = [lib.ptr(o) for o in outs]
    bad_n, null_addr = np.array([1000, 0], np.int64), np.array([lib.ptr(scans[0]), 0], np.uint64)
    cases = [
        (h, lib.ptr(addr), lib.ptr(n), 0, None, lib.ptr(T0), 2, 1.0),           # S = 0
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 0, 1.0),           # B = 0
        (h, lib.ptr(addr), lib.ptr(bad_n), 2, None, lib.ptr(T0), 2, 1.0),       # n[s] = 0
        (h, lib.ptr(null_addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, 1.0),      # NULL scan
        (h, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(np.array([0, 2], np.int32)), lib.ptr(T0), 2, 1.0),
        (h, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(np.array([-1, 0], np.int32)), lib.ptr(T0), 2, 1.0),
        (h, lib.ptr(addr), lib.ptr(n), 1, None, lib.ptr(T0), 2, 1.0),           # B != S, no scan_of
        (h, None, lib.ptr(n), 2, None, lib.ptr(T0), 2, 1.0),
        (h, lib.ptr(addr), None, 2, None, lib.ptr(T0), 2, 1.0),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, None, 2, 1.0),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, -1.0),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, float("nan")),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, -np.inf),
    ]
    for i, args in enumerate(cases):
        assert f(*args, *tail) == lib.PLS_E_INVALID, i
        assert all(np.all(o == 7) for o in outs), i
    assert _twin_state(lma, a) == _twin_state(lmb, b)
    for odo in (_odometry(), _odometry(local_map="projective_local_map")):   # no map yet; a projective map
        assert f(odo.ctx.handle, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T0), 2, 1.0, *tail) == lib.PLS_E_INVALID
        assert all(np.all(o == 7) for o in outs)


# ------------------------------------------------------------------------------------------------ changed map
def test_changed_map_gated_recovers_the_truth():
    from oracle import gated_registration_reference as gr
    import test_gated_registration_cpu as cpu
    prior, scan, truth, start = gr.changed_map_scene(0)
    odo = _odometry("default", max_iters=30)
    _set_map(odo, prior)
    _, Tg, _, _ = odo.register_new_frames([scan], start[None], max_distance=cpu.CHANGED_MAP_GATE)
    assert odo.last_registrations_inliers[0] == 18000   # the room's rows; none of the object's
    _, Tu, _, _ = odo.register_new_frames([scan], start[None])
    et, er_ = gr.pose_error(Tg[0], truth)
    assert et <= cpu.CHANGED_MAP_TOL[0] and er_ <= cpu.CHANGED_MAP_TOL[1], (et, er_)
    assert gr.pose_error(Tu[0], truth)[0] >= cpu.CHANGED_MAP_UNGATED_MIN
