"""The quality of many registrations on a prior map in one call: pls_kdmap_evaluate_poses and
ICPFrameToModel.evaluate_registrations.

  * at max_distance = inf, entries 0..29 are bit for bit the sums of a one-alignment pls_register_frame, for every
    scheme, on a cfg2-sized map and on one above KD_COLD_MAP_POINTS, at k = 10 and a wide k;
  * with finite gates the inlier set is the reference's over the GPU's own matches and normals (p' from
    transform_point's bits, oracle/projection_reference.transform32); gates met exactly count;
  * a batch equals single-pose calls bit for bit at every chunk edge, with scans at the residual kernel's block edges
    and a scan of only NaN rows;
  * host, device and mixed pointers; every refusal leaves the outputs and the context untouched;
  * the Python layer on a planar map and on a scan with outliers.
"""
import os
import re
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
COLD_MAP_POINTS = 2_000_000  # kdmap.cu: KD_COLD_MAP_POINTS
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


def _kd_threads():
    src = open(os.path.join(ROOT, "pylidar_slam_b200", "csrc", "kdmap.cu")).read()
    return int(re.search(r"constexpr int KD_THREADS = (\d+);", src).group(1))


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


def _odometry(scheme="geman_mcclure", k=10, max_iters=1, local_map="kdtree_local_map"):
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
    """Map points with noise; size < 0: that many rows with every 97th row NaN; size 0: 50 rows of NaN only."""
    rng = np.random.RandomState(seed)
    out = []
    for n in sizes:
        if n == 0:
            out.append(np.full((50, 3), np.nan, np.float32))
            continue
        s = warm[rng.choice(len(warm), abs(n), replace=abs(n) > len(warm))]
        s = np.ascontiguousarray((s + rng.normal(0, noise, s.shape)).astype(np.float32))
        if n < 0:
            s[::97] = np.nan
        out.append(s)
    return out


def _poses(B, seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(1, B):
        T[b, :3, :3] = Rotation.from_euler("z", rng.uniform(-4, 4), degrees=True).as_matrix()
        T[b, :3, 3] = rng.uniform(-0.8, 0.8, 3) * [1, 1, 0.1]
    return T


def _eval(lib, ctx, scans, T, scan_of=None, max_distance=np.inf, out=None):
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([s.shape[0] for s in scans], np.int64)
    B = T.shape[0]
    out = np.zeros((B, 32), np.float64) if out is None else out
    st = lib.load().pls_kdmap_evaluate_poses(ctx.handle, lib.ptr(addr), lib.ptr(n), len(scans),
                                             None if scan_of is None else lib.ptr(np.asarray(scan_of, np.int32)),
                                             lib.ptr(T), B, float(max_distance), lib.ptr(out))
    return st, out


def _single_icp_sums(lib, ctx, scan, T0):
    import ctypes as C
    T, p, losses, iters = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(1, np.float32), C.c_int(0)
    lib.load().pls_register_frame(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(T0), lib.ptr(T), lib.ptr(p),
                                  lib.ptr(losses), C.byref(iters))
    nq = int(np.sum(~np.isnan(scan).any(1)))
    sums = np.empty(30, np.float64)
    assert lib.load().pls_kdmap_last_correspondences(ctx.handle, nq, None, None, None, None, lib.ptr(sums)) == lib.PLS_OK
    return sums


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
def test_inf_gate_is_the_first_icp_iteration_bit_for_bit(lib, maps, which, k, scheme):
    odo = _odometry(scheme, k)
    _set_map(odo, maps[which])
    scans = _scans(maps["warm"], [-6000, 3000], 1)
    T = _poses(4, 2)
    of = np.array([0, 1, 0, 1], np.int32)
    st, rows = _eval(lib, odo.ctx, scans, T, of)
    assert st == lib.PLS_OK
    for b in range(4):
        sums = _single_icp_sums(lib, odo.ctx, scans[of[b]], T[b])
        assert rows[b, :30].tobytes() == sums.tobytes(), b
        assert rows[b, 31] == np.sum(~np.isnan(scans[of[b]]).any(1))
        assert rows[b, 29] == rows[b, 31]   # every valid row matched and admitted


# ------------------------------------------------------------------------------------------------ gated sums
@pytest.mark.parametrize("max_distance", [0.02, 0.05, 0.1, 0.5])
def test_gated_sums_against_the_reference(lib, maps, max_distance):
    from oracle import evaluate_poses_reference as er
    from oracle import projection_reference as pr
    odo = _odometry("geman_mcclure")
    _set_map(odo, maps["warm"])
    scan = _scans(maps["warm"], [-20000], 5)[0]
    T = _poses(2, 6)[1:]
    st, row = _eval(lib, odo.ctx, [scan], T, max_distance=max_distance)
    assert st == lib.PLS_OK
    valid = scan[~np.isnan(scan).any(1)]
    idx, nb, nrm, last_sums = _last(lib, odo.ctx, len(valid))
    p = pr.transform32(T[0], valid)
    ref, keep = er.evaluate_row(p, nb, nrm, idx >= 0, max_distance, "geman_mcclure", 0.3)
    assert 0 < keep.sum() < len(valid)
    assert row[0, 29] == keep.sum() and row[0, 31] == ref[31]
    assert last_sums.tobytes() == row[0, :30].tobytes()
    np.testing.assert_allclose(row[0, 30], ref[30], rtol=1e-12)
    # the float32 residual terms against their float64 images
    np.testing.assert_allclose(row[0, :29], ref[:29], rtol=2e-4, atol=1e-6 * np.abs(ref[:29]).max())


def test_gates_met_exactly_count(lib):
    """A dyadic map (4 m grid) and a scan 0.5 m beside it: every d is exactly 0.5."""
    g = np.mgrid[0:40:4.0, 0:40:4.0, 0:12:4.0].reshape(3, -1).T.astype(np.float32)
    odo = _odometry("default")
    _set_map(odo, g)
    scan = np.ascontiguousarray(g + np.float32([0.5, 0, 0]))
    T = np.eye(4, dtype=np.float32)[None]
    for md, want in ((0.5, len(g)), (np.nextafter(0.5, 0), 0), (np.inf, len(g))):
        st, row = _eval(lib, odo.ctx, [scan], T, max_distance=md)
        assert st == lib.PLS_OK and row[0, 29] == want and row[0, 31] == len(g)
        assert row[0, 30] == 0.25 * want
    st, row = _eval(lib, odo.ctx, [np.ascontiguousarray(g[::3])], T, max_distance=0.0)
    assert st == lib.PLS_OK and row[0, 29] == len(g[::3]) and row[0, 30] == 0.0


# ------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("B", [1, 2, 63, 64, 65, 130])
def test_batch_equals_single_calls(lib, maps, B):
    kt = _kd_threads()
    odo = _odometry("cauchy")
    _set_map(odo, maps["warm"])
    sizes = [kt - 1, kt, kt + 1, 8 * kt, 0, -5000, 1, 2]
    scans = _scans(maps["warm"], sizes, B)
    rng = np.random.RandomState(B)
    of = rng.randint(0, len(scans), B).astype(np.int32)
    of[: min(B, len(scans))] = np.arange(min(B, len(scans)))
    T = _poses(B, B)
    st, rows = _eval(lib, odo.ctx, scans, T, of, max_distance=0.3)
    assert st == lib.PLS_OK
    for b in range(B):
        st1, r1 = _eval(lib, odo.ctx, [scans[of[b]]], T[b:b + 1], max_distance=0.3)
        assert st1 == lib.PLS_OK and r1[0].tobytes() == rows[b].tobytes(), b
    nan_rows = rows[of == 4]
    assert np.all(nan_rows == 0)


def test_host_device_and_mixed_pointers(lib, maps):
    import torch
    odo = _odometry()
    _set_map(odo, maps["warm"])
    scans = _scans(maps["warm"], [3000, -4000], 9)
    T = _poses(3, 9)
    of = np.array([1, 0, 1], np.int32)
    st, host = _eval(lib, odo.ctx, scans, T, of, 0.2)
    assert st == lib.PLS_OK
    dev = [torch.from_numpy(s).cuda() for s in scans]
    Td = torch.from_numpy(T).cuda()
    for mix in ([dev[0], dev[1]], [scans[0], dev[1]], [dev[0], scans[1]]):
        addr = np.array([s.data_ptr() if isinstance(s, torch.Tensor) else lib.ptr(s) for s in mix], np.uint64)
        n = np.array([s.shape[0] for s in mix], np.int64)
        out = torch.zeros((3, 32), dtype=torch.float64, device="cuda")
        assert lib.load().pls_kdmap_evaluate_poses(odo.ctx.handle, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(of),
                                                   Td.data_ptr(), 3, 0.2, out.data_ptr()) == lib.PLS_OK
        assert out.cpu().numpy().tobytes() == host.tobytes()


# ------------------------------------------------------------------------------------------------ refusals
def _twin_state(lm, odo):
    from pylidar_slam_b200 import synthetic as syn
    pts, counts = lm.points().tobytes(), list(lm.frame_counts())
    scan = _scans(np.asarray(lm.points()), [2000], 13)[0]
    _, T, _ = odo.register_new_frame(scan, np.eye(4, dtype=np.float32))
    pc = np.ascontiguousarray(syn.scan(0, 16, 256), np.float32)
    d = {"numpy_pc": pc}
    odo.process_next_frame(d)
    return pts, counts, T.tobytes(), odo.get_relative_poses().tobytes()


def test_refusals_leave_outputs_and_context_unchanged(lib, maps):
    a, b = _odometry(max_iters=4), _odometry(max_iters=4)
    lma, lmb = _set_map(a, maps["warm"]), _set_map(b, maps["warm"])
    scans = _scans(maps["warm"], [1000, 2000], 4)
    T = _poses(2, 4)
    addr = np.array([lib.ptr(s) for s in scans], np.uint64)
    n = np.array([1000, 2000], np.int64)
    f = lib.load().pls_kdmap_evaluate_poses
    h = a.ctx.handle
    out = np.full((2, 32), 7.0)
    bad_n = np.array([1000, 0], np.int64)
    null_addr = np.array([lib.ptr(scans[0]), 0], np.uint64)
    cases = [
        (h, lib.ptr(addr), lib.ptr(n), 0, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),           # S = 0
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 0, 1.0, lib.ptr(out)),           # B = 0
        (h, lib.ptr(addr), lib.ptr(bad_n), 2, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),       # n[s] = 0
        (h, lib.ptr(null_addr), lib.ptr(n), 2, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),      # NULL scan
        (h, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(np.array([0, 2], np.int32)), lib.ptr(T), 2, 1.0, lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 2, lib.ptr(np.array([-1, 0], np.int32)), lib.ptr(T), 2, 1.0, lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 1, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),           # B != S, no scan_of
        (h, None, lib.ptr(n), 2, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),
        (h, lib.ptr(addr), None, 2, None, lib.ptr(T), 2, 1.0, lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, None, 2, 1.0, lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 2, 1.0, None),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 2, -1.0, lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 2, float("nan"), lib.ptr(out)),
        (h, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 2, -np.inf, lib.ptr(out)),
    ]
    for i, args in enumerate(cases):
        assert f(*args) == lib.PLS_E_INVALID, i
        assert np.all(out == 7.0), i
    assert _twin_state(lma, a) == _twin_state(lmb, b)
    # no map yet, and a projective map
    for odo in (_odometry(), _odometry(local_map="projective_local_map")):
        assert f(odo.ctx.handle, lib.ptr(addr), lib.ptr(n), 2, None, lib.ptr(T), 2, 1.0, lib.ptr(out)) == \
            lib.PLS_E_INVALID
        assert np.all(out == 7.0)


def test_map_and_frames_unchanged_and_last_search_adopted(lib, maps):
    a, b = _odometry(max_iters=4), _odometry(max_iters=4)
    lma, lmb = _set_map(a, maps["warm"]), _set_map(b, maps["warm"])
    scans = _scans(maps["warm"], [3000, -5000], 8)
    T = _poses(3, 8)
    st, rows = _eval(lib, a.ctx, scans, T, np.array([0, 1, 1], np.int32))
    assert st == lib.PLS_OK
    nq = int(np.sum(~np.isnan(scans[1]).any(1)))
    assert _last(lib, a.ctx, nq)[3].tobytes() == rows[2, :30].tobytes()
    assert _twin_state(lma, a) == _twin_state(lmb, b)


# ------------------------------------------------------------------------------------------------ Python layer
def test_planar_map_leaves_its_free_directions_unconstrained():
    rng = np.random.RandomState(0)
    plane = np.c_[rng.uniform(-30, 30, (60000, 2)), np.zeros(60000)].astype(np.float32)
    odo = _odometry("default")
    _set_map(odo, plane)
    scan = np.ascontiguousarray(plane[rng.choice(len(plane), 4000, replace=False)] + np.float32([0.01, 0.02, 0.0]))
    q = odo.evaluate_registrations([scan], np.eye(4, dtype=np.float32)[None], 0.5)[0]
    assert q.valid == 4000 and q.inliers == 4000 and q.fitness == 1.0
    free = q.eigenvectors[:, :3]
    for axis in (0, 1, 5):   # tx, ty, rz: the plane's free directions
        e = np.zeros(6)
        e[axis] = 1.0
        assert np.linalg.norm(free.T @ e) > 0.99
    # the cached normals are eigenvectors of float32 moments: the free directions are nearly, not exactly, null
    assert q.eigenvalues[2] < 1e-2 * q.eigenvalues[3]
    if q.covariance is not None:
        assert min(q.covariance[0, 0], q.covariance[1, 1], q.covariance[5, 5]) > 1e2 * q.covariance[2, 2]


def test_fitness_and_rmse_with_injected_outliers(maps):
    odo = _odometry("geman_mcclure")
    _set_map(odo, maps["warm"])
    rng = np.random.RandomState(1)
    on = maps["warm"][rng.choice(len(maps["warm"]), 8000, replace=False)]
    off = on[:2000] + np.float32([0, 0, 25.0])
    scan = np.ascontiguousarray(np.concatenate([on, off]))
    q, q_all = odo.evaluate_registrations([scan, scan], np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)), 1.0,
                                          [0, 0])[0], odo.evaluate_registrations([scan], np.eye(4, dtype=np.float32)[None])[0]
    assert q.valid == 10000 and q_all.inliers == 10000
    assert q.inliers >= 8000 and q.fitness < 0.85
    assert q.rmse < 0.05 and q_all.rmse > 1.0
