"""Localisation against a prior map on the GPU: KdTreeLocalMap.set_map_pointcloud, get_last_frame of both maps, and
ICPFrameToModel.register_new_frame_hypotheses (pls_register_hypotheses).

  * a set map holds the cloud in order, and every 1-NN search on it is exact against brute force, at sizes across the
    tile and wave edges of the kd kernels, at 5 M points, on a 2 km-wide sparse map (coarsened cells) and on 1 point;
  * the reference's own results (tests/golden/prior_map.npz) within the kd tolerances of tests/test_gpu_parity.py,
    including the eviction of prior-map rows and the errors it raises;
  * B hypotheses in one call are bit-identical to B pls_register_frame calls, on a cfg2-sized map and on one above
    KD_COLD_MAP_POINTS (the batched four-launch path), for B = 1, 2, 63, 64 and 65 (chunks), with a hypothesis that
    diverges and one that hits the tiny-residual guard; the launches of a later iteration do not grow with B.
"""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prior_map.npz")
COLD_MAP_POINTS = 2_000_000  # kdmap.cu: KD_COLD_MAP_POINTS
TILE, WAVE = 256, 8 * 132 * 256


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def kd_map(lib, size=3, ctx=None):
    import pylidar_slam_b200 as b200
    return b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=size), ctx=ctx)


def assert_exact_nn(lm, cloud, queries):
    res = lm.nearest_neighbor_search(np.ascontiguousarray(queries, np.float32), with_normals=False)
    d_mine = np.linalg.norm(res.neighbor_points.astype(np.float64) - queries.astype(np.float64), axis=1)
    d_ref, _ = cKDTree(cloud.astype(np.float64)).query(queries.astype(np.float64))
    np.testing.assert_allclose(d_mine, d_ref, rtol=1e-5, atol=1e-7)
    # the neighbour is a map point
    assert np.all(np.isin(res.neighbor_points.view(np.dtype((np.void, 12))).ravel(),
                          cloud.astype(np.float32).view(np.dtype((np.void, 12))).ravel()))


def _cloud(n, seed, extent=(60.0, 60.0, 4.0)):
    rng = np.random.RandomState(seed)
    ex = np.asarray(extent)
    return np.ascontiguousarray(rng.uniform(-ex / 2, ex / 2, (n, 3)).astype(np.float32))


@pytest.mark.parametrize("n", [1, 2, TILE - 1, TILE, TILE + 1, 132 * TILE, 132 * TILE + 1, WAVE - 1, WAVE + 1])
def test_set_points_in_order_and_exact_nn(lib, n):
    cloud = _cloud(n, n)
    lm = kd_map(lib)
    lm.set_map_pointcloud(cloud)
    assert lm.points().tobytes() == cloud.tobytes()
    assert lm.frame_counts() == []
    rng = np.random.RandomState(1)
    q = np.concatenate([cloud[rng.randint(0, n, 500)] + rng.normal(0, 0.2, (500, 3)).astype(np.float32),
                        _cloud(500, 2, (80.0, 80.0, 10.0))])
    assert_exact_nn(lm, cloud, q)


def test_set_points_five_million(lib):
    cloud = _cloud(5_000_000, 5, (200.0, 200.0, 10.0))
    lm = kd_map(lib)
    lm.set_map_pointcloud(cloud)
    assert lm.num_points() == 5_000_000
    assert lm.points().tobytes() == cloud.tobytes()
    rng = np.random.RandomState(3)
    q = cloud[rng.randint(0, len(cloud), 20000)] + rng.normal(0, 0.1, (20000, 3)).astype(np.float32)
    assert_exact_nn(lm, cloud, q)


def test_two_km_sparse_map_is_searched_exactly(lib):
    """Wider than 1024 level-0 cells of 0.2 m: the cells are coarser, the search stays exact."""
    cloud = _cloud(300_000, 9, (2000.0, 2000.0, 20.0))
    lm = kd_map(lib)
    lm.set_map_pointcloud(cloud)
    rng = np.random.RandomState(4)
    q = np.concatenate([cloud[rng.randint(0, len(cloud), 5000)] + rng.normal(0, 0.5, (5000, 3)).astype(np.float32),
                        _cloud(5000, 10, (2400.0, 2400.0, 40.0))])
    assert_exact_nn(lm, cloud, q)


def test_one_point_map(lib):
    cloud = np.array([[3.0, -2.0, 0.5]], np.float32)
    lm = kd_map(lib)
    lm.set_map_pointcloud(cloud)
    res = lm.nearest_neighbor_search(_cloud(100, 11), with_normals=False)
    assert np.all(res.neighbor_points == cloud)


def test_float64_cloud_is_rounded(lib):
    cloud = _cloud(10000, 12).astype(np.float64) + 1e-4
    lm = kd_map(lib)
    lm.set_map_pointcloud(cloud)
    assert lm.points().tobytes() == cloud.astype(np.float32).tobytes()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 1e300])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_non_finite_rows_are_refused_before_any_change(lib, bad, dtype):
    if dtype == np.float32 and bad == 1e300:
        pytest.skip("not a float32 value")
    lm = kd_map(lib)
    before = _cloud(1000, 13)
    lm.set_map_pointcloud(before)
    cloud = _cloud(2000, 14).astype(dtype)
    cloud[1234, 1] = bad
    with pytest.raises(AssertionError, match="NaN or infinite"):
        lm.set_map_pointcloud(cloud)
    assert lm.points().tobytes() == before.tobytes()


def test_empty_cloud_leaves_an_empty_map(lib):
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    odo = b200.ICPFrameToModel(dict(algorithm="icp_F2M", max_num_alignments=5), projector=proj)
    odo.init()
    lm = kd_map(lib, ctx=odo.ctx)
    lm.set_map_pointcloud(_cloud(100, 15))
    lm.set_map_pointcloud(np.zeros((0, 3), np.float32))
    assert lm.num_points() == 0
    with pytest.raises(RuntimeError, match="empty"):
        lm.nearest_neighbor_search(_cloud(10, 16))
    with pytest.raises(AssertionError, match="search before any update"):
        odo.register_new_frame_hypotheses(syn.scan(0, 16, 256), np.eye(4, dtype=np.float32)[None])


# ---- the reference's own results --------------------------------------------------------------------------------------
def test_golden_searches(lib, g):
    q = g["pm_queries"]
    for tag in ("32", "64"):
        lm = kd_map(lib)
        lm.set_map_pointcloud(g[f"pm_cloud{tag}"])
        res = lm.nearest_neighbor_search(q, with_normals=False)
        np.testing.assert_allclose(res.neighbor_points, g[f"pm_nb{tag}_off"], atol=2e-5)
        res = lm.nearest_neighbor_search(q)
        np.testing.assert_allclose(res.neighbor_points, g[f"pm_nb{tag}"], atol=2e-5)
        dots = np.abs((res.neighbor_normals * g[f"pm_nrm{tag}"]).sum(-1))
        assert np.mean(dots > 1 - 1e-4) > 0.99, tag


def test_golden_errors(lib, g):
    import torch
    lm = kd_map(lib)
    lm.set_map_pointcloud(g["pm_cloud32"], normals=np.zeros_like(g["pm_cloud32"]))
    res = lm.nearest_neighbor_search(g["pm_queries"], with_normals=False)
    np.testing.assert_allclose(res.neighbor_points, g["pm_nb_given_off"], atol=2e-5)
    kind, msg = g["pm_err_given_normals"]
    with pytest.raises(IndexError, match=msg):
        lm.nearest_neighbor_search(g["pm_queries"])
    assert kind == "IndexError"
    # typeguard 2, which the reference pins, raises TypeError (the installed typeguard's TypeCheckError in the golden)
    with pytest.raises(TypeError, match=str(g["pm_err_torch_cloud"][1])):
        lm.set_map_pointcloud(torch.from_numpy(g["pm_cloud32"]))
    lm.set_map_pointcloud(g["pm_cloud32"][:500])
    with pytest.raises(IndexError, match=str(g["pm_err_last_after_set"][1])):
        lm.get_last_frame()
    lm.update(np.eye(4, dtype=np.float32))   # a move without a frame: still none held
    with pytest.raises(IndexError):
        lm.get_last_frame()
    lm.update(np.eye(4, dtype=np.float32), new_pc_data=g["pm_queries"][:10])
    lm.nearest_neighbor_search(g["pm_queries"])   # the update rebuilt the normal cache


def test_golden_eviction_of_prior_rows(lib, g):
    lm = kd_map(lib, size=3)
    lm.set_map_pointcloud(g["pm_ev_prior"])
    for k in range(6):
        lm.update(g[f"pm_ev_rel_{k}"], new_pc_data=g[f"pm_ev_pts_{k}"])
        ref = g[f"pm_ev_map_{k}"]
        mine = lm.points()
        assert mine.shape == ref.shape, k
        np.testing.assert_allclose(mine, ref, atol=5e-5)
        assert lm.frame_counts() == list(g[f"pm_ev_counts_{k}"]), k
        last = lm.get_last_frame().numpy()
        assert last.shape == g[f"pm_ev_last_{k}"].shape, k
        np.testing.assert_allclose(last, g[f"pm_ev_last_{k}"], atol=5e-5)


def test_golden_projective_last_frame(lib, g):
    import pylidar_slam_b200 as b200
    H, W = g["pm_proj_v1"].shape[1:]
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    pm = b200.ProjectiveLocalMap(b200.ProjectiveLocalMapConfig(local_map_size=3), projector=proj)
    pm.init()
    with pytest.raises(TypeError, match=str(g["pm_err_proj_empty"][1])):
        pm.get_last_frame()
    pm.update(np.eye(4, dtype=np.float32), new_vertex_map=g["pm_proj_v0"][None])
    pm.update(g["pm_proj_rel"], new_vertex_map=g["pm_proj_v1"][None])
    assert pm.get_last_frame().numpy().tobytes() == g["pm_proj_last"].tobytes()


def _odometry(max_iters=12, threshold=1e-4, size=20):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=max_iters, threshold_delta_pose=threshold,
               local_map=dict(type="kdtree_local_map", local_map_size=size),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def test_golden_registration_on_a_set_map(lib, g):
    odo = _odometry()
    kd_map(lib, ctx=odo.ctx).set_map_pointcloud(g["pm_cloud32"])
    params, T, losses, iters = odo.register_new_frame_hypotheses(g["pm_reg_scan"], g["pm_reg_T0"])
    for b in range(len(g["pm_reg_T0"])):
        np.testing.assert_allclose(T[b], g["pm_reg_T"][b], atol=2e-3)
        assert abs(int(iters[b]) - int(g["pm_reg_iters"][b])) <= 1
        p1, T1, l1 = odo.register_new_frame(g["pm_reg_scan"], g["pm_reg_T0"][b])
        assert T1.tobytes() == T[b].tobytes() and p1.tobytes() == params[b].tobytes() and l1 == losses[b]


# ---- B hypotheses against B single calls ----------------------------------------------------------------------------
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
    cold = np.ascontiguousarray(np.concatenate([warm, fill]))
    return dict(warm=warm, cold=cold)


def _hypotheses(B, cloud, seed):
    """The scan is map points (hypothesis 0 starts exactly on them: the tiny-residual guard), hypothesis 1 starts 40 m
    and 120 degrees away (diverges), the others within a few metres and degrees."""
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T0s = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(1, B):
        far = b == 1
        T0s[b, :3, :3] = Rotation.from_euler("z", 120.0 if far else rng.uniform(-8, 8), degrees=True).as_matrix()
        T0s[b, :3, 3] = [40.0, -30.0, 2.0] if far else rng.uniform(-2.0, 2.0, 3) * [1, 1, 0.1]
    return T0s


def _single(lib, ctx, scan, T0, M):
    T, p, losses, iters = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(M, np.float32), C.c_int(0)
    st = lib.load().pls_register_frame(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(T0), lib.ptr(T), lib.ptr(p),
                                       lib.ptr(losses), C.byref(iters))
    return st, T, p, losses, iters.value


def _readback(lib, ctx, nq):
    out = dict(idx=np.empty(nq, np.int64), nb=np.empty((nq, 3), np.float32), nrm=np.empty((nq, 3), np.float32),
               state=np.empty((nq, 4), np.float32), sums=np.empty(30, np.float64))
    st = lib.load().pls_kdmap_last_correspondences(ctx.handle, nq, lib.ptr(out["idx"]), lib.ptr(out["nb"]),
                                                    lib.ptr(out["nrm"]), lib.ptr(out["state"]), lib.ptr(out["sums"]))
    assert st == lib.PLS_OK
    return out


@pytest.mark.parametrize("which", ["warm", "cold"])
@pytest.mark.parametrize("B", [1, 2, 63, 64, 65])
def test_hypotheses_bit_identical_to_single_calls(lib, maps, which, B):
    cloud = maps[which]
    odo = _odometry(max_iters=15)
    kd_map(lib, ctx=odo.ctx).set_map_pointcloud(cloud)
    rng = np.random.RandomState(B)
    scan = np.ascontiguousarray(maps["warm"][rng.choice(len(maps["warm"]), 30000, replace=False)])
    scan[::97] = np.nan   # NaN rows are dropped from the queries, as register_frame drops them
    T0s = _hypotheses(B, cloud, B)
    M = 15
    params, T, losses, iters = odo.register_new_frame_hypotheses(scan, T0s)
    status = odo.last_hypotheses_status
    hyp_last = _readback(lib, odo.ctx, int(np.sum(~np.isnan(scan).any(1))))
    seen = set()
    for b in range(B):
        st, T1, p1, l1, it1 = _single(lib, odo.ctx, scan, T0s[b], M)
        assert (st == lib.PLS_E_SINGULAR) == (status[b] == lib.PLS_E_SINGULAR), b
        assert T1.tobytes() == T[b].reshape(16).tobytes(), b
        assert p1.tobytes() == params[b].tobytes(), b
        assert it1 == iters[b], b
        assert np.asarray(l1[:it1], np.float32).tobytes() == np.asarray(losses[b], np.float32).tobytes(), b
        seen.add(int(status[b]))
    single_last = _readback(lib, odo.ctx, int(np.sum(~np.isnan(scan).any(1))))
    for k in hyp_last:
        assert hyp_last[k].tobytes() == single_last[k].tobytes(), k
    assert status[0] == lib.PLS_W_TINY_RESIDUAL
    if B > 1:
        assert iters[1] == M or status[1] == lib.PLS_E_SINGULAR   # the far hypothesis does not converge
        assert np.linalg.norm(T[1][:3, 3]) > 5.0
    if B > 2:
        assert lib.PLS_OK in seen or lib.PLS_W_TINY_RESIDUAL in seen


def test_later_iteration_launches_do_not_grow_with_B(lib, maps):
    """threshold_delta_pose = 0: every hypothesis runs max_num_alignments iterations.  One more iteration is the four
    launches verify / 1-NN / normals / residual on a map above KD_COLD_MAP_POINTS, whatever B."""
    scan = np.ascontiguousarray(maps["warm"][::20])
    counts = {}
    for M in (3, 4):
        odo = _odometry(max_iters=M, threshold=0.0)
        kd_map(lib, ctx=odo.ctx).set_map_pointcloud(maps["cold"])
        for B in (1, 8, 64):
            before = odo.ctx.launch_count()
            odo.register_new_frame_hypotheses(scan, _hypotheses(B, maps["cold"], 5))
            counts[B, M] = odo.ctx.launch_count() - before
    for B in (1, 8, 64):
        assert counts[B, 4] - counts[B, 3] == 4, counts
        assert counts[B, 3] == counts[1, 3], counts
