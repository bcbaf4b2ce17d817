"""The kd map's normals from more than 31 neighbours (32 <= k <= 255: warp_knn_wide, warp_second_moments_wide and the
kernels that call them), against the reference's own float32 moments and results.

  * lists: pls_kdmap_knn at map points and off-map probes of every scene of oracle/kd_normals_scenes.py equals
    oracle knn_lists (checked as tests/test_kd_normals_knn_gpu.py checks k <= 31), with the PLS_KD_STATS path counters;
  * normals: pls_kdmap_nn_search within tight_normal_bound of the float64 eigenvector of reference_covs;
  * ICP: every iteration of the cfg2 scenario of tests/test_kd_icp_iterations_gpu.py, whose later iterations take the
    four launches at these k; odometry poses and searches against tests/golden/wide_normals.npz;
  * batches: pls_process_frames with k = 10, 40 and 255 in one call and register_new_frame_hypotheses at k = 64 are
    bit-identical to independent calls;
  * maps of at most k + 1 points, and the range [3, 255] at pls_create and pls_kdmap_knn.
"""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import kd_icp_reference as ref_mod
from oracle import kd_normals_scenes as scenes
import test_kd_normals_knn_gpu as narrow
from test_kd_icp_iterations_gpu import _cfg2_runs, _check_runs, _first_matched_late, ref, scene  # noqa: F401
from test_kd_normals_knn_gpu import check_lists, check_normals, lib  # noqa: F401

pytestmark = pytest.mark.gpu

KS = [32, 33, 63, 64, 65, 127, 128, 200, 255]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_normals.npz")
MAP_QUERIES, PROBES = 3000, 1000    # per scene: a sample of the map points and of the off-map probes
_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        m, probes = scenes.build(name)
        rng = np.random.RandomState(len(m))
        sub = np.sort(rng.choice(len(m), min(len(m), MAP_QUERIES), replace=False))
        _SCENES[name] = (m, probes[:PROBES], sub, ref_mod.kernel_sort_positions(m), cKDTree(m.astype(np.float64)))
    return _SCENES[name]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", scenes.SCENES)
def test_wide_lists_normals_and_paths(lib, name, k):  # noqa: F811
    m, probes, sub, positions, tree = _scene(name)
    tag = f"{name} k={k}"
    ctx = narrow._context(lib, k)
    narrow._insert(lib, ctx, m)
    q = np.ascontiguousarray(np.concatenate([m[sub], probes]))
    s0 = narrow._stats(lib, ctx)
    idx, d2, pos = narrow._knn(lib, ctx, q, k)
    ds = narrow._stats(lib, ctx) - s0
    r_idx, amb = check_lists(m, positions, tree, q, k, idx, d2, pos, tag)
    # level 0 restated against the counters of the same search: every wide list streams its candidates, so a query
    # exact at level 0 scans exactly its block
    K = k + 1
    kth = np.where(idx[:, K - 1] >= 0, d2[:, K - 1], np.float32(np.inf))
    total, exact = ref_mod.level0_paths(m, q, k, kth)
    assert ds[4] == len(q), (tag, ds[4])
    assert ds[5] == exact.sum() and ds[6] == len(q) - exact.sum(), (tag, ds[5], int(exact.sum()))
    assert ds[7] >= total.sum() and (ds[7] == total.sum()) == exact.all(), (tag, ds[7], int(total.sum()))
    if exact.any():
        a = narrow._stats(lib, ctx)
        narrow._knn(lib, ctx, np.ascontiguousarray(q[exact]), k)
        d = narrow._stats(lib, ctx) - a
        assert d[4] == d[5] == exact.sum() and d[7] == total[exact].sum(), (tag, d[4:8])
    # normals kd_normals_wide_kernel computes at the sampled map points, over the reference's and the GPU's lists
    pts = np.ascontiguousarray(m[sub])
    nb, nrm = np.empty_like(pts), np.empty_like(pts)
    ctx.call("pls_kdmap_nn_search", lib.ptr(pts), pts.shape[0], lib.ptr(nb), lib.ptr(nrm), None)
    ctx.close()
    assert np.array_equal(nb, pts), tag
    n = len(sub)
    sure = ~amb[:n]
    check_normals(m, sub[sure], r_idx[:n][sure], k, nrm[sure], tag + " reference lists")
    check_normals(m, sub, idx[:n], k, nrm, tag + " own lists")
    print(tag, dict(exact0=int(exact.sum()), coarser=int((~exact).sum()), ambiguous=int(amb.sum())))


@pytest.mark.parametrize("k", [32, 127, 255])
def test_maps_of_at_most_k_plus_one_points(lib, k):  # noqa: F811
    """M = 1, 2, k and k + 1: with M <= k the moments are those of the M - 1 others divided by k, as for k <= 31."""
    for M in sorted({1, 2, k, k + 1}):
        m = scenes.tiny(M)
        probes = np.random.RandomState(M).uniform(-2, 2, (64, 3)).astype(np.float32)
        p = narrow.run_scene(lib, m, probes, ref_mod.kernel_sort_positions(m), cKDTree(m.astype(np.float64)), k,
                             tag=f"M={M} k={k}")
        assert (p["found_lt_K"] > 0) == (M < k + 1)


@pytest.mark.parametrize("k", [32, 127, 255])
def test_cfg2_six_iterations_through_the_four_launches(lib, ref, scene, k):  # noqa: F811
    """Every iteration's matches, normals and sums against the float64 reference.  The later iterations verify, search
    the unproven queries and compute the new normals with kd_normals_wide_kernel."""
    runs = _cfg2_runs(lib, scene, k)
    matched = _check_runs(lib, ref, scene["m"], scene["tree"], scene["q"], scene["T0"], runs, tag=f"cfg2 k={k}", k=k)
    assert len(_first_matched_late(matched)) >= 100
    assert not np.array_equal(runs[0]["nrm"], _cfg2_runs(lib, scene, 31)[0]["nrm"])


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("k", [32, 64, 255])
def test_golden_searches_and_poses(golden, k):
    import pylidar_slam_b200 as b200
    from oracle import icp_oracle as orc
    from pylidar_slam_b200 import synthetic as syn
    g = golden
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=1, num_neighbors_normals=k))
    lm.init()
    lm.set_map_pointcloud(g["wn_map"])
    res = lm.nearest_neighbor_search(g["wn_queries"])
    lm.ctx.close()
    np.testing.assert_allclose(res.neighbor_points, g[f"wn_nb_{k}"], atol=2e-5)
    dots = np.abs((res.neighbor_normals * g[f"wn_nrm_{k}"]).sum(-1))
    assert np.mean(dots > 1 - 1e-4) > 0.99, k
    # the generator's odometry (make_golden_wide_normals.stream_poses) on the GPU
    H, W = 32, 512
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=4, num_neighbors_normals=k),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                              max_iters=1)),
        max_num_alignments=8, data_key="numpy_pc")
    algo = b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0")
    algo.init()
    want = g[f"wn_pose_{k}"]
    for f in range(want.shape[0]):
        s, _ = orc.grid_sample(syn.scan(f, H, W), 0.4)
        algo.process_next_frame({"numpy_pc": np.ascontiguousarray(s, np.float32)})
    got = np.asarray(algo.get_relative_poses(), np.float64)
    for f in range(1, want.shape[0]):
        Ta, Tb = got[f], want[f].astype(np.float64)
        dt = np.linalg.norm(Ta[:3, 3] - Tb[:3, 3]) / max(np.linalg.norm(Tb[:3, 3]), 1e-12)
        dR = Tb[:3, :3].T @ Ta[:3, :3]
        ang = np.linalg.norm(0.5 * np.array([dR[2, 1] - dR[1, 2], dR[0, 2] - dR[2, 0], dR[1, 0] - dR[0, 1]]))
        assert dt <= 1e-4 and ang <= 1e-5, (k, f, dt, ang)


def test_batch_with_narrow_and_wide_k(lib):  # noqa: F811
    """k = 10, 40 and 255 in one pls_process_frames call: bit-identical per sequence to independent contexts."""
    import test_multi_sequence_gpu as ms
    ks = (10, 40, 255)
    pair = ms.Pair(lib, 3, per_seq=[dict(num_neighbors_normals=k) for k in ks])
    for f in range(8):
        pair.step([ms.Frame(lib, kind, ms.sampled(f)) for kind in ("tensor", "ndarray", "tensor")], tag=f)
        if f == 1:
            nq = int(pair.outs[0]["info"][2])
            nrm = [ms.readback(lib, c, nq)[1]["nrm"] for c in pair.bat]
            assert all(not np.array_equal(nrm[i], nrm[j]) for i, j in ((0, 1), (0, 2), (1, 2)))
    assert max(max(it) for it in pair.iters) >= 2, pair.iters
    pair.finish()


def test_hypotheses_at_k64_bit_identical_to_single_calls(lib):  # noqa: F811
    import pylidar_slam_b200 as b200
    import test_prior_map_gpu as pm
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=12, threshold_delta_pose=1e-4,
               local_map=dict(type="kdtree_local_map", local_map_size=20, num_neighbors_normals=64),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    cloud = pm._scene_cloud()
    b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20, num_neighbors_normals=64),
                        ctx=odo.ctx).set_map_pointcloud(cloud)
    rng = np.random.RandomState(4)
    scan = np.ascontiguousarray(cloud[rng.choice(len(cloud), 30000, replace=False)])
    B = 5
    T0s = pm._hypotheses(B, cloud, 9)
    params, T, losses, iters = odo.register_new_frame_hypotheses(scan, T0s)
    for b in range(B):
        st, T1, p1, l1, it1 = pm._single(lib, odo.ctx, scan, T0s[b], 12)
        assert T1.tobytes() == T[b].reshape(16).tobytes(), b
        assert p1.tobytes() == params[b].tobytes(), b
        assert it1 == iters[b], b
        assert np.asarray(l1[:it1], np.float32).tobytes() == np.asarray(losses[b], np.float32).tobytes(), b
    odo.ctx.close()


@pytest.mark.parametrize("k", [2, 256])
def test_k_out_of_range_is_refused(lib, k):  # noqa: F811
    """pls_create refuses k outside [3, 255] and the Python error names the range; a live context is untouched, and
    its pls_kdmap_knn refuses k above 255."""
    m, _ = scenes.build("clusters")
    ctx = narrow._context(lib, 255)
    narrow._insert(lib, ctx, m)
    q = np.ascontiguousarray(m[:500])
    before = narrow._knn(lib, ctx, q, 255)
    with pytest.raises(AssertionError, match=r"\[3, 255\]"):
        narrow._context(lib, k)
    assert lib.load().pls_kdmap_knn(ctx.handle, lib.ptr(q), q.shape[0], 255 + (k == 256), lib.ptr(np.empty((500, 257),
                                    np.int64)), lib.ptr(np.empty((500, 257), np.float32)), None) == \
        (lib.PLS_E_INVALID if k == 256 else lib.PLS_OK)
    after = narrow._knn(lib, ctx, q, 255)
    ctx.close()
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
