"""Many scans registered against one prior map in one call: pls_register_scans and ICPFrameToModel.register_new_frames.

  * every registration is bit-identical to a pls_register_frame call with its scan and initial estimate, on a
    cfg2-sized map (the refine kernel) and on one above KD_COLD_MAP_POINTS (four launches), with 10 and 64 normal
    neighbours (the wide normals kernel), for S = 1, 2, 63, 64 and 65 scans and up to 130 registrations (chunks), with
    scans of 1, 2047, 2048, 2049 and 131 072 rows, a scan with NaN rows and scans listed under several estimates;
  * S = 1 is pls_register_hypotheses, bit for bit;
  * the map is not touched, the context ends as if pls_register_frame had run the last registration last, and every
    refusal leaves it unchanged;
  * the launches of one more ICP iteration do not grow with B.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

COLD_MAP_POINTS = 2_000_000  # kdmap.cu: KD_COLD_MAP_POINTS


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


def _odometry(max_iters=12, threshold=1e-4, k=10):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=max_iters, threshold_delta_pose=threshold, data_key="numpy_pc",
               local_map=dict(type="kdtree_local_map", local_map_size=20, num_neighbors_normals=k),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def _set_map(odo, cloud):
    import pylidar_slam_b200 as b200
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20), ctx=odo.ctx)
    lm.set_map_pointcloud(cloud)
    return lm


def _scans(warm, sizes, seed):
    """Scans of map points (a scan at the identity starts exactly on the map: the tiny-residual guard); size < 0: that
    many rows with every 97th row NaN."""
    rng = np.random.RandomState(seed)
    out = []
    for n in sizes:
        s = np.ascontiguousarray(warm[rng.choice(len(warm), abs(n), replace=abs(n) > len(warm))])
        if n < 0:
            s[::97] = np.nan
        out.append(s)
    return out


def _estimates(B, seed):
    """Registration 0 starts at the identity (on the map), registration 1 40 m and 120 degrees away (runs every
    iteration or goes singular), the others within a few metres and degrees."""
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T0s = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(1, B):
        far = b == 1
        T0s[b, :3, :3] = Rotation.from_euler("z", 120.0 if far else rng.uniform(-8, 8), degrees=True).as_matrix()
        T0s[b, :3, 3] = [40.0, -30.0, 2.0] if far else rng.uniform(-2.0, 2.0, 3) * [1, 1, 0.1]
    return T0s


EDGE_SIZES = [1, 2047, 2048, 2049, 131072, -30000]


def _case(case, warm):
    """(scans, scan_of or None, B) of one test set."""
    rng = np.random.RandomState(len(case))
    if case == "S1":
        return _scans(warm, [-30000], 1), np.zeros(3, np.int32), 3
    if case == "S2":
        return _scans(warm, [2047, 2049], 2), np.array([0, 1, 1, 0], np.int32), 4
    S = {"S63": 63, "S64": 64, "S65": 65, "B130": 65}[case]
    sizes = EDGE_SIZES + list(rng.randint(200, 6000, S - len(EDGE_SIZES)))
    scans = _scans(warm, sizes, S)
    if case == "S63" or case == "S65":
        return scans, None, S
    if case == "S64":   # a permutation with one scan listed twice (and one left out)
        of = rng.permutation(S).astype(np.int32)
        of[7] = of[3]
        return scans, of, S
    return scans, np.concatenate([np.arange(S), rng.randint(0, S, 130 - S)]).astype(np.int32), 130


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
    icp = np.empty(30, np.float64)
    it = C.c_int(0)
    assert lib.load().pls_last_icp_sums(ctx.handle, lib.ptr(icp), C.byref(it)) == lib.PLS_OK
    out["icp_sums"], out["icp_iters"] = icp, np.array([it.value])
    return out


def _valid(scan):
    return int(np.sum(~np.isnan(scan).any(1)))


def _map_bytes(lm):
    return lm.points().tobytes(), list(lm.frame_counts())


@pytest.mark.parametrize("case", ["S1", "S2", "S63", "S64", "S65", "B130"])
@pytest.mark.parametrize("k", [10, 64])
@pytest.mark.parametrize("which", ["warm", "cold"])
def test_registrations_bit_identical_to_single_calls(lib, maps, which, k, case):
    M = 15
    odo = _odometry(max_iters=M, k=k)
    lm = _set_map(odo, maps[which])
    scans, scan_of, B = _case(case, maps["warm"])
    T0s = _estimates(B, len(scans))
    before = _map_bytes(lm)
    params, T, losses, iters = odo.register_new_frames(scans, T0s, scan_of)
    status = odo.last_registrations_status
    of = np.arange(B) if scan_of is None else scan_of
    last = _readback(lib, odo.ctx, _valid(scans[of[-1]]))
    assert _map_bytes(lm) == before
    seen = set()
    for b in range(B):
        st, T1, p1, l1, it1 = _single(lib, odo.ctx, scans[of[b]], T0s[b], M)
        assert (st == lib.PLS_E_SINGULAR) == (status[b] == lib.PLS_E_SINGULAR), b
        assert T1.tobytes() == T[b].reshape(16).tobytes(), b
        assert p1.tobytes() == params[b].tobytes(), b
        assert it1 == iters[b], b
        assert np.asarray(l1[:it1], np.float32).tobytes() == np.asarray(losses[b], np.float32).tobytes(), b
        seen.add(int(status[b]))
    single_last = _readback(lib, odo.ctx, _valid(scans[of[-1]]))
    for key in last:
        assert last[key].tobytes() == single_last[key].tobytes(), key
    assert _map_bytes(lm) == before
    assert status[0] == lib.PLS_W_TINY_RESIDUAL or scans[of[0]].shape[0] == 1
    # the far estimate does not come back to the map
    assert iters[1] == M or status[1] == lib.PLS_E_SINGULAR or np.linalg.norm(T[1][:3, 3]) > 5.0
    assert lib.PLS_OK in seen or lib.PLS_W_TINY_RESIDUAL in seen


@pytest.mark.parametrize("which", ["warm", "cold"])
def test_one_scan_is_register_hypotheses(lib, maps, which):
    odo = _odometry(max_iters=15)
    _set_map(odo, maps[which])
    scan = _scans(maps["warm"], [-30000], 7)[0]
    T0s = _estimates(65, 7)
    a = odo.register_new_frames([scan], T0s, np.zeros(65, np.int32))
    status_a = odo.last_registrations_status.copy()
    last_a = _readback(lib, odo.ctx, _valid(scan))
    b = odo.register_new_frame_hypotheses(scan, T0s)
    last_b = _readback(lib, odo.ctx, _valid(scan))
    for x, y in zip(a[:2] + a[3:], b[:2] + b[3:]):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    assert [np.asarray(l, np.float32).tobytes() for l in a[2]] == [np.asarray(l, np.float32).tobytes() for l in b[2]]
    assert status_a.tobytes() == odo.last_hypotheses_status.tobytes()
    for key in last_a:
        assert last_a[key].tobytes() == last_b[key].tobytes(), key


def test_later_frames_follow_the_last_registration(lib, maps):
    """After the call the context is a twin's that ran pls_register_frame on the last registration: the same map and
    search state, and the next three odometry frames give the same bits."""
    from pylidar_slam_b200 import synthetic as syn
    scans = _scans(maps["warm"], [4000, -9000, 2500], 11)
    T0s = _estimates(5, 11)
    of = np.array([2, 0, 1, 1, 1], np.int32)
    a, b = _odometry(), _odometry()
    lma, lmb = _set_map(a, maps["warm"]), _set_map(b, maps["warm"])
    a.register_new_frames(scans, T0s, of)
    b.register_new_frame(scans[1], T0s[-1])
    assert _map_bytes(lma) == _map_bytes(lmb)
    ra, rb = _readback(lib, a.ctx, _valid(scans[1])), _readback(lib, b.ctx, _valid(scans[1]))
    for key in ra:
        assert ra[key].tobytes() == rb[key].tobytes(), key
    for k in range(3):
        pc = np.ascontiguousarray(syn.scan(k, 16, 256), np.float32)
        for o in (a, b):
            o.process_next_frame({"numpy_pc": pc.copy()})
    assert np.asarray(a.get_relative_poses()).tobytes() == np.asarray(b.get_relative_poses()).tobytes()
    assert _map_bytes(lma) == _map_bytes(lmb)


def _call(lib, ctx, scans, n, S, scan_of, T0s, B):
    M = 16
    addr = np.array([0 if s is None else lib.ptr(s) for s in scans] or [0], np.uint64)
    out = [np.zeros(max(B, 1) * w, t) for w, t in ((16, np.float32), (6, np.float32), (M, np.float32), (1, np.int32),
                                                   (1, np.int32))]
    return lib.load().pls_register_scans(ctx.handle, lib.ptr(addr), lib.ptr(np.asarray(n, np.int64)), S,
                                         None if scan_of is None else lib.ptr(np.asarray(scan_of, np.int32)),
                                         None if T0s is None else lib.ptr(T0s), B, *(lib.ptr(o) for o in out))


def test_refusals_leave_the_context_unchanged(lib, maps):
    import pylidar_slam_b200 as b200
    odo = _odometry(max_iters=4)
    lm = _set_map(odo, maps["warm"])
    scans = _scans(maps["warm"], [3000, 2000], 13)
    odo.register_new_frames(scans, _estimates(2, 13))
    before = _map_bytes(lm), _readback(lib, odo.ctx, _valid(scans[1]))
    T0s = _estimates(3, 13)
    bad = [
        (scans, [3000, 2000], 0, None, T0s[:0], 0),       # S = 0, B = 0
        (scans, [3000, 2000], 2, [0, 1], T0s[:2], 0),     # B = 0
        (scans, [3000, 2000], -1, [0, 0], T0s[:2], 2),    # S < 0
        (scans, [3000, 0], 2, [0, 1], T0s[:2], 2),        # n[1] = 0
        (scans, [-5, 2000], 2, [0, 1], T0s[:2], 2),       # n[0] < 0
        (scans, [3000, 2000], 2, [0, 2], T0s[:2], 2),     # scan_of out of range
        (scans, [3000, 2000], 2, [-1, 0], T0s[:2], 2),
        (scans, [3000, 2000], 2, None, T0s, 3),           # no scan_of, B != S
        ([scans[0], None], [3000, 2000], 2, None, T0s[:2], 2),
        (scans, [3000, 2000], 2, None, None, 2),
    ]
    for args in bad:
        assert _call(lib, odo.ctx, *args) == lib.PLS_E_INVALID, args[2:4]
        after = _map_bytes(lm), _readback(lib, odo.ctx, _valid(scans[1]))
        assert after[0] == before[0]
        for key in before[1]:
            assert after[1][key].tobytes() == before[1][key].tobytes(), key
    # a map that has had no update, gn_max_iters != 1, a projective map
    fresh = _odometry()
    assert _call(lib, fresh.ctx, scans, [3000, 2000], 2, None, T0s[:2], 2) == lib.PLS_E_INVALID
    assert "before any update" in lib.load().pls_last_error(fresh.ctx.handle).decode()
    gn2 = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20, gn_max_iters=2)
    gn2.call("pls_kdmap_set_points", lib.ptr(maps["warm"]), 0, maps["warm"].shape[0])
    assert _call(lib, gn2, scans, [3000, 2000], 2, None, T0s[:2], 2) == lib.PLS_E_INVALID
    assert "max_iters" in lib.load().pls_last_error(gn2.handle).decode()
    proj = b200.SphericalProjector(height=16, width=256, up_fov=3.0, down_fov=-24.0)
    po = b200.ICPFrameToModel(dict(algorithm="icp_F2M", max_num_alignments=5, data_key="numpy_pc",
                                   local_map=dict(type="projective_local_map")), projector=proj)
    po.init()
    assert _call(lib, po.ctx, scans, [3000, 2000], 2, None, T0s[:2], 2) == lib.PLS_E_INVALID
    assert "kd-tree" in lib.load().pls_last_error(po.ctx.handle).decode()


def test_later_iteration_launches_do_not_grow_with_B(lib, maps):
    """threshold_delta_pose = 0: every registration runs max_num_alignments iterations.  One more iteration is the four
    launches verify / 1-NN / normals / residual on a map above KD_COLD_MAP_POINTS, whatever B; the packing of the S
    scans is one launch."""
    counts = {}
    for M in (3, 4):
        odo = _odometry(max_iters=M, threshold=0.0)
        _set_map(odo, maps["cold"])
        for B in (1, 8, 64):
            scans = _scans(maps["warm"], list(np.random.RandomState(B).randint(1000, 4000, B)), B)
            before = odo.ctx.launch_count()
            odo.register_new_frames(scans, _estimates(B, 5))
            counts[B, M] = odo.ctx.launch_count() - before
    for B in (1, 8, 64):
        assert counts[B, 4] - counts[B, 3] == 4, counts
        assert counts[B, 3] == counts[1, 3], counts


def test_device_scans_and_given_normals(lib, maps):
    """Device tensors are read in place and give the bits of host arrays; a map set with normals refuses to register,
    as register_new_frame does."""
    import torch
    odo = _odometry(max_iters=8)
    lm = _set_map(odo, maps["warm"])
    scans = _scans(maps["warm"], [5000, -7000], 17)
    T0s = _estimates(4, 17)
    of = np.array([1, 0, 1, 0], np.int32)
    host = odo.register_new_frames(scans, T0s, of)
    dev = odo.register_new_frames([torch.from_numpy(s).cuda() for s in scans], torch.from_numpy(T0s),
                                  torch.from_numpy(of))
    for x, y in zip(host[:2] + host[3:], dev[:2] + dev[3:]):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    assert host[2] == dev[2]
    lm.set_map_pointcloud(maps["warm"], normals=np.zeros_like(maps["warm"]))
    with pytest.raises(IndexError):
        odo.register_new_frames(scans, T0s, of)


def test_golden_registrations_of_three_scans(lib):
    """The reference's register_new_frame on a set map (tests/golden/register_scans.npz): three scans of different sizes,
    two initial estimates each, within the tolerances of test_prior_map_gpu's registration on a set map."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "register_scans.npz"))
    odo = _odometry(max_iters=12)
    _set_map(odo, g["rs_cloud"])
    scans = [g[f"rs_scan_{s}"] for s in range(3)]
    params, T, losses, iters = odo.register_new_frames(scans, g["rs_T0"], g["rs_scan_of"])
    for b in range(len(g["rs_T0"])):
        np.testing.assert_allclose(T[b], g["rs_T"][b], atol=2e-3)
        assert abs(int(iters[b]) - int(g["rs_iters"][b])) <= 1
