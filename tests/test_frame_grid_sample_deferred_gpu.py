"""pls_process_frame_grid_sample, whose frames after the first read the sample count on the device and are enqueued
without a host wait, against pls_grid_sample + pls_process_frame on the same clouds, bit for bit: pose, params,
has-pose, the 12 info values, the return code and the sums of the last ICP iteration, after every frame.

Covered: the cfg2 stream in both point layouts; sample counts whose residual grid is 1, 2, 1 055, 1 056 and (capped)
1 057 blocks, with more raw rows than samples so that the launch is wider than the grid the kernels use; a frame whose
voxel hashes overflow the compact sort keys (run again on the raw keys), followed by more frames on the same context;
and a frame that needs a second round of ICP launches.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VOXEL = 0.3


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def make_ctx(lib, H, W):
    return lib.Context(local_map_type=lib.MAP_KDTREE, height=H, width=W, local_map_size=20,
                       scheme=lib.SCHEMES["geman_mcclure"], sigma=0.3, max_num_alignments=10, gn_max_iters=1)


def outputs():
    return np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)


def sums_of(lib, ctx):
    sums, iters = np.zeros(30), C.c_int(0)
    st = lib.load().pls_last_icp_sums(ctx.handle, lib.ptr(sums), C.byref(iters))
    return sums if st == 0 else None


def fused(lib, ctx, pts, layout, init):
    """One pls_process_frame_grid_sample call on the raw rows (device-resident)."""
    import torch
    d = torch.from_numpy(pts).cuda()
    torch.cuda.synchronize()
    pose, params, info, has = outputs()
    rc = lib.load().pls_process_frame_grid_sample(ctx.handle, d.data_ptr(), pts.shape[0], VOXEL, layout, lib.ptr(init),
                                                  lib.ptr(pose), lib.ptr(params), C.byref(has), lib.ptr(info))
    return rc, dict(pose=pose, params=params, has=np.int32(has.value), info=info, sums=sums_of(lib, ctx))


def staged(lib, ctx, pts, layout, init):
    """pls_grid_sample, then pls_process_frame on its samples (same layout), reporting the sample count as info[4]."""
    import torch
    n = pts.shape[0]
    out, idx, count = np.zeros((n, 3), np.float32), np.zeros(n, np.int64), C.c_int64(0)
    assert lib.load().pls_grid_sample(ctx.handle, lib.ptr(pts), 0, n, VOXEL, lib.ptr(out), lib.ptr(idx), C.byref(count)) == 0
    S = count.value
    samples = torch.from_numpy(np.ascontiguousarray(out[:S])).cuda()
    torch.cuda.synchronize()
    pose, params, info, has = outputs()
    rc = lib.load().pls_process_frame(ctx.handle, samples.data_ptr(), layout | lib.PTR_DEVICE, S, lib.ptr(init),
                                      lib.ptr(pose), lib.ptr(params), C.byref(has), lib.ptr(info))
    if rc == 0:
        info[4] = S
    return rc, dict(pose=pose, params=params, has=np.int32(has.value), info=info, sums=sums_of(lib, ctx))


def run_pair(lib, H, W, frames, layout, chain_poses=True):
    """The same frames on two fresh contexts, one per path; returns the per-frame (return code, info) of the fused path."""
    a, b = make_ctx(lib, H, W), make_ctx(lib, H, W)
    init_a = init_b = None
    infos = []
    for k, pts in enumerate(frames):
        pts = np.ascontiguousarray(pts, np.float32)
        rc_a, oa = fused(lib, a, pts, layout, init_a)
        rc_b, ob = staged(lib, b, pts, layout, init_b)
        assert rc_a == rc_b, (k, rc_a, rc_b, a.err if hasattr(a, "err") else None)
        for key in oa:
            assert np.asarray(oa[key]).tobytes() == np.asarray(ob[key]).tobytes(), (k, key, oa[key], ob[key])
        infos.append((rc_a, oa["info"].copy()))
        if chain_poses and oa["has"]:
            init_a, init_b = oa["pose"].reshape(4, 4).copy(), ob["pose"].reshape(4, 4).copy()
    return infos


@pytest.mark.parametrize("layout_name", ["INPUT_TENSOR", "INPUT_NDARRAY"])
def test_cfg2_stream(lib, layout_name):
    from pylidar_slam_b200 import synthetic as syn
    frames = [syn.scan(k, 64, 2048) for k in range(6)]
    infos = run_pair(lib, 64, 2048, frames, getattr(lib, layout_name))
    assert all(rc == 0 and i[0] >= 1 for rc, i in infos[1:])  # every frame after the first ran ICP


def room(S, extra, seed):
    """S points in S distinct voxels on a floor and two walls (voxel centres, jittered inside their voxel within the
    surface), then `extra` rows repeating voxels already taken: exactly S samples out of S + extra rows."""
    rng = np.random.RandomState(0)
    side = int(np.ceil(np.sqrt(S / 3.0))) + 2
    u, v = np.meshgrid(np.arange(-side // 2, side - side // 2), np.arange(side), indexing="ij")
    u, v = u.ravel(), v.ravel()
    # far enough out for the sensor's -24 degree lower field of view to see the floor (frame 0 builds the map from the
    # vertex map)
    floor = np.stack([u, v + 20, np.full_like(u, -6)], 1)
    wall_x = np.stack([np.full_like(u, side // 2 + 20), u + 20, v - 5], 1)
    wall_y = np.stack([u, np.full_like(u, side + 30), v - 5], 1)
    cells = np.concatenate([floor, wall_x, wall_y])
    cells = cells[rng.permutation(len(cells))[:S]]
    assert len(np.unique(cells, axis=0)) == S
    r = np.random.RandomState(seed)
    jitter = r.uniform(-0.12, 0.12, cells.shape)
    on_floor = cells[:, 2] == -6
    on_wx = cells[:, 0] == side // 2 + 20
    on_wy = cells[:, 1] == side + 30
    jitter[on_floor, 2] = 0.0
    jitter[on_wx & ~on_floor, 0] = 0.0
    jitter[on_wy & ~on_floor & ~on_wx, 1] = 0.0
    pts = (cells + jitter) * VOXEL
    rep = pts[r.randint(0, S, extra)] + r.uniform(-0.02, 0.02, (extra, 3)) * np.array([1, 1, 0])
    return np.concatenate([pts, rep]).astype(np.float32)


@pytest.mark.parametrize("S", [250, 500, 1055 * 256, 1056 * 256, 1056 * 256 + 1])
def test_residual_grid_edges(lib, S):
    """NDARRAY layout: the queries are the valid samples, so the residual grid is ceil(S / 256) blocks, capped at
    8 * 132; the raw rows (S + 3000) size the launch."""
    frames = [room(S, 3000, seed) for seed in range(3)]
    infos = run_pair(lib, 64, 2048, frames, lib.INPUT_NDARRAY)
    # (both paths return the same code; a frame that ends in an error reports no info)
    assert all(int(i[4]) == S for rc, i in infos if rc == 0)


def test_overflowing_hashes_then_more_frames(lib):
    """A frame with one row far enough out for its voxel hash to leave the 40-bit sort keys: the fused call finds the
    overflow only with the frame's result and runs the frame again on the raw keys.  The frames after it continue on
    the same context."""
    from pylidar_slam_b200 import synthetic as syn
    frames = []
    for k in range(5):
        pts = syn.scan(k, 64, 2048)
        if k == 2:
            pts = np.concatenate([pts, np.array([[4.0e5, 1.0, 1.0]], np.float32)])
        frames.append(pts)
    infos = run_pair(lib, 64, 2048, frames, lib.INPUT_TENSOR)
    assert infos[2][0] == 0 and infos[2][1][0] >= 1


def test_second_round_of_icp_launches(lib):
    """Consecutive frames, each from the identity, then a frame six scans further on: it needs more iterations than
    the previous frame's count + 1 enqueued up front."""
    from pylidar_slam_b200 import synthetic as syn
    frames = [syn.scan(k, 64, 2048) for k in (0, 1, 2, 3)] + [syn.scan(9, 64, 2048)]
    a, b = make_ctx(lib, 64, 2048), make_ctx(lib, 64, 2048)
    iters = []
    for k, pts in enumerate(frames):
        init = None
        rc_a, oa = fused(lib, a, pts, lib.INPUT_TENSOR, init)
        rc_b, ob = staged(lib, b, pts, lib.INPUT_TENSOR, init)
        assert rc_a == rc_b == 0, (k, rc_a, rc_b)
        for key in oa:
            assert np.asarray(oa[key]).tobytes() == np.asarray(ob[key]).tobytes(), (k, key)
        iters.append(int(oa["info"][0]))
    assert iters[-1] > iters[-2] + 1, iters
