"""The kd map update of pls_process_frame_grid_sample, decided on the device and enqueued behind the frame's ICP launches,
against pls_process_frames at B = 1, whose update the host decides after the frame and enqueues with the next call,
bit for bit after every frame: pose, params, has-pose, the 12 info values, the return code, the sums of the last ICP
iteration (pls_last_icp_sums), the last correspondences (matched map points, their normals and search states), and the
map's points and per-frame counts.  Every frame after the first must have taken the device-decided path: its update
is enqueued by the frame call itself, so reading the map afterwards launches fewer kernels on that context than on the
other one, whose pending update the read enqueues first.

Covered: the cfg2 stream across the map-size eviction boundary (frames 20 and 21 at local_map_size 20, and a 3-frame
map that evicts from frame 3 on -- its raw rows alone would exceed the capacity planned at the first frame, so the
update's launches are sized for that capacity); a frame whose voxel hashes overflow the compact sort keys (run again on
the raw keys), followed by more frames; a frame that is not a key frame; and a frame that needs a second round of ICP
launches.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

H, W, VOXEL = 64, 2048, 0.3


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def make_ctx(lib, local_map_size):
    return lib.Context(local_map_type=lib.MAP_KDTREE, height=H, width=W, local_map_size=local_map_size,
                       scheme=lib.SCHEMES["geman_mcclure"], sigma=0.3, max_num_alignments=10, gn_max_iters=1)


def outputs():
    return np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)


def eager(lib, ctx, d, n, init):
    """One pls_process_frame_grid_sample call on the device-resident raw rows d."""
    pose, params, info, has = outputs()
    rc = lib.load().pls_process_frame_grid_sample(ctx.handle, d.data_ptr(), n, VOXEL, lib.INPUT_TENSOR, lib.ptr(init),
                                                  lib.ptr(pose), lib.ptr(params), C.byref(has), lib.ptr(info))
    return rc, dict(pose=pose, params=params, has=np.int32(has.value), info=info)


def deferred(lib, ctx, d, n, init):
    """One pls_process_frames call with this context alone."""
    handles = (C.c_void_p * 1)(ctx.handle.value)
    data = (C.c_void_p * 1)(d.data_ptr())
    layouts = (C.c_int * 1)(lib.INPUT_TENSOR | lib.PTR_DEVICE)
    ns = (C.c_int64 * 1)(n)
    ip = (C.c_void_p * 1)(None if init is None else lib.ptr(init))
    pose, params, has = np.zeros((1, 16), np.float32), np.zeros((1, 6), np.float32), np.zeros(1, np.int32)
    info, status = np.zeros((1, 12)), np.full(1, -1, np.int32)
    rc = lib.load().pls_process_frames(handles, 1, data, layouts, ns, VOXEL, ip, lib.ptr(pose), lib.ptr(params),
                                       lib.ptr(has), lib.ptr(info), lib.ptr(status))
    assert rc == status[0], (rc, status)
    return rc, dict(pose=pose[0], params=params[0], has=has[0], info=info[0])


def launches(lib):
    n = C.c_int64(0)
    assert lib.load().pls_launch_count(C.byref(n)) == 0
    return n.value


def state_of(lib, ctx, nq):
    """What the context exposes after a frame: the last ICP sums, the last correspondences, the map."""
    L = lib.load()
    out = {}
    sums, iters = np.zeros(30), C.c_int(0)
    out["rc_sums"] = L.pls_last_icp_sums(ctx.handle, lib.ptr(sums), C.byref(iters))
    out["sums"], out["iters"] = sums, iters.value
    corr = dict(idx=np.empty(nq, np.int64), nb=np.empty((nq, 3), np.float32), nrm=np.empty((nq, 3), np.float32),
                state=np.empty((nq, 4), np.float32), sums=np.empty(30, np.float64))
    out["rc_corr"] = L.pls_kdmap_last_correspondences(ctx.handle, nq, lib.ptr(corr["idx"]), lib.ptr(corr["nb"]),
                                                      lib.ptr(corr["nrm"]), lib.ptr(corr["state"]), lib.ptr(corr["sums"]))
    if out["rc_corr"] == 0:
        out.update({"corr_" + k: v for k, v in corr.items()})
    m = C.c_int64(0)
    assert L.pls_kdmap_size(ctx.handle, C.byref(m)) == 0
    pts = np.empty((m.value, 3), np.float32)
    assert L.pls_kdmap_points(ctx.handle, lib.ptr(pts)) == 0
    out["points"] = pts
    counts, num = np.zeros(256, np.int64), C.c_int(0)
    assert L.pls_kdmap_frames(ctx.handle, lib.ptr(counts), C.byref(num)) == 0
    out["frames"] = counts[:num.value].copy()
    return out


def run(lib, frames, local_map_size):
    """frames: (points, chain) pairs -- chain: start from the last frame's pose, else from the identity.  Returns the
    per-frame (return code, info, map frame counts)."""
    import torch
    a, b = make_ctx(lib, local_map_size), make_ctx(lib, local_map_size)
    prev = None
    log = []
    try:
        for k, (pts, chain) in enumerate(frames):
            pts = np.ascontiguousarray(pts, np.float32)
            d = torch.from_numpy(pts).cuda()
            torch.cuda.synchronize()
            init = prev if chain else None
            rc_a, oa = eager(lib, a, d, pts.shape[0], init)
            rc_b, ob = deferred(lib, b, d, pts.shape[0], init)
            assert rc_a == rc_b, (k, rc_a, rc_b)
            for key in oa:
                assert np.asarray(oa[key]).tobytes() == np.asarray(ob[key]).tobytes(), (k, key, oa[key], ob[key])
            nq = int(oa["info"][2])
            l0 = launches(lib)
            sa = state_of(lib, a, nq)
            l1 = launches(lib)
            sb = state_of(lib, b, nq)
            l2 = launches(lib)
            if k > 0:  # a's update was enqueued by its frame call, b's is enqueued by this read
                assert l1 - l0 < l2 - l1, (k, l1 - l0, l2 - l1)
            assert sa.keys() == sb.keys(), k
            for key in sa:
                assert np.asarray(sa[key]).tobytes() == np.asarray(sb[key]).tobytes(), (k, key)
            log.append((rc_a, oa["info"].copy(), sa["frames"]))
            if oa["has"]:
                prev = oa["pose"].reshape(4, 4).copy()
    finally:
        a.close()
        b.close()
    return log


@pytest.mark.parametrize("local_map_size", [20, 3])
def test_cfg2_stream_across_eviction(lib, local_map_size):
    from pylidar_slam_b200 import synthetic as syn
    frames = [(syn.scan(k, H, W), True) for k in range(23)]
    log = run(lib, frames, local_map_size)
    assert all(rc == 0 for rc, _, _ in log)
    held = [len(f) for _, _, f in log]
    assert max(held) == local_map_size and held[-1] == local_map_size, held
    # frames 20 and 21 at local_map_size 20: the first frames whose insertion evicts one
    inserted = [k for k, (_, info, _) in enumerate(log) if k > 0 and info[7] == 1.0]
    assert len(inserted) + 1 > local_map_size, inserted


def test_overflow_non_key_frame_and_second_round(lib):
    from pylidar_slam_b200 import synthetic as syn
    far = np.array([[4.0e5, 1.0, 1.0]], np.float32)
    frames = [(syn.scan(k, H, W), True) for k in range(4)]
    frames.append((np.concatenate([syn.scan(4, H, W), far]), True))  # 4: hashes beyond the compact sort keys
    frames.append((syn.scan(5, H, W), True))
    frames.append((syn.scan(5, H, W), False))                         # 6: the same scan again: not a key frame
    frames += [(syn.scan(k, H, W), False) for k in (6, 7)]            # from the identity: a few iterations each
    frames.append((syn.scan(13, H, W), False))                        # 9: six scans on: a second round of launches
    frames += [(syn.scan(k, H, W), True) for k in (14, 15, 16)]
    log = run(lib, frames, 20)
    assert all(rc == 0 for rc, _, _ in log)
    info = [i for _, i, _ in log]
    assert info[4][0] >= 1 and info[5][0] >= 1
    assert info[6][7] == 0.0 and info[5][7] == 1.0, (info[5][7], info[6][7])
    assert info[9][0] > info[8][0] + 1, [i[0] for i in info]
