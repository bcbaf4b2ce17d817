"""pls_process_frames / ICPFrameToModelBatch on projective local maps against independent contexts, bit for bit.

Every test runs the same sequences twice: batched, several projective contexts advanced by one pls_process_frames call
per step, and independently, each context with its own pls_process_frame (pls_process_frame_grid_sample with voxel > 0).
After every frame the pose, params, has-pose, all 12 info values and the last ICP iteration's 30 sums and iteration
count (pls_last_icp_sums) must be the same bits; at the end the model (pls_projmap_model, vertex and normal maps) and
pls_projmap_num_frames too.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOXEL = 0.3
_scans = {}


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def _lib_mod():
    from pylidar_slam_b200 import _lib
    return _lib


def scan(frame, H, W):
    key = (frame, H, W)
    if key not in _scans:
        from pylidar_slam_b200 import synthetic as syn
        _scans[key] = syn.scan(frame, H, W)
    return _scans[key]


def make_ctx(lib, H=64, W=720, **kw):
    args = dict(local_map_type=lib.MAP_PROJECTIVE, height=H, width=W, local_map_size=20,
                scheme=lib.SCHEMES["geman_mcclure"], sigma=0.3, max_num_alignments=10, gn_max_iters=1)
    args.update(kw)
    return lib.Context(**args)


class Frame:
    """One frame's input in one of the layouts: (address, layout with residency hint, n), kept alive by the object."""

    def __init__(self, lib, kind, pts, H, W):
        import torch
        self.pts = pts
        if kind == "tensor":
            self.keep = torch.from_numpy(pts).cuda()
            self.args = (self.keep.data_ptr(), lib.INPUT_TENSOR | lib.PTR_DEVICE, pts.shape[0])
        elif kind == "tensor64":
            self.keep = torch.from_numpy(pts.astype(np.float64)).cuda()
            self.args = (self.keep.data_ptr(), lib.INPUT_TENSOR_F64 | lib.PTR_DEVICE, pts.shape[0])
        elif kind == "ndarray":
            self.keep = np.ascontiguousarray(pts, np.float32)
            self.args = (lib.ptr(self.keep), lib.INPUT_NDARRAY | lib.PTR_HOST, pts.shape[0])
        elif kind == "f64":
            self.keep = np.ascontiguousarray(pts, np.float64)
            self.args = (lib.ptr(self.keep), lib.INPUT_NDARRAY_F64 | lib.PTR_HOST, pts.shape[0])
        elif kind in ("vmap", "vmap_host"):
            import pylidar_slam_b200 as b200
            proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
            vm = proj.build_projection_map(torch.from_numpy(pts).cuda()[None]).contiguous()
            if kind == "vmap":
                self.keep = vm
                self.args = (self.keep.data_ptr(), lib.INPUT_VERTEX_MAP, 0)
            else:
                self.keep = np.ascontiguousarray(vm.cpu().numpy(), np.float32)
                self.args = (lib.ptr(self.keep), lib.INPUT_VERTEX_MAP, 0)
        else:
            raise AssertionError(kind)
        torch.cuda.synchronize()


def single(lib, ctx, frame, voxel, init):
    """pls_process_frame (pls_process_frame_grid_sample) on one context: (status, outputs)."""
    pose, params, info, has = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    address, layout, n = frame.args
    if voxel > 0:
        st = lib.load().pls_process_frame_grid_sample(ctx.handle, address, n, voxel, layout & 0xff, lib.ptr(init),
                                                      lib.ptr(pose), lib.ptr(params), C.byref(has), lib.ptr(info))
    else:
        st = lib.load().pls_process_frame(ctx.handle, address, layout, n, lib.ptr(init), lib.ptr(pose), lib.ptr(params),
                                          C.byref(has), lib.ptr(info))
    return st, dict(pose=pose, params=params, has=np.int32(has.value), info=info)


def batch(lib, ctxs, frames, voxel, inits):
    """One pls_process_frames call: (return code, per-sequence status, per-sequence outputs)."""
    B = len(ctxs)
    handles = (C.c_void_p * B)(*[c.handle.value for c in ctxs])
    data = (C.c_void_p * B)(*[None if f is None else f.args[0] for f in frames])
    layouts = (C.c_int * B)(*[0 if f is None else f.args[1] for f in frames])
    n = (C.c_int64 * B)(*[0 if f is None else f.args[2] for f in frames])
    ip = (C.c_void_p * B)(*[None if i is None else lib.ptr(i) for i in inits])
    poses, params, has = np.zeros((B, 16), np.float32), np.zeros((B, 6), np.float32), np.zeros(B, np.int32)
    info, status = np.zeros((B, 12)), np.full(B, -1, np.int32)
    rc = lib.load().pls_process_frames(handles, B, data, layouts, n, voxel, ip, lib.ptr(poses), lib.ptr(params),
                                       lib.ptr(has), lib.ptr(info), lib.ptr(status))
    return rc, status, [dict(pose=poses[i], params=params[i], has=has[i], info=info[i]) for i in range(B)]


def last_sums(lib, ctx):
    sums, iters = np.zeros(30, np.float64), C.c_int(-1)
    st = lib.load().pls_last_icp_sums(ctx.handle, lib.ptr(sums), C.byref(iters))
    return st, dict(sums=sums, iters=np.int32(iters.value))


def model(lib, ctx):
    k = C.c_int(0)
    ctx.call("pls_projmap_num_frames", C.byref(k))
    H, W = int(ctx.cfg.height), int(ctx.cfg.width)
    vm, nm = np.zeros((k.value, 3, H, W), np.float32), np.zeros((k.value, 3, H, W), np.float32)
    if k.value:
        ctx.call("pls_projmap_model", lib.ptr(vm), lib.ptr(nm))
    return k.value, vm, nm


def same(a, b, tag):
    for key in a:
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), (tag, key, a[key], b[key])


class Pair:
    """B projective sequences, batched and independent, driven step by step.  per_seq: each sequence's context
    settings (height H and width W included)."""

    def __init__(self, lib, per_seq, voxel=0.0):
        self.lib, self.B, self.voxel = lib, len(per_seq), voxel
        self.shapes = [(kw.get("H", 64), kw.get("W", 720)) for kw in per_seq]
        self.bat = [make_ctx(lib, **kw) for kw in per_seq]
        self.ind = [make_ctx(lib, **kw) for kw in per_seq]
        self.prev = [None] * self.B
        self.iters = [[] for _ in range(self.B)]
        self.statuses = [[] for _ in range(self.B)]

    def frame(self, i, kind, k):
        H, W = self.shapes[i]
        return Frame(self.lib, kind, scan(k, H, W), H, W)

    def step(self, frames, inits=None, tag=""):
        lib = self.lib
        inits = inits or [self.prev[i] for i in range(self.B)]
        rc, status, outs = batch(lib, self.bat, frames, self.voxel, inits)
        self.outs = outs
        first_bad = next((int(s) for s in status if s != lib.PLS_OK), lib.PLS_OK)
        assert rc == first_bad, (tag, rc, status)
        for i, f in enumerate(frames):
            if f is None:
                assert status[i] == lib.PLS_OK
                continue
            st, ref = single(lib, self.ind[i], f, self.voxel, inits[i])
            assert st == status[i], (tag, i, st, status[i])
            self.statuses[i].append(st)
            if st == lib.PLS_E_SINGULAR:
                assert lib.load().pls_last_error(self.bat[i].handle) == lib.load().pls_last_error(self.ind[i].handle)
            else:
                same(outs[i], ref, (tag, i))
                self.iters[i].append(int(ref["info"][0]))
                if ref["has"]:
                    self.prev[i] = ref["pose"].reshape(4, 4).copy()
            sa, ra = last_sums(lib, self.bat[i])
            sb, rb = last_sums(lib, self.ind[i])
            assert sa == sb, (tag, i, sa, sb)
            if sa == lib.PLS_OK:
                same(ra, rb, (tag, i, "sums"))
        return status

    def finish(self):
        for i in range(self.B):
            ka, va, na = model(self.lib, self.bat[i])
            kb, vb, nb = model(self.lib, self.ind[i])
            assert ka == kb, i
            assert va.tobytes() == vb.tobytes() and na.tobytes() == nb.tobytes(), i
        for c in self.bat + self.ind:
            c.close()


def test_five_kitti_shaped_vertex_map_sequences(lib):
    """64x720, K = 20, vertex maps on the device: the maps fill (frame 20) and then evict."""
    pair = Pair(lib, [{}] * 5)
    for k in range(30):
        pair.step([pair.frame(i, "vmap", 200 * i + k) for i in range(5)], tag=k)
    assert all(len(it) == 30 for it in pair.iters)
    assert all(model(lib, c)[0] == 20 for c in pair.bat)
    pair.finish()


SCHEMES = ["least_square", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
MIXED = [dict(H=16, W=512, local_map_size=1, normals_kernel_size=3, max_num_alignments=1),
         dict(H=64, W=720, local_map_size=2, normals_kernel_size=5, max_num_alignments=10),
         dict(H=64, W=1024, local_map_size=10, normals_kernel_size=7, max_num_alignments=20),
         dict(H=128, W=2048, local_map_size=20, normals_kernel_size=5, max_num_alignments=10),
         dict(H=64, W=720, local_map_size=30, normals_kernel_size=3, max_num_alignments=20),
         dict(H=16, W=512, local_map_size=20, normals_kernel_size=7, max_num_alignments=10),
         dict(H=64, W=1024, local_map_size=30, normals_kernel_size=5, max_num_alignments=1)]


def _mixed(lib):
    per = []
    for j, kw in enumerate(MIXED):
        kw = dict(kw, scheme=lib.SCHEMES[SCHEMES[j]], sigma=0.3 + 0.1 * j)
        per.append(kw)
    return per


def test_mixed_shapes_sizes_schemes_and_alignments(lib):
    """16x512, 64x720, 64x1024 and 128x2048 in one call; K 1, 2, 10, 20, 30; the seven weighting schemes; normals
    kernels 3, 5, 7; 1, 10 and 20 alignments.  Different tile counts, TMA block counts and candidate splits side by
    side."""
    pair = Pair(lib, _mixed(lib))
    kinds = ["tensor", "ndarray", "tensor", "vmap", "tensor", "f64", "tensor"]
    for k in range(24):
        pair.step([pair.frame(i, kinds[i], 300 * i + k) for i in range(pair.B)], tag=k)
    assert sum(pair.iters[0][1:]) == len(pair.iters[0]) - 1   # one alignment
    pair.finish()


def test_every_input_layout(lib):
    kinds = ["tensor", "tensor64", "ndarray", "f64", "vmap", "vmap_host"]
    pair = Pair(lib, [{}] * len(kinds))
    for k in range(12):
        pair.step([pair.frame(i, kinds[i], 200 * i + k) for i in range(len(kinds))], tag=k)
    pair.finish()


def test_grid_sampled_sequences(lib):
    kinds = ["tensor", "ndarray", "tensor", "ndarray"]
    pair = Pair(lib, [{}, {}, dict(H=128, W=2048), dict(H=16, W=512, local_map_size=5)], voxel=VOXEL)
    for k in range(12):
        pair.step([pair.frame(i, kinds[i], 200 * i + k) for i in range(4)], tag=k)
    assert all(int(o["info"][4]) > 0 for o in pair.outs)
    pair.finish()


def test_direct_path_sequence_beside_tma_sequences(lib):
    """33x500 pixels are no whole number of 128-pixel tiles: that sequence runs proj_icp_iter_kernel through its own
    launches, in the same call as two TMA sequences."""
    pair = Pair(lib, [{}, dict(H=33, W=500, local_map_size=5), dict(H=64, W=1024)])
    for k in range(12):
        pair.step([pair.frame(i, "tensor", 200 * i + k) for i in range(3)], tag=k)
    pair.finish()


def _no_tma_body():
    lib = _lib_mod()
    pair = Pair(lib, [{}, dict(H=33, W=500, local_map_size=5), dict(H=16, W=512, local_map_size=3)])
    for k in range(8):
        pair.step([pair.frame(i, "tensor", 200 * i + k) for i in range(3)], tag=k)
    pair.finish()


def test_whole_batch_without_tma_in_a_subprocess():
    env = dict(os.environ, PLS_PROJ_NO_TMA="1", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_multi_sequence_projective_gpu as t; t._no_tma_body(); print('no-tma ok')"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "no-tma ok" in r.stdout, r.stdout + r.stderr


def test_sequences_at_different_phases(lib):
    """Sequence 1 joins at step 8 (its frame 0 inside the batch), 2 stops at step 14, 3 is re-initialised at 10."""
    pair = Pair(lib, [{}, dict(H=64, W=1024), {}, dict(H=16, W=512)])
    start = {0: 0, 1: 8, 2: 0, 3: 0}
    kinds = ["tensor", "ndarray", "vmap", "tensor"]
    for k in range(18):
        if k == 10:
            for c in (pair.bat[3], pair.ind[3]):
                c.call("pls_odometry_init")
            pair.prev[3] = None
            start[3] = 10
        frames = []
        for i in range(4):
            if k < start[i] or (i == 2 and k >= 14):
                frames.append(None)
            else:
                frames.append(pair.frame(i, kinds[i], 200 * i + k - start[i]))
        pair.step(frames, tag=k)
    assert pair.iters[1][0] == 0 and pair.iters[3][10] == 0   # frame 0 of a sequence inside the batch
    pair.finish()


def test_iteration_spread_and_extra_rounds(lib):
    """Sequence 0 never stops early (threshold_delta_pose = 0, 20 alignments), sequence 1 stops at 2 alignments, and
    sequence 2 takes every third frame from the identity on odd steps: more iterations than its previous frame's + 1."""
    pair = Pair(lib, [dict(threshold_delta_pose=0.0, max_num_alignments=20), dict(max_num_alignments=2),
                      dict(max_num_alignments=30)])
    for k in range(14):
        inits = [pair.prev[0], pair.prev[1], None if k % 2 else pair.prev[2]]
        pair.step([pair.frame(0, "tensor", k), pair.frame(1, "ndarray", 200 + k), pair.frame(2, "tensor", 3 * k)],
                  inits=inits, tag=k)
    assert pair.iters[0][1:] == [20] * 13, pair.iters[0]
    assert max(pair.iters[1][1:]) == 2, pair.iters[1]
    it2 = pair.iters[2]
    assert any(it2[k] > it2[k - 1] + 1 for k in range(2, len(it2))), it2   # the extra-round path ran
    pair.finish()


def _two_points(k):
    """Two finite points of scan k: two correspondences leave the 6x6 normal equations singular."""
    pts = scan(k, 64, 720)
    ok = np.flatnonzero(np.isfinite(pts).all(axis=1) & (np.abs(pts).sum(axis=1) > 0))
    return np.ascontiguousarray(pts[ok[[len(ok) // 3, 2 * len(ok) // 3]]])


def test_singular_sequence_among_healthy_ones(lib):
    """Two points per frame after a full frame 0 leave the normal equations singular: only that sequence's status fails,
    and its next frame runs as on a context that saw the same error alone."""
    pair = Pair(lib, [{}, {}, dict(H=64, W=1024)])
    for k in range(6):
        pts = scan(200 + k, 64, 720) if k == 0 else _two_points(200 + k)
        frames = [pair.frame(0, "tensor", k), Frame(lib, "ndarray", pts, 64, 720), pair.frame(2, "tensor", 400 + k)]
        status = pair.step(frames, tag=k)
        if k >= 1:
            assert status[0] == status[2] == lib.PLS_OK, status
    assert lib.PLS_E_SINGULAR in pair.statuses[1][1:], pair.statuses[1]
    pair.finish()


def test_one_sequence_equals_process_frame(lib):
    pair = Pair(lib, [{}])
    for k in range(12):
        pair.step([pair.frame(0, "tensor", k)], tag=k)
    pair.finish()


def test_sixty_four_kitti_shaped_sequences(lib):
    pair = Pair(lib, [{}] * lib.MAX_SEQUENCES)
    kinds = ["tensor", "vmap"]
    for k in range(4):
        pair.step([pair.frame(i, kinds[i % 2], 10 * i + k) for i in range(pair.B)], tag=k)
    pair.finish()


def test_rejections_change_no_context(lib):
    pair = Pair(lib, [{}, dict(H=16, W=512)])
    frames = lambda k: [pair.frame(0, "tensor", k), pair.frame(1, "tensor", 200 + k)]  # noqa: E731
    pair.step(frames(0))
    pair.step(frames(1))
    kd = make_ctx(lib, local_map_type=lib.MAP_KDTREE)
    fine = make_ctx(lib, gn_max_iters=2)
    f = frames(2)
    for ctxs, why in (([pair.bat[0], kd], "kd-tree"), ([pair.bat[1], fine], "max_iters == 1")):
        rc, status, _ = batch(lib, ctxs, f, 0.0, [None] * len(ctxs))
        assert rc == lib.PLS_E_INVALID, rc
        assert why in lib.load().pls_last_error(ctxs[0].handle).decode(), why
    for c in (kd, fine):
        c.close()
    for k in range(2, 5):   # the refused calls left both sequences where they were; an all-projective call runs
        pair.step(frames(k), tag=k)
    pair.finish()


# ---------------------------------------------------------------------------------------------------------- Python
def _algos(b200, B, device):
    proj = b200.SphericalProjector(height=64, width=720, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.ProjectiveLocalMapConfig(local_map_size=20),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
        max_num_alignments=10, data_key="input_data")
    algos = [b200.ICPFrameToModel(cfg, projector=proj, device=device) for _ in range(B)]
    for a in algos:
        a.init()
    return algos


def test_python_batch_equals_independent_runs():
    import torch
    import pylidar_slam_b200 as b200
    B = 3
    batched, alone = _algos(b200, B, "cuda:0"), _algos(b200, B, "cuda:0")
    group = b200.ICPFrameToModelBatch(batched)
    prev_a, prev_b = [None] * B, [None] * B

    def dicts(k, prev):
        return [{"input_data": torch.from_numpy(scan(200 * i + k, 64, 720)).cuda(), "init_rpose": prev[i]} for i in range(B)]

    for k in range(10):
        da, db = dicts(k, prev_a), dicts(k, prev_b)
        if k % 4 == 3:   # mixing: this step through process_next_frame on the batched objects
            for a, dd in zip(batched, da):
                a.process_next_frame(dd)
        else:
            group.process_next_frames(da)
        for b, dd in zip(alone, db):
            b.process_next_frame(dd)
        for i in range(B):
            for key in ("odometry_pose", "odometry_pc"):
                assert (key in da[i]) == (key in db[i]), key
                if key in da[i]:
                    assert np.asarray(da[i][key]).tobytes() == np.asarray(db[i][key]).tobytes(), (k, i, key)
            assert batched[i].get_relative_poses().tobytes() == alone[i].get_relative_poses().tobytes()
            if "odometry_pose" in da[i]:
                prev_a[i] = da[i]["odometry_pose"].astype(np.float64)
                prev_b[i] = db[i]["odometry_pose"].astype(np.float64)
    for a in batched + alone:
        a.ctx.close()
