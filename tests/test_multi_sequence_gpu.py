"""pls_process_frames / ICPFrameToModelBatch against independent contexts, bit for bit.

Every test runs the same sequences twice: batched, several contexts advanced by one pls_process_frames call per step,
and independently, each context with its own pls_process_frame (pls_process_frame_grid_sample with voxel > 0).  After
every frame the pose, params, has-pose, all 12 info values and the last kd search (pls_kdmap_last_correspondences:
indices, neighbours, normals, search states, the 30 sums) must be the same bits; at the end the map points too.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

H, W, VOXEL = 64, 2048, 0.3
_scans = {}


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def scan(frame):
    if frame not in _scans:
        from pylidar_slam_b200 import synthetic as syn
        _scans[frame] = syn.scan(frame, H, W)
    return _scans[frame]


def sampled(frame):
    import pylidar_slam_b200 as b200
    key = ("gs", frame)
    if key not in _scans:
        _scans[key] = np.ascontiguousarray(b200.grid_sample(scan(frame), VOXEL)[0])
    return _scans[key]


def make_ctx(lib, **kw):
    args = dict(local_map_type=lib.MAP_KDTREE, height=H, width=W, local_map_size=20, scheme=lib.SCHEMES["geman_mcclure"],
                sigma=0.3, max_num_alignments=10, gn_max_iters=1)
    args.update(kw)
    return lib.Context(**args)


class Frame:
    """One frame's input in one of the layouts: (address, layout with residency hint, n), kept alive by the object."""

    def __init__(self, lib, kind, pts):
        import torch
        self.pts = pts
        if kind == "tensor":
            self.keep = torch.from_numpy(pts).cuda()
            self.args = (self.keep.data_ptr(), lib.INPUT_TENSOR | lib.PTR_DEVICE, pts.shape[0])
        elif kind == "ndarray":
            self.keep = np.ascontiguousarray(pts, np.float32)
            self.args = (lib.ptr(self.keep), lib.INPUT_NDARRAY | lib.PTR_HOST, pts.shape[0])
        elif kind == "f64":
            self.keep = np.ascontiguousarray(pts, np.float64)
            self.args = (lib.ptr(self.keep), lib.INPUT_NDARRAY_F64 | lib.PTR_HOST, pts.shape[0])
        elif kind == "vmap":
            import pylidar_slam_b200 as b200
            proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
            self.keep = proj.build_projection_map(torch.from_numpy(pts).cuda()[None]).contiguous()
            self.args = (self.keep.data_ptr(), lib.INPUT_VERTEX_MAP, 0)
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


def readback(lib, ctx, nq):
    out = dict(idx=np.empty(nq, np.int64), nb=np.empty((nq, 3), np.float32), nrm=np.empty((nq, 3), np.float32),
               state=np.empty((nq, 4), np.float32), sums=np.empty(30, np.float64))
    st = lib.load().pls_kdmap_last_correspondences(ctx.handle, nq, lib.ptr(out["idx"]), lib.ptr(out["nb"]), lib.ptr(out["nrm"]),
                                                    lib.ptr(out["state"]), lib.ptr(out["sums"]))
    return st, out


def map_points(ctx):
    import pylidar_slam_b200 as b200
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(), ctx=ctx)
    return lm.points()


def same(a, b, tag):
    for key in a:
        assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes(), (tag, key, a[key], b[key])


class Pair:
    """B sequences, batched and independent, driven step by step from a plan."""

    def __init__(self, lib, B, voxel=0.0, **ctx_kw):
        self.lib, self.B, self.voxel = lib, B, voxel
        kws = ctx_kw.get("per_seq") or [{}] * B
        self.bat = [make_ctx(lib, **kw) for kw in kws]
        self.ind = [make_ctx(lib, **kw) for kw in kws]
        self.prev = [None] * B
        self.iters = [[] for _ in range(B)]
        self.statuses = [[] for _ in range(B)]

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
            nq = int(ref["info"][2])
            sa, ra = readback(lib, self.bat[i], nq)
            sb, rb = readback(lib, self.ind[i], nq)
            assert sa == sb, (tag, i, sa, sb)
            if sa == lib.PLS_OK:
                same(ra, rb, (tag, i, "correspondences"))
        return status

    def finish(self):
        for i in range(self.B):
            a, b = map_points(self.bat[i]), map_points(self.ind[i])
            assert a.tobytes() == b.tobytes(), i
        for c in self.bat + self.ind:
            c.close()


def test_five_sequences_mixed_layouts(lib):
    kinds = ["tensor", "ndarray", "vmap", "f64", "tensor"]
    pair = Pair(lib, 5)
    for k in range(30):
        pair.step([Frame(lib, kinds[i], sampled(200 * i + k)) for i in range(5)], tag=k)
    assert all(len(st) == 30 for st in pair.statuses)
    assert all(len(pair.iters[i]) == 30 for i in (0, 1, 3, 4)), [len(it) for it in pair.iters]
    pair.finish()


def test_grid_sampled_sequences(lib):
    kinds = ["tensor", "ndarray", "tensor", "ndarray", "tensor"]
    pair = Pair(lib, 5, voxel=VOXEL)
    for k in range(30):
        pair.step([Frame(lib, kinds[i], scan(200 * i + k)) for i in range(5)], tag=k)
    pair.finish()


def test_grid_sampled_sequence_beyond_the_compact_sort_keys(lib):
    """Sequence 2's scans are shifted by 5e5 m: its voxel hashes exceed the 40-bit sort keys, and the batched call samples
    it once more on the raw 64-bit keys, as pls_process_frame_grid_sample does.  Its frame 0 lies outside the vertical
    field of view, so its kd map is filled from that scan before the ICP frames."""
    from oracle import icp_oracle as orc
    import pylidar_slam_b200 as b200
    pair = Pair(lib, 3, voxel=VOXEL)
    eye = np.eye(4, dtype=np.float32)
    for k in range(6):
        far = np.ascontiguousarray(scan(400 + k) + np.float32(5.0e5))
        assert np.abs(orc.voxel_hashes(orc.voxel_coords(far, VOXEL))).max() >= 2 ** 39
        pair.step([Frame(lib, "tensor", scan(k)), Frame(lib, "ndarray", scan(200 + k)), Frame(lib, "ndarray", far)], tag=k)
        if pair.statuses[2][-1] == lib.PLS_OK:
            assert int(pair.outs[2]["info"][4]) == orc.grid_sample(far, VOXEL)[1].shape[0], k
        if k == 0:
            fill = np.ascontiguousarray(b200.grid_sample(far, VOXEL)[0])
            for c in (pair.bat[2], pair.ind[2]):
                c.call("pls_kdmap_update_points", lib.ptr(eye), lib.ptr(fill), fill.shape[0])
    assert pair.statuses[2][0] == lib.PLS_OK and pair.iters[2][0] == 0, pair.statuses[2]
    assert sum(it > 0 for it in pair.iters[2][1:]) >= 2, (pair.iters[2], pair.statuses[2])
    pair.finish()


def test_one_sequence_equals_process_frame(lib):
    pair = Pair(lib, 1)
    for k in range(12):
        pair.step([Frame(lib, "tensor", sampled(k))], tag=k)
    pair.finish()


def test_sequences_at_different_phases(lib):
    """Sequence 1 joins at step 10 (its frame 0 inside the batch), 2 stops at step 20, 3 is re-initialised at 15."""
    pair = Pair(lib, 4)
    start = {0: 0, 1: 10, 2: 0, 3: 0}
    for k in range(26):
        if k == 15:
            for c in (pair.bat[3], pair.ind[3]):
                c.call("pls_odometry_init")
            pair.prev[3] = None
            start[3] = 15
        frames = []
        for i in range(4):
            if k < start[i] or (i == 2 and k >= 20):
                frames.append(None)
            else:
                frames.append(Frame(lib, "tensor", sampled(200 * i + k - start[i])))
        pair.step(frames, tag=k)
    assert pair.iters[1][0] == 0 and pair.iters[3][15] == 0   # frame 0 of a sequence inside the batch
    pair.finish()


def test_sequences_with_different_normal_neighbour_counts(lib):
    """k = 3, 10 and 31 normal neighbours in one call: the normals and refine kernels read each sequence's own k from
    its descriptor.  All three run the same frames, so their normals must differ from one another."""
    ks = (3, 10, 31)
    pair = Pair(lib, 3, per_seq=[dict(num_neighbors_normals=k) for k in ks])
    for k in range(16):
        f = sampled(k)
        pair.step([Frame(lib, kind, f) for kind in ("tensor", "ndarray", "tensor")], tag=k)
        if k == 1:
            nq = int(pair.outs[0]["info"][2])
            nrm = [readback(lib, c, nq)[1]["nrm"] for c in pair.bat]
            assert all(not np.array_equal(nrm[i], nrm[j]) for i, j in ((0, 1), (0, 2), (1, 2)))
    assert all(len(it) == 16 for it in pair.iters) and max(max(it) for it in pair.iters) >= 2, pair.iters
    pair.finish()


def test_iteration_spread_and_extra_rounds(lib):
    """Sequence 0 takes every third frame and starts from the identity on odd steps: more iterations than the previous
    frame's count + 1, beside a sequence that converges in one or two."""
    pair = Pair(lib, 2, per_seq=[dict(max_num_alignments=30), dict(max_num_alignments=10)])
    for k in range(16):
        inits = [None if k % 2 else pair.prev[0], pair.prev[1]]
        pair.step([Frame(lib, "tensor", sampled(3 * k)), Frame(lib, "ndarray", sampled(200 + k))], inits=inits, tag=k)
    it0 = pair.iters[0]
    assert any(it0[k] > it0[k - 1] + 1 for k in range(2, len(it0))), it0   # the extra-round path ran
    assert min(pair.iters[1][1:]) <= 2, pair.iters[1]
    pair.finish()


def test_cold_map_sequence_beside_a_cfg2_one(lib):
    """A map filled to 2 M points takes the four-launch path for its later iterations, in the same batch."""
    pair = Pair(lib, 2, per_seq=[dict(local_map_size=40), {}])
    rng = np.random.RandomState(3)
    fill = np.ascontiguousarray(rng.uniform([-60, -60, -2], [60, 60, 4], (2_000_000, 3)).astype(np.float32))
    eye = np.eye(4, dtype=np.float32)
    for k in range(8):
        if k == 1:
            for c in (pair.bat[0], pair.ind[0]):
                c.call("pls_kdmap_update_points", lib.ptr(eye), lib.ptr(fill), fill.shape[0])
        pair.step([Frame(lib, "tensor", sampled(k)), Frame(lib, "tensor", sampled(200 + k))], tag=k)
        if k >= 1:
            assert pair.prev[0] is not None
    n = C.c_int64(0)
    pair.bat[0].call("pls_kdmap_size", C.byref(n))
    assert n.value >= 2_000_000
    pair.finish()


def _plane(shift):
    g = np.arange(-20.0, 20.0, 0.25)
    x, y = np.meshgrid(g, g)
    keep = np.hypot(x, y) > 5.0
    return np.ascontiguousarray(np.stack([x[keep], y[keep], np.full(keep.sum(), -1.5 + shift)], 1).astype(np.float32))


def test_singular_sequence_among_healthy_ones(lib):
    pair = Pair(lib, 3)
    for k in range(6):
        frames = [Frame(lib, "tensor", sampled(k)), Frame(lib, "ndarray", _plane(0.0 if k == 0 else 0.05 * k)),
                  Frame(lib, "tensor", sampled(400 + k))]
        status = pair.step(frames, tag=k)
        if k >= 1:
            assert status[1] == lib.PLS_E_SINGULAR and status[0] == status[2] == lib.PLS_OK, status
    assert pair.statuses[1][1:] == [lib.PLS_E_SINGULAR] * 5
    pair.finish()


def test_rejections_change_no_context(lib):
    pair = Pair(lib, 2)
    frames = lambda k: [Frame(lib, "tensor", sampled(k)), Frame(lib, "tensor", sampled(200 + k))]  # noqa: E731
    pair.step(frames(0))
    pair.step(frames(1))
    proj = make_ctx(lib, local_map_type=lib.MAP_PROJECTIVE)
    fine = make_ctx(lib, gn_max_iters=2)
    many = [pair.bat[0]] + [make_ctx(lib) for _ in range(64)]   # 65 distinct contexts: only the count is wrong
    f = frames(2)
    for ctxs, fr, why in (([pair.bat[0], proj], f, "kd-tree"), ([pair.bat[0], pair.bat[0]], f, "twice"),
                          ([pair.bat[1], fine], f, "max_iters == 1"), (many, [f[0]] * 65, "PLS_MAX_SEQUENCES")):
        rc, status, _ = batch(lib, ctxs, fr, 0.0, [None] * len(ctxs))
        assert rc == lib.PLS_E_INVALID, rc
        assert why in lib.load().pls_last_error(ctxs[0].handle).decode(), why
    for c in [proj, fine] + many[1:]:
        c.close()
    for k in range(2, 5):   # the refused calls left both sequences where they were
        pair.step(frames(k), tag=k)
    pair.finish()


# ---------------------------------------------------------------------------------------------------------- Python
def _algos(b200, B, device):
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=20),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
        max_num_alignments=10, data_key="input_data")
    algos = [b200.ICPFrameToModel(cfg, projector=proj, device=device) for _ in range(B)]
    for a in algos:
        a.init()
    return algos


def _check_python(a, b, da, db):
    for key in ("odometry_pose", "odometry_pc"):
        assert (key in da) == (key in db), key
        if key in da:
            assert np.asarray(da[key]).tobytes() == np.asarray(db[key]).tobytes(), key
    assert a.get_relative_poses().tobytes() == b.get_relative_poses().tobytes()
    assert np.asarray(a.absolute_poses).tobytes() == np.asarray(b.absolute_poses).tobytes()


@pytest.mark.parametrize("route", ["shipped_chain", "device_tensors"])
def test_python_batch_equals_independent_runs(route):
    import torch
    import pylidar_slam_b200 as b200
    B = 3
    batched, alone = _algos(b200, B, "cuda:0"), _algos(b200, B, "cuda:0")
    group = b200.ICPFrameToModelBatch(batched)
    pre = b200.Preprocessing(b200.PreprocessingConfig(filters={
        "2": dict(filter_name="grid_sample", voxel_size=VOXEL, pointcloud_key="numpy_pc"),
        "3": dict(filter_name="to_tensor", keys=dict(sample_points="input_data"))}))
    prev_a, prev_b = [None] * B, [None] * B

    def dicts(k, prev):
        out = []
        for i in range(B):
            if route == "shipped_chain":
                dd = {"numpy_pc": scan(200 * i + k), "init_rpose": prev[i]}
                pre.forward(dd)
            else:
                dd = {"input_data": torch.from_numpy(sampled(200 * i + k)).cuda(), "init_rpose": prev[i]}
            out.append(dd)
        return out

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
            _check_python(batched[i], alone[i], da[i], db[i])
            if "odometry_pose" in da[i]:
                prev_a[i] = da[i]["odometry_pose"].astype(np.float64)
                prev_b[i] = db[i]["odometry_pose"].astype(np.float64)
    assert all(len(a.elapsed) == 10 for a in batched)
    group.process_next_frames([None] * B)   # nothing to do: nothing changes
    assert all(len(a.relative_poses) == 10 for a in batched)
    for a in batched + alone:
        a.ctx.close()
