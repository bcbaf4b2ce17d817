"""ICPFrameToModelBatch over projective local maps without a GPU, through the fake context of
tests/test_multi_sequence_cpu.py (the CPU oracle's ICP behind pls_process_frames): homogeneous projective batches are
accepted and fill their data_dicts like independent runs, mixed batches are refused naming the kd-tree, and every input
layout reaches pls_process_frames as process_next_frame would hand it to pls_process_frame.  The kernels themselves are
tested by tests/test_multi_sequence_projective_gpu.py."""
import numpy as np
import pytest

import test_multi_sequence_cpu as base
from test_multi_sequence_cpu import FakeBatchContext


@pytest.fixture
def b200(monkeypatch):
    import pylidar_slam_b200 as pkg
    from pylidar_slam_b200 import _lib
    monkeypatch.setattr(_lib, "Context", FakeBatchContext)
    return pkg


def _proj_algos(b200, B, size=4, data_key="numpy_pc"):
    proj = b200.SphericalProjector(height=base.H, width=base.W, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.ProjectiveLocalMapConfig(local_map_size=size),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
        max_num_alignments=6, data_key=data_key)
    algos = [b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0") for _ in range(B)]
    for a in algos:
        a.init()
    return algos


def test_projective_batch_is_accepted_and_equals_independent_runs(b200):
    from pylidar_slam_b200 import _lib
    B = 3
    batched, alone = _proj_algos(b200, B), _proj_algos(b200, B)
    assert all(a.ctx.cfg.local_map_type == _lib.MAP_PROJECTIVE for a in batched)
    group = b200.ICPFrameToModelBatch(batched)
    prev_a, prev_b = [None] * B, [None] * B
    for k in range(4):
        skip = {2} if k == 1 else set()
        da, db = base._dicts(B, k, prev_a, skip), base._dicts(B, k, prev_b, skip)
        if k == 3:   # mixed with process_next_frame on the same objects
            for a, dd in zip(batched, da):
                a.process_next_frame(dd)
        else:
            group.process_next_frames(da)
        for b, dd in zip(alone, db):
            if dd is not None:
                b.process_next_frame(dd)
        for i in range(B):
            if da[i] is None:
                continue
            assert set(da[i]) == set(db[i]), (k, i)
            for key in ("odometry_pose", "odometry_pc"):
                if key in db[i]:
                    np.testing.assert_array_equal(da[i][key], db[i][key])
            if "odometry_pose" in da[i]:
                prev_a[i], prev_b[i] = da[i]["odometry_pose"].astype(np.float64), db[i]["odometry_pose"].astype(np.float64)
    for a, b in zip(batched, alone):
        np.testing.assert_array_equal(a.get_relative_poses(), b.get_relative_poses())
    assert [len(a.relative_poses) for a in batched] == [4, 4, 3]
    assert sum(a.ctx.batched_calls for a in batched) == 3


def test_projective_batches_of_different_sizes_are_accepted(b200):
    a, = _proj_algos(b200, 1, size=2)
    b, = _proj_algos(b200, 1, size=7)
    group = b200.ICPFrameToModelBatch([a, b])
    group.process_next_frames(base._dicts(2, 0, [None, None]))
    assert len(a.relative_poses) == len(b.relative_poses) == 1


@pytest.mark.parametrize("order", ["projective_first", "kd_first"])
def test_mixed_map_types_are_refused(b200, order):
    kd, = base._algos(b200, 1)
    proj, = _proj_algos(b200, 1)
    pair = [proj, kd] if order == "projective_first" else [kd, proj]
    with pytest.raises(AssertionError, match="kd-tree"):
        b200.ICPFrameToModelBatch(pair)
    assert kd.ctx.frame_calls == 0 and proj.ctx.frame_calls == 0


def test_projective_rejections_as_on_the_kd_batch(b200):
    a, b = _proj_algos(b200, 2)
    with pytest.raises(AssertionError, match="twice"):
        b200.ICPFrameToModelBatch([a, a])
    (fine,) = base._algos(b200, 1, gn_iters=3, local_map=b200.ProjectiveLocalMapConfig(local_map_size=4))
    with pytest.raises(AssertionError, match="max_iters == 1"):
        b200.ICPFrameToModelBatch([a, fine])
    b.ctx.cfg.device = 1
    with pytest.raises(AssertionError, match="one CUDA device"):
        b200.ICPFrameToModelBatch([a, b])


class Recorder(FakeBatchContext):
    """Records the (data, layout, n) triples pls_process_frames receives, and what pls_process_frame receives."""
    batched = []
    single = []

    def process_frames(self, handles, num, data, layouts, n, voxel, *rest):
        Recorder.batched.append([(bool(data[i]), int(layouts[i]), int(n[i])) for i in range(num)])
        return super().process_frames(handles, num, data, layouts, n, voxel, *rest)

    def pls_process_frame(self, data, layout, n, *rest):
        Recorder.single.append((bool(data), int(layout), int(n)))
        return super().pls_process_frame(data, layout, n, *rest)


def test_layouts_handed_to_process_frames(monkeypatch):
    """float32 and float64 ndarrays, float32 / float64 CPU tensors: the batch passes each sequence the
    layout and row count that process_next_frame passes to pls_process_frame."""
    import torch
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import _lib
    monkeypatch.setattr(_lib, "Context", Recorder)
    Recorder.batched.clear()
    Recorder.single.clear()
    pts = base._frame(0, 0)
    inputs = [pts.astype(np.float32), pts.astype(np.float64), torch.from_numpy(pts.astype(np.float32)),
              torch.from_numpy(pts.astype(np.float64))]
    B = len(inputs)
    batched, alone = _proj_algos(b200, B, data_key="input_data"), _proj_algos(b200, B, data_key="input_data")
    group = b200.ICPFrameToModelBatch(batched)
    group.process_next_frames([{"input_data": x} for x in inputs])
    Recorder.single.clear()
    for a, x in zip(alone, inputs):
        a.process_next_frame({"input_data": x})
    assert len(Recorder.batched) == 1
    got = Recorder.batched[0]
    assert [g[0] for g in got] == [True] * B
    assert [(g[1] & 0xff, g[2]) for g in got] == [(s[1] & 0xff, s[2]) for s in Recorder.single]
    assert [g[1] & 0xff for g in got] == [_lib.INPUT_NDARRAY, _lib.INPUT_NDARRAY_F64, _lib.INPUT_TENSOR,
                                          _lib.INPUT_TENSOR_F64]
    assert all(g[2] == pts.shape[0] for g in got)
