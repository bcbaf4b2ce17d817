"""Host logic of ICPFrameToModelBatch without a GPU: a fake context whose pls_process_frames loops over the fake
pls_process_frame of tests/dryrun_next_rows.FakeContext (the CPU oracle's ICP behind the C ABI).  Checks data_dict
filling against independent process_next_frame runs, None skips, `elapsed`, the singular-error semantics and the
constructor's rejections.  The kernels themselves are tested by tests/test_multi_sequence_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import dryrun_next_rows as dry
from oracle import icp_oracle as orc
from pylidar_slam_b200 import synthetic as syn

H, W = 32, 512


class FakeBatchContext(dry.FakeContext):
    """FakeContext with a handle and pls_process_frames.  `failing_calls`: indices of this context's frame calls that
    report a status (PLS_E_SINGULAR, PLS_E_CUDA) instead of running (the frame is not advanced, as after the real error)."""
    by_handle = {}

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.cfg.local_map_type = int(kwargs.get("local_map_type", 0))
        self.handle = C.c_void_p(id(self))
        self.failing_calls = {}   # frame call index -> status it reports instead of running
        self.frame_calls = 0
        self.batched_calls = 0
        FakeBatchContext.by_handle[id(self)] = self

    def check(self, status):
        from pylidar_slam_b200 import _lib
        return _lib.check(None, status)

    def process_frames(self, handles, num, data, layouts, n, voxel, inits, poses, params, has, info, status):
        from pylidar_slam_b200 import _lib
        self.batched_calls += 1
        st = dry.arr(status, (num,), np.int32)
        has_out = dry.arr(has, (num,), np.int32)
        first = _lib.PLS_OK
        for i in range(num):
            if not data[i]:
                continue
            ctx = FakeBatchContext.by_handle[handles[i]]
            ctx.frame_calls += 1
            failure = ctx.failing_calls.get(ctx.frame_calls - 1)
            if failure:   # the frame does not run
                st[i] = failure
                first = first or failure
                continue
            h = C.c_int(0)
            ctx.pls_process_frame(data[i], layouts[i], n[i], inits[i], poses + 64 * i, params + 24 * i, C.byref(h),
                                  info + 96 * i)
            has_out[i] = h.value
            st[i] = _lib.PLS_OK
        return first


@pytest.fixture
def b200(monkeypatch):
    import pylidar_slam_b200 as pkg
    from pylidar_slam_b200 import _lib
    monkeypatch.setattr(_lib, "Context", FakeBatchContext)
    return pkg


def _algos(b200, B, **cfg_kw):
    proj = b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=cfg_kw.pop("local_map", b200.KdTreeLocalMapConfig(local_map_size=4)),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                              max_iters=cfg_kw.pop("gn_iters", 1))),
        max_num_alignments=6, data_key="numpy_pc")
    algos = [b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0") for _ in range(B)]
    for a in algos:
        a.init()
    return algos


def _frame(seq, k):
    s, _ = orc.grid_sample(syn.scan(100 * seq + k, H, W), 0.4)
    return s


def _dicts(B, k, prev, skip=()):
    return [None if i in skip else {"numpy_pc": _frame(i, k), "init_rpose": prev[i]} for i in range(B)]


def test_batch_fills_data_dicts_like_independent_runs_and_skips_none(b200):
    B = 3
    batched, alone = _algos(b200, B), _algos(b200, B)
    group = b200.ICPFrameToModelBatch(batched)
    prev_a, prev_b = [None] * B, [None] * B
    for k in range(4):
        skip = {1} if k == 2 else set()
        da, db = _dicts(B, k, prev_a, skip), _dicts(B, k, prev_b, skip)
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
                    assert da[i][key].dtype == db[i][key].dtype
            if "odometry_pose" in da[i]:
                prev_a[i], prev_b[i] = da[i]["odometry_pose"].astype(np.float64), db[i]["odometry_pose"].astype(np.float64)
    for a, b in zip(batched, alone):
        np.testing.assert_array_equal(a.get_relative_poses(), b.get_relative_poses())
        np.testing.assert_array_equal(np.asarray(a.absolute_poses), np.asarray(b.absolute_poses))
    assert [len(a.relative_poses) for a in batched] == [4, 3, 4]
    assert [len(a.elapsed) for a in batched] == [4, 3, 4]
    assert batched[0].ctx.batched_calls + batched[1].ctx.batched_calls + batched[2].ctx.batched_calls == 3


def test_elapsed_is_the_call_time_shared_by_its_frames(b200, monkeypatch):
    import types
    import pylidar_slam_b200.odometry as odo
    batched = _algos(b200, 3)
    group = b200.ICPFrameToModelBatch(batched)
    clock = iter([10.0, 16.0, 20.0])
    monkeypatch.setattr(odo, "time", types.SimpleNamespace(time=lambda: next(clock)))
    group.process_next_frames(_dicts(3, 0, [None] * 3, skip={2}))
    assert batched[0].elapsed == [3.0] and batched[1].elapsed == [3.0] and batched[2].elapsed == []
    group.process_next_frames([None, None, None])   # no frame: no call, no time
    assert batched[0].elapsed == [3.0]


def test_singular_sequence_raises_after_the_others_are_filled(b200):
    B = 3
    batched, alone = _algos(b200, B), _algos(b200, B)
    group = b200.ICPFrameToModelBatch(batched)
    prev = [None] * B
    group.process_next_frames(_dicts(B, 0, prev))
    for b, dd in zip(alone, _dicts(B, 0, prev)):
        b.process_next_frame(dd)
    batched[1].ctx.failing_calls[1] = 3   # PLS_E_SINGULAR
    da, db = _dicts(B, 1, prev), _dicts(B, 1, prev)
    with pytest.raises(RuntimeError, match=r"^Invalid Jacobian in Gauss Newton minimization.*\[1\]"):
        group.process_next_frames(da)
    for i in (0, 2):
        alone[i].process_next_frame(db[i])
        np.testing.assert_array_equal(da[i]["odometry_pose"], db[i]["odometry_pose"])
        np.testing.assert_array_equal(da[i]["odometry_pc"], db[i]["odometry_pc"])
    assert "odometry_pose" not in da[1]
    assert len(batched[1].relative_poses) == 1 and len(batched[1].elapsed) == 1
    assert len(batched[0].relative_poses) == 2 and len(batched[0].elapsed) == 2
    # the next frame of the failed sequence runs as on a context that saw the same error alone
    group.process_next_frames(_dicts(B, 2, prev))


def test_constructor_rejections(b200):
    a, b = _algos(b200, 2)
    with pytest.raises(AssertionError, match="twice"):
        b200.ICPFrameToModelBatch([a, a])
    with pytest.raises(AssertionError):
        b200.ICPFrameToModelBatch([])
    (fine,) = _algos(b200, 1, gn_iters=3)
    with pytest.raises(AssertionError, match="max_iters == 1"):
        b200.ICPFrameToModelBatch([a, fine])
    (proj,) = _algos(b200, 1, local_map=b200.ProjectiveLocalMapConfig(local_map_size=4))
    with pytest.raises(AssertionError, match="kd-tree"):
        b200.ICPFrameToModelBatch([proj, b])
    b.ctx.cfg.device = 1
    with pytest.raises(AssertionError, match="one CUDA device"):
        b200.ICPFrameToModelBatch([a, b])
    with pytest.raises(AssertionError, match="ICPFrameToModel"):
        b200.ICPFrameToModelBatch([a, object()])


def test_bad_inputs_leave_every_sequence_untouched(b200):
    batched = _algos(b200, 2)
    group = b200.ICPFrameToModelBatch(batched)
    with pytest.raises(AssertionError):
        group.process_next_frames([{"numpy_pc": _frame(0, 0)}, {"wrong_key": _frame(1, 0)}])
    with pytest.raises(AssertionError):
        group.process_next_frames([{"numpy_pc": _frame(0, 0)}, {"numpy_pc": np.zeros((5, 4), np.float32)}])
    with pytest.raises(AssertionError):
        group.process_next_frames([{"numpy_pc": _frame(0, 0)}])
    assert all(a.ctx.frame_calls == 0 and a.relative_poses == [] for a in batched)


def test_failed_call_still_records_the_sequences_that_completed(b200):
    """A failure that is not one sequence's singular solve (status PLS_E_CUDA for sequence 1): sequence 0, whose frame
    completed, still gets its outputs and its pose list stays in step with its context; then the error is raised."""
    batched = _algos(b200, 2)
    group = b200.ICPFrameToModelBatch(batched)
    batched[1].ctx.failing_calls[0] = 2   # PLS_E_CUDA
    dd = _dicts(2, 0, [None] * 2)
    with pytest.raises(RuntimeError, match="status 2"):
        group.process_next_frames(dd)
    assert len(batched[0].relative_poses) == 1 and batched[0].elapsed and batched[0].ctx.frame_calls == 1
    assert batched[1].relative_poses == [] and batched[1].elapsed == []
