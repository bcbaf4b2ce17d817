"""ICPFrameToModel.register_new_frame_hypotheses on a projective configuration, without a GPU: over a stand-in context
that records what the mirror passes to pls_register_hypotheses and answers with known values, the mirror passes the
scan, the T0s and B, accepts torch T0s, reshapes every output, logs singular hypotheses, and refuses malformed scans or
T0s before the library is called."""
import ctypes as C
import logging

import numpy as np
import pytest
import torch

from pylidar_slam_b200 import _lib


def _array(address, shape, dtype):
    count = int(np.prod(shape))
    buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(address)
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


class ProjectiveStandIn:
    """Answers pls_register_hypotheses as a projective context would be asked it; hypothesis b is singular if
    b % 4 == 3."""

    def __init__(self, max_num_alignments=6):
        class Cfg:
            pass
        self.cfg = Cfg()
        self.cfg.local_map_type = _lib.MAP_PROJECTIVE
        self.cfg.height, self.cfg.width = 64, 720
        self.M = max_num_alignments
        self.calls = []

    def call(self, name, *a):
        assert name == "pls_register_hypotheses", name
        pts, n, T0, B, T, params, losses, iters, status = a
        self.calls.append(dict(scan=_array(pts, (n, 3), np.float32).copy(), T0=_array(T0, (B, 16), np.float32).copy(),
                               B=B, outputs=[T, params, losses, iters, status]))
        _array(T, (B, 16), np.float32)[:] = _array(T0, (B, 16), np.float32) * 2
        _array(params, (B, 6), np.float32)[:] = np.arange(B)[:, None]
        _array(losses, (B, self.M), np.float32)[:] = np.arange(self.M) + 0.5
        _array(iters, (B,), np.int32)[:] = np.arange(B) % self.M + 1
        _array(status, (B,), np.int32)[:] = np.where(np.arange(B) % 4 == 3, _lib.PLS_E_SINGULAR, _lib.PLS_OK)


def _odometry(ctx):
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = ctx
    odo.config = ICPFrameToModelConfig(max_num_alignments=ctx.M,
                                       local_map=dict(type="projective_local_map", local_map_size=20))
    return odo


def _inputs(B, n=500, seed=0):
    rng = np.random.RandomState(seed)
    scan = rng.uniform(-20, 20, (n, 3)).astype(np.float64)   # float64: the mirror rounds it to float32
    T0 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    T0[:, :3, 3] = rng.randn(B, 3)
    return scan, T0


@pytest.mark.parametrize("B", [1, 4, 65])
def test_shapes_pointers_and_values(B):
    ctx = ProjectiveStandIn()
    odo = _odometry(ctx)
    scan, T0 = _inputs(B)
    for init in (T0, torch.from_numpy(T0)):
        params, T, losses, iters = odo.register_new_frame_hypotheses(scan, init)
        rec = ctx.calls[-1]
        assert rec["B"] == B
        np.testing.assert_array_equal(rec["scan"], scan.astype(np.float32))
        np.testing.assert_array_equal(rec["T0"], T0.reshape(B, 16))
        assert len(set(rec["outputs"])) == 5 and all(rec["outputs"])   # five distinct, non-null output buffers
        assert params.shape == (B, 6) and T.shape == (B, 4, 4) and iters.shape == (B,)
        np.testing.assert_array_equal(T, T0 * 2)
        np.testing.assert_array_equal(params[:, 0], np.arange(B))
        assert [len(l) for l in losses] == list(iters)
        assert all(list(l) == list(np.arange(len(l)) + 0.5) for l in losses)
        np.testing.assert_array_equal(odo.last_hypotheses_status == _lib.PLS_E_SINGULAR, np.arange(B) % 4 == 3)
    assert len(ctx.calls) == 2


def test_singular_hypotheses_are_logged(caplog):
    ctx = ProjectiveStandIn()
    odo = _odometry(ctx)
    scan, T0 = _inputs(8)
    with caplog.at_level(logging.ERROR):
        odo.register_new_frame_hypotheses(scan, T0)
    assert "Invalid Jacobian" in caplog.text and "[3, 7]" in caplog.text
    caplog.clear()
    scan, T0 = _inputs(3)
    with caplog.at_level(logging.ERROR):
        odo.register_new_frame_hypotheses(scan, T0)
    assert "Invalid Jacobian" not in caplog.text


@pytest.mark.parametrize("bad", ["scan_2d", "scan_4cols", "T0_3x4", "T0_flat"])
def test_malformed_inputs_are_refused_before_the_library(bad):
    ctx = ProjectiveStandIn()
    odo = _odometry(ctx)
    scan, T0 = _inputs(3)
    if bad == "scan_2d":
        scan = scan[:, :2]
    elif bad == "scan_4cols":
        scan = np.concatenate([scan, scan[:, :1]], 1)
    elif bad == "T0_3x4":
        T0 = T0[:, :3]
    else:
        T0 = T0.reshape(3, 16)
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        odo.register_new_frame_hypotheses(scan, T0)
    assert ctx.calls == []
