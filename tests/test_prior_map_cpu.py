"""Localisation against a prior map, without a GPU: the host model (oracle/prior_map_oracle.py) against the reference's
goldens (tests/golden/prior_map.npz), and the host logic of the Python mirrors -- argument checks, the errors the
reference raises, get_last_frame's slicing and the shapes of register_new_frame_hypotheses -- over a stand-in context
that keeps the map in the host model."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle.prior_map_oracle import PriorMapOracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prior_map.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def _array(address, shape, dtype):
    count = int(np.prod(shape))
    buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(address)
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


class HostContext:
    """Answers the kd-map entry points the mirrors call from a PriorMapOracle (the library needs a GPU)."""

    def __init__(self, local_map_size=3, max_num_alignments=5):
        class Cfg:
            pass
        self.cfg = Cfg()
        self.cfg.local_map_size = local_map_size
        self.map = PriorMapOracle(local_map_size)
        self.calls = []
        self.M = max_num_alignments

    def call(self, name, *a):
        self.calls.append(name)
        if name == "pls_kdmap_set_points":
            addr, is64, n = a
            self.map.set_map_pointcloud(_array(addr, (n, 3), np.float64 if is64 else np.float32) if n else np.zeros((0, 3)))
        elif name == "pls_kdmap_update_points":
            rel, pts, n = a
            self.map.update(_array(rel, (4, 4), np.float32), _array(pts, (n, 3), np.float32) if pts else None)
        elif name == "pls_kdmap_size":
            a[0]._obj.value = 0 if self.map.rows is None else self.map.rows.shape[0]
        elif name == "pls_kdmap_points":
            _array(a[0], self.map.rows.shape, np.float32)[:] = self.map.rows
        elif name == "pls_kdmap_frames":
            c = self.map.counts
            _array(a[0], (len(c),), np.int64)[:] = c
            a[1]._obj.value = len(c)
        elif name == "pls_register_hypotheses":
            pts, n, T0, B, T, params, losses, iters, status = a
            _array(T, (B, 16), np.float32)[:] = _array(T0, (B, 16), np.float32)
            _array(params, (B, 6), np.float32)[:] = np.arange(B)[:, None]
            _array(losses, (B, self.M), np.float32)[:] = np.arange(self.M)
            _array(iters, (B,), np.int32)[:] = np.arange(B) % self.M + 1
            _array(status, (B,), np.int32)[:] = 0
        else:
            raise AssertionError(f"unexpected call {name}")


def kd_map(ctx):
    import pylidar_slam_b200 as b200
    return b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=ctx.cfg.local_map_size), ctx=ctx)


def test_oracle_eviction_matches_the_reference(g):
    m = PriorMapOracle(3)
    m.set_map_pointcloud(g["pm_ev_prior"])
    with pytest.raises(IndexError):
        m.get_last_frame()
    for k in range(6):
        m.update(g[f"pm_ev_rel_{k}"], g[f"pm_ev_pts_{k}"])
        np.testing.assert_array_equal(m.rows, g[f"pm_ev_map_{k}"])
        assert m.counts == list(g[f"pm_ev_counts_{k}"])
        np.testing.assert_array_equal(m.get_last_frame(), g[f"pm_ev_last_{k}"])
    # the first eviction (update 3) dropped frame 0's row count from the front: prior rows, while frame 0 stays
    c0 = int(g["pm_ev_counts_2"][0])
    prior = g["pm_ev_prior"]
    assert c0 < prior.shape[0]
    moved = prior
    for k in range(4):
        inv = np.linalg.inv(g[f"pm_ev_rel_{k}"])
        moved = np.einsum("ij,nj->ni", inv[:3, :3], moved) + inv[:3, 3].reshape(1, 3)
    np.testing.assert_array_equal(g["pm_ev_map_3"][:prior.shape[0] - c0], moved[c0:])
    # the frame of NaN rows only (k = 3) held zero rows, and get_last_frame then returned the whole map
    assert g["pm_ev_counts_3"][-1] == 0 and g["pm_ev_last_3"].shape == g["pm_ev_map_3"].shape


def test_mirror_get_last_frame_and_counts_follow_the_reference(g):
    ctx = HostContext(3)
    lm = kd_map(ctx)
    lm.set_map_pointcloud(g["pm_ev_prior"])
    assert lm.frame_counts() == []
    with pytest.raises(IndexError, match=str(g["pm_err_last_after_set"][1])):
        lm.get_last_frame()
    for k in range(6):
        lm.update(g[f"pm_ev_rel_{k}"], new_pc_data=g[f"pm_ev_pts_{k}"])
        last = lm.get_last_frame()
        assert isinstance(last, torch.Tensor)
        np.testing.assert_array_equal(last.numpy(), g[f"pm_ev_last_{k}"])
        assert lm.frame_counts() == list(g[f"pm_ev_counts_{k}"])


def test_mirror_argument_checks(g):
    ctx = HostContext()
    lm = kd_map(ctx)
    cloud = g["pm_cloud32"]
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        lm.set_map_pointcloud(cloud[:, :2])
    with pytest.raises(TypeError, match=str(g["pm_err_torch_cloud"][1])):
        lm.set_map_pointcloud(torch.from_numpy(cloud))
    assert ctx.calls == []  # refused before the library is called
    # normals of the wrong shape: the map is already set when the reference's check fails, and searches work
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        lm.set_map_pointcloud(cloud, normals=np.zeros((cloud.shape[0], 4), np.float32))
    assert ctx.calls == ["pls_kdmap_set_points"] and not getattr(ctx, "kd_given_normals", False)
    # normals of the right shape: every search with normals raises the reference's IndexError until the next update
    lm.set_map_pointcloud(cloud, normals=np.zeros_like(cloud))
    kind, msg = g["pm_err_given_normals"]
    assert kind == "IndexError"
    with pytest.raises(IndexError, match=msg):
        lm.nearest_neighbor_search(g["pm_queries"])
    lm.update(np.eye(4, dtype=np.float32))
    assert not ctx.kd_given_normals
    lm.set_map_pointcloud(cloud, normals=np.zeros_like(cloud))
    # the odometry sharing the context refuses to register on such a map, as the reference's search would
    odo = _odometry(ctx)
    with pytest.raises(IndexError, match=msg):
        odo.register_new_frame_hypotheses(g["pm_reg_scan"], g["pm_reg_T0"])
    with pytest.raises(IndexError, match=msg):
        odo.register_new_frame(g["pm_reg_scan"], g["pm_reg_T0"][0])


def _odometry(ctx):
    from pylidar_slam_b200.odometry import ICPFrameToModel, ICPFrameToModelConfig
    odo = ICPFrameToModel.__new__(ICPFrameToModel)
    odo.ctx = ctx
    odo.config = ICPFrameToModelConfig(max_num_alignments=ctx.M)
    return odo


@pytest.mark.parametrize("B", [1, 3, 65])
def test_hypotheses_shapes(g, B):
    ctx = HostContext(max_num_alignments=5)
    odo = _odometry(ctx)
    rng = np.random.RandomState(B)
    T0 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    T0[:, :3, 3] = rng.randn(B, 3)
    for init in (T0, torch.from_numpy(T0)):
        params, T, losses, iters = odo.register_new_frame_hypotheses(g["pm_reg_scan"], init)
        assert params.shape == (B, 6) and T.shape == (B, 4, 4) and iters.shape == (B,)
        np.testing.assert_array_equal(T, T0)
        assert len(losses) == B and [len(l) for l in losses] == list(iters)
        assert odo.last_hypotheses_status.shape == (B,)
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        odo.register_new_frame_hypotheses(g["pm_reg_scan"], T0[:, :3])
    with pytest.raises(AssertionError, match="BAD TENSOR SHAPE"):
        odo.register_new_frame_hypotheses(g["pm_reg_scan"][:, :2], T0)


def test_goldens_are_self_consistent(g):
    """The reference's registrations from several initial estimates converge on the map they were set on."""
    assert g["pm_reg_T0"].shape[0] == g["pm_reg_T"].shape[0] == g["pm_reg_iters"].shape[0] >= 3
    for b in range(g["pm_reg_T"].shape[0]):
        it = int(g["pm_reg_iters"][b])
        assert np.all(np.isfinite(g["pm_reg_losses"][b, :it])) and np.all(np.isnan(g["pm_reg_losses"][b, it:]))
    assert g["pm_proj_last"].shape == (g["pm_proj_v1"].shape[1] * g["pm_proj_v1"].shape[2], 3)
    np.testing.assert_array_equal(g["pm_proj_last"], np.transpose(g["pm_proj_v1"], (1, 2, 0)).reshape(-1, 3))
