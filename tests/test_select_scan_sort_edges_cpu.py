"""The edges test_select_scan_sort_edges_gpu.py runs at, read from the CUDA sources (so they move when the code does),
and the voxel coordinates its hash cases are built from, against the oracle's wrapping int64 hash."""
import os
import re

import numpy as np

from conftest import ROOT
from oracle import icp_oracle as orc
from test_select_scan_sort_edges_gpu import (COMPACT, EPOCH_CYCLE, HASH_VOXEL, NUM_SMS, SEL_MAX_N, SIZES, TILE, _lattice,
                                             case_points, float32_carries, half_points, hash_cases, int64_wrap)

CSRC = os.path.join(ROOT, "pylidar_slam_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(rf"constexpr\s+(?:int|int64_t|unsigned long long)\s+{name}\s*=\s*(\d+)\s*;", text)
    assert m, name
    return int(m.group(1))


def _tile(text, prefix):
    assert re.search(rf"constexpr\s+int\s+{prefix}_TILE\s*=\s*{prefix}_THREADS\s*\*\s*{prefix}_ITEMS\s*;", text), prefix
    return _const(text, f"{prefix}_THREADS") * _const(text, f"{prefix}_ITEMS")


def test_edge_sizes_follow_the_sources():
    sel, prim, internal = _source("select_device.cuh"), _source("primitives.cu"), _source("internal.cuh")
    factor = re.search(r"SEL_MAX_N\s*=\s*\(int64_t\)SEL_TILE\s*\*\s*(\d+)\s*\*\s*kNumSMs\s*;", sel)
    sms = re.search(r"constexpr\s+int\s+kNumSMs\s*=\s*(\d+)\s*;", internal)
    assert factor and sms
    assert NUM_SMS == int(sms.group(1))
    assert TILE == _tile(sel, "SEL") == _tile(prim, "SCAN") == _tile(prim, "SORT")
    assert SEL_MAX_N == TILE * int(factor.group(1)) * NUM_SMS == 1_081_344
    epoch_bits = re.search(r"SEL_EPOCH_BITS\s*=\s*(\d+)", sel)
    assert epoch_bits and EPOCH_CYCLE == 2 ** int(epoch_bits.group(1)) - 1
    assert "s.epoch = 1;" in sel                                 # after a wrap the next launch is epoch 1
    assert COMPACT == 2 ** (_const(_source("grid_sample.cu"), "GS_COMPACT_BITS") - 1)
    # the grid sample leaves the selection above SEL_MAX_N, the kd frame input's fused selection likewise
    assert "if (n <= SEL_MAX_N) {" in _source("grid_sample.cu")
    assert "n <= SEL_MAX_N" in _source("odometry.cu")
    for k in (1, 2):
        assert {k * TILE - 1, k * TILE, k * TILE + 1} <= set(SIZES)
    assert {SEL_MAX_N - 1, SEL_MAX_N, SEL_MAX_N + 1} <= set(SIZES) and max(SIZES) > 2 * SEL_MAX_N


def test_hash_cases_hit_their_hashes():
    """Each constructed case: the integer hash value it was solved for, the oracle's int64 hash equal to that value
    wrapped modulo 2^64 (numba's arithmetic), and points that round back to its voxel coordinates in every dtype the
    GPU test feeds it in."""
    cases = hash_cases()
    true = {name: [orc.HASH_PX * x + orc.HASH_PY * y + orc.HASH_PZ * z for x, y, z in c] for name, c in cases.items()}
    assert true["compact_min"] == [-COMPACT] and true["compact_max"] == [COMPACT - 1]
    assert true["first_repeat"] == [COMPACT] and true["first_repeat_below"] == [-COMPACT - 1]
    assert true["wrap_up"][0] > 2 ** 63 - 1 and true["wrap_down"][0] < -2 ** 63
    assert true["collision"][0] == true["collision"][1] and cases["collision"][0] != cases["collision"][1]
    assert true["collision_wrap"] == [0, 2 ** 64]
    for name, coords in cases.items():
        h = orc.voxel_hashes(np.array(coords, np.int64))
        assert h.tolist() == [int64_wrap(v) for v in true[name]], name
        for dtype in (np.float32, np.float64) if float32_carries(coords) else (np.float64,):
            pts = case_points(coords, dtype)
            assert np.array_equal(orc.voxel_coords(pts, HASH_VOXEL), np.repeat(np.array(coords), 3, axis=0)), (name, dtype)
    assert sum(float32_carries(c) for c in cases.values()) == 4      # the compact-key bounds run in float32 too
    for dtype in (np.float32, np.float64):
        for pts, voxel in zip(*[iter(half_points(dtype))] * 2):
            q = pts.astype(np.float64) / voxel
            assert (q - np.floor(q) == 0.5).all()                    # exactly on the half
            c = orc.voxel_coords(pts, voxel)
            assert (c == 2 * np.round(q / 2)).all() and (c < 0).any()  # to even


def test_lattice_hashes_are_distinct():
    """The 'every point in its own voxel' clouds: the box the largest one draws from (every smaller cloud draws from a
    box inside it) has distinct hashes."""
    s = int(np.ceil(max(SIZES) ** (1 / 3))) // 2 + 1
    full = np.stack(np.meshgrid(*[np.arange(-s, s)] * 3, indexing="ij"), -1).reshape(-1, 3)
    assert full.shape[0] >= max(SIZES) and _lattice(max(SIZES), np.random.RandomState(0)).shape[0] == max(SIZES)
    assert np.unique(orc.voxel_hashes(full)).shape[0] == full.shape[0]
