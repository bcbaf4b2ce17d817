"""The bucket grid sample (grid_sample.cu: compact keys, n <= SEL_MAX_N) at the edges of its buckets, bit for bit against
the oracle's grid sample.

The path hashes every point, counts 2^16 bins (the top 16 bits of the 40-bit compact key), cuts buckets of whole bins
(bucket b: the bins whose first key ranks in [b, b + 1) * GS_BUCKET_TARGET), sorts each bucket in shared memory when it
holds at most GS_BUCKET_CAP keys and through global memory otherwise, and chains the buckets' sample counts.  The clouds
below are built voxel by voxel from hash values (solve_hash), so the bins and with them the bucket sizes are known: a
bucket of CAP - 1, CAP and CAP + 1 keys, a bin that starts exactly on a bucket boundary, an oversized bucket between two
ordinary ones, every point in one voxel, every point in its own voxel, one point, the compact keys' bounds and the first
hash past them, and the last size on the path next to the first one past it.  One context runs every case, forwards
then backwards, so each call starts from the bins and control words the previous one left behind.
"""
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import icp_oracle as orc
from test_select_scan_sort_edges_gpu import (COMPACT, SEL_MAX_N, _lattice, check_sample, cloud, grid_sample,
                                             grid_sample_staged, hash_cases, solve_hash)

pytestmark = pytest.mark.gpu

VOXEL = 0.5
BIN = 2 ** 24            # hash units per bin


def _const(name):
    with open(os.path.join(ROOT, "pylidar_slam_b200", "csrc", "grid_sample.cu")) as f:
        m = re.search(rf"constexpr\s+uint32_t\s+{name}\s*=\s*(\d+)\s*;", f.read())
    assert m, name
    return int(m.group(1))


TARGET, CAP = _const("GS_BUCKET_TARGET"), _const("GS_BUCKET_CAP")


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def bucket_sizes(pts, voxel):
    """The bucket sizes the device cuts for these points, by the same rule, from the oracle's hashes."""
    h = orc.voxel_hashes(orc.voxel_coords(pts, voxel))
    assert h.min() >= -COMPACT and h.max() < COMPACT
    bins = (h + COMPACT) >> 24
    counts = np.bincount(bins, minlength=2 ** 16)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]])
    return np.bincount(first[bins] // TARGET, minlength=math.ceil(pts.shape[0] / TARGET))


_voxels = {}


def voxel_at(h):
    if h not in _voxels:
        _voxels[h] = solve_hash(h, span=2000)
    return _voxels[h]


def binned_cloud(spec, dtype, seed):
    """spec: per bin (bin number relative to the bin of hash 0, [(hash offset inside the bin, points), ...]); the points
    of a voxel spread inside it, every row in random order."""
    rng = np.random.RandomState(seed)
    coords = []
    for rel, voxels in spec:
        for off, count in voxels:
            coords += [voxel_at(rel * BIN + off)] * count
    c = np.array(coords, np.float64)
    pts = ((c + rng.uniform(-0.4, 0.4, c.shape)) * VOXEL).astype(dtype)
    return pts[rng.permutation(pts.shape[0])]


def split(m, offsets):
    """m points over voxels at the given hash offsets inside one bin (every voxel at least one point)."""
    k = len(offsets)
    return [(o, m // k + (i < m % k)) for i, o in enumerate(offsets)]


IN_BIN = [0, 1, 2, 1000, 2 ** 23, BIN - 1]


def cases(dtype):
    """name -> (points, voxel, the bucket sizes the case is built for: a check of its construction)."""
    out = {}
    for name, m in (("cap_minus_1", CAP - 1), ("cap", CAP), ("cap_plus_1", CAP + 1)):
        # one point in a lower bin, then m - 1 points in one bin: bucket 0 holds both bins, m points
        pts = binned_cloud([(-1, [(5, 1)]), (0, split(m - 1, IN_BIN)), (1, split(700, [3, 77])), (2, split(700, [9]))],
                           dtype, m)
        out[name] = (pts, VOXEL, lambda s, m=m: s[0] == m and s.sum() == m + 1400)
    # a bin that starts exactly at rank TARGET: it opens bucket 1
    pts = binned_cloud([(-1, split(TARGET, [1, 2, 3])), (0, split(500, IN_BIN)), (1, split(600, [11, 2 ** 20]))], dtype, 1)
    out["bin_on_boundary"] = (pts, VOXEL, lambda s: s[0] == TARGET and s[1] == 1100)
    # a bucket past shared memory between two ordinary ones
    pts = binned_cloud([(-3, split(1500, IN_BIN)), (0, [(17, CAP + 900)]), (4, split(800, IN_BIN))], dtype, 2)
    out["oversized_middle"] = (pts, VOXEL, lambda s: (s > CAP).sum() == 1 and s[1] > CAP)
    rng = np.random.RandomState(3)
    out["one_voxel"] = ((rng.uniform(-0.45, 0.45, (3 * CAP, 3)) * VOXEL).astype(dtype), VOXEL,
                        lambda s: s[0] == 3 * CAP)
    pts = ((_lattice(50000, rng) + rng.uniform(-0.4, 0.4, (50000, 3))) * VOXEL).astype(dtype)
    out["all_distinct"] = (pts, VOXEL, lambda s: (s <= CAP).all())
    out["one_point"] = (np.array([[1.25, -3.5, 0.75]], dtype), VOXEL, lambda s: s.tolist() == [1])
    pts = cloud("lidar", 64 * 2048, dtype)
    out["lidar"] = (pts, 0.3, lambda s: (s <= CAP).all() and s.shape[0] > 100)
    return out


def check_both(lib, ctx, pts, voxel, tag):
    _, ref = orc.grid_sample(pts, voxel)
    for api in (grid_sample, grid_sample_staged):
        check_sample(api(lib, ctx, pts, voxel), pts, ref, (tag, api.__name__))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bucket_edges(lib, dtype):
    ctx = lib.Context()
    built = cases(dtype)
    for name, (pts, voxel, shape_ok) in built.items():
        assert shape_ok(bucket_sizes(pts, voxel)), name
    for name in list(built) + list(built)[::-1]:
        pts, voxel, _ = built[name]
        before = ctx.launch_count()
        check_both(lib, ctx, pts, voxel, name)
        # three launches for the sample, one more for the staged call's host copy
        assert ctx.launch_count() - before == 7, name
    ctx.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bucket_path_bound_and_compact_bounds(lib, dtype):
    """SEL_MAX_N points take the bucket path, one more point the radix sort; hashes at the compact keys' bounds stay on
    the bucket path inside a many-bucket cloud, and the first hash past them repeats the call on 64-bit keys."""
    ctx = lib.Context()
    counts = {}
    for n in (SEL_MAX_N, SEL_MAX_N + 1):
        pts = cloud("lidar", n, dtype)
        before = ctx.launch_count()
        s, i = grid_sample(lib, ctx, pts, 0.3)
        counts[n] = ctx.launch_count() - before
        check_sample((s, i), pts, orc.grid_sample(pts, 0.3)[1], n)
    assert counts[SEL_MAX_N] == 3 < counts[SEL_MAX_N + 1], counts
    filler = cloud("lidar", 20000, dtype)
    hc = hash_cases()
    for names, repeat in ((("compact_min", "compact_max"), False), (("compact_min", "compact_max", "first_repeat"), True)):
        coords = [c for nm in names for c in hc[nm]]
        if dtype == np.float32 and max(abs(v) for t in coords for v in t) >= 2 ** 20:
            continue
        c = np.repeat(np.array(coords, np.float64), 3, axis=0)
        case = ((c + np.tile([[0.0, 0.0, 0.0], [0.25, -0.25, 0.125], [-0.25, 0.125, -0.25]], (len(coords), 1)))
                * VOXEL).astype(dtype)
        pts = np.concatenate([filler, case])[np.random.RandomState(5).permutation(filler.shape[0] + case.shape[0])]
        before = ctx.launch_count()
        check_both(lib, ctx, pts, VOXEL, names)
        assert (ctx.launch_count() - before > 7) == repeat, names
    ctx.close()
