"""The kd map's normals against the reference's own float32 moments, for every k the map accepts and every path of the
(k+1)-NN selection (kdmap_device.cuh: warp_knn, warp_second_moments).

Per scene (oracle/kd_normals_scenes.py) and k:
  * lists: pls_kdmap_knn at every map point and at off-map probes equals oracle knn_lists -- same entries in the same
    (d^2, sorted position) order where the query is not ambiguous, the same float64 distances within the float32
    band where it is; every float32 d^2 within float32 error; every sorted position that of kernel_sort_positions;
  * normals: pls_kdmap_nn_search at the map points returns, for each, the normal kd_normals_warp_kernel computed.  It
    is within tight_normal_bound of the float64 eigenvector of reference_covs (the reference's float32 expression)
    over the reference's list, and of the GPU's own list -- so a list error and a moments error are told apart;
  * paths: the level-0 block of every query is restated (level0_paths) and the selection paths it implies are
    counted and checked against the PLS_KD_STATS counters of the same search.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import kd_icp_reference as ref
from oracle import kd_normals_scenes as scenes

pytestmark = pytest.mark.gpu

KS = [3, 4, 9, 10, 11, 15, 16, 17, 30, 31]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        m, probes = scenes.build(name)
        _SCENES[name] = (m, probes, ref.kernel_sort_positions(m), cKDTree(m.astype(np.float64)))
    return _SCENES[name]


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("PLS_KD_STATS", "1")  # read when a map is (re)initialised: every context here counts its searches
        yield _lib


def _context(lib, k):
    return lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=1, num_neighbors_normals=k)


def _insert(lib, ctx, m):
    ctx.call("pls_kdmap_update_points", lib.ptr(np.eye(4, dtype=np.float32)), lib.ptr(m), m.shape[0])


def _stats(lib, ctx):
    out = np.zeros(16, np.uint64)
    ctx.call("pls_kdmap_stats", lib.ptr(out))
    return out.astype(np.int64)


def _knn(lib, ctx, q, k):
    n, K = q.shape[0], k + 1
    idx, d2, pos = np.empty((n, K), np.int64), np.empty((n, K), np.float32), np.empty((n, K), np.int32)
    ctx.call("pls_kdmap_knn", lib.ptr(np.ascontiguousarray(q)), n, k, lib.ptr(idx), lib.ptr(d2), lib.ptr(pos))
    return idx, d2, pos


def check_lists(m, positions, tree, q, k, idx, d2, pos, tag=""):
    """The GPU lists of queries q against knn_lists.  Returns the reference (idx, ambiguous)."""
    r_idx, r_pos, r_d2, amb = ref.knn_lists(m, q, k, positions, tree)
    valid = idx >= 0
    assert np.array_equal(valid, r_idx >= 0), (tag, "list lengths")
    # every entry: its sorted position is the emulated one, its float32 d^2 is that of its point
    assert np.array_equal(np.where(valid, positions[np.maximum(idx, 0)], -1), pos), (tag, "sorted positions")
    diff = m[np.maximum(idx, 0)].astype(np.float64) - q[:, None, :].astype(np.float64)
    g64 = (diff * diff).sum(-1)
    err = np.abs(d2.astype(np.float64) - g64)
    assert (err[valid] <= ref.D2_REL * g64[valid] + 1e-45).all(), (tag, "float32 d^2")
    # unambiguous queries: the same list in the same order
    bad = ~amb & (idx != r_idx).any(1)
    assert not bad.any(), (tag, "lists differ", int(bad.sum()), np.nonzero(bad)[0][:5])
    # ambiguous ones: distinct entries whose float64 distances are the reference's within the band
    s = np.sort(np.where(valid, idx, -1 - np.arange(idx.shape[1])), 1)
    assert (s[:, 1:] != s[:, :-1]).all(), (tag, "repeated entry")
    gap = np.abs(np.where(valid, g64, 0) - np.where(valid, r_d2, 0))
    assert (gap[amb] <= 2 * ref.D2_REL * np.where(valid, r_d2, 0)[amb] + 1e-45).all(), (tag, "ambiguous lists")
    return r_idx, amb


def check_normals(m, centre, lists, k, nrm, tag=""):
    """GPU normals nrm [n, 3] of map points `centre` against eigh of reference_covs over `lists`.  Returns the largest
    |sin| / bound."""
    covs = ref.reference_covs(m, centre, lists, k).astype(np.float64)
    v = np.linalg.eigh(covs)[1][:, :, 0]
    bound, gap = ref.tight_normal_bound(covs)
    g = nrm.astype(np.float64)
    assert np.isfinite(g).all() and np.abs(np.linalg.norm(g, axis=1) - 1).max() <= 1e-6, (tag, "unit normals")
    sin = np.linalg.norm(np.cross(g, v), axis=1)
    ok = gap > 1e-9
    worst = float((sin[ok] / bound[ok]).max()) if ok.any() else 0.0
    assert worst <= 1.0, (tag, "normals off the tight bound", int((sin[ok] > bound[ok]).sum()), worst)
    return worst


def run_scene(lib, m, probes, positions, tree, k, expect_stats=True, tag=""):
    """Lists, normals and level-0 paths of one map at one k.  Returns the path counts."""
    ctx = _context(lib, k)
    _insert(lib, ctx, m)
    q = np.ascontiguousarray(np.concatenate([m, probes]) if len(probes) else m)
    s0 = _stats(lib, ctx)
    idx, d2, pos = _knn(lib, ctx, q, k)
    s1 = _stats(lib, ctx)
    r_idx, amb = check_lists(m, positions, tree, q, k, idx, d2, pos, tag)
    # level 0 of every query, restated, against the counters of the same search (slots 4 queries, 5 exact at level
    # 0, 6 on to coarser levels, 7 candidates of every level)
    K = k + 1
    kth = np.where(idx[:, K - 1] >= 0, d2[:, K - 1], np.float32(np.inf))
    total, exact = ref.level0_paths(m, q, k, kth)
    ds = s1 - s0
    if expect_stats:
        assert ds[4] == len(q), (tag, ds[4])
        assert ds[5] == exact.sum() and ds[6] == len(q) - exact.sum(), (tag, ds[5], int(exact.sum()))
        assert ds[7] >= total.sum() and (ds[7] == total.sum()) == exact.all(), (tag, ds[7], int(total.sum()))
        # each selection path on its own: the queries exact at level 0 that take it, searched again, scan exactly
        # the candidates the restated block holds
        for path, sel in (("small2", total <= 64), ("small4", (total > 64) & (total <= 128)), ("stream0", total > 128)):
            sel = sel & exact
            if sel.any():
                a = _stats(lib, ctx)
                _knn(lib, ctx, np.ascontiguousarray(q[sel]), k)
                d = _stats(lib, ctx) - a
                assert d[4] == d[5] == sel.sum() and d[7] == total[sel].sum(), (tag, path, d[4:8], int(total[sel].sum()))
    # queries that certainly search past level L: the (k+1)-th distance exceeds the largest exactness radius a level-L
    # block can have, 1.5 cell sides (cell side plus at most half a side of clearance)
    mn, scale = ref.kernel_grid(m)
    dk = np.sqrt(np.where(np.isfinite(kth), kth, np.inf).astype(np.float64))
    beyond = [int((dk > 1.5 * 8 * 2 ** L / float(scale)).sum()) for L in range(4)]
    # the normals kd_normals_warp_kernel computed at every map point (a point is its own match, or its lowest-position
    # duplicate is, which has the same coordinates and list)
    nb, nrm = np.empty_like(m), np.empty_like(m)
    ctx.call("pls_kdmap_nn_search", lib.ptr(m), m.shape[0], lib.ptr(nb), lib.ptr(nrm), None)
    ctx.close()
    assert np.array_equal(nb, m), tag
    M = m.shape[0]
    centre = np.arange(M)
    sure = ~amb[:M]
    worst = check_normals(m, centre[sure], r_idx[:M][sure], k, nrm[sure], tag + " reference lists")
    worst = max(worst, check_normals(m, centre, idx[:M], k, nrm, tag + " own lists"))
    # stream0: more than 128 candidates at level 0, where every key survives (no bound yet): at least four staged
    # batches of 32, so at least three merges through warp_merge_keys
    paths = dict(small2=int((total <= 64).sum()), small4=int(((total > 64) & (total <= 128)).sum()),
                 stream0=int((total > 128).sum()), coarser=int((~exact).sum()), found_lt_K=int((idx < 0).any(1).sum()),
                 ambiguous=int(amb.sum()), beyond=beyond, worst=worst)
    print(tag, paths)
    return paths


# Per scene: the paths it must drive at least `need` queries through, for the k where they can occur.
def _expect(name, k, p):
    need = 200
    if name == "cfg2":
        assert p["small2"] >= need and p["coarser"] >= need
    elif name == "clusters":
        assert p["small4"] >= need and p["stream0"] >= need and p["coarser"] >= need
    elif name == "overflow":
        # level 3's table overflows in this context (local_map_size 1, one frame): queries past level 2 skip it
        from test_kd_overflow_gpu import _table_cells
        m, _ = scenes.build(name)
        levels = _table_cells(m, local_map_size=1)
        assert all(c <= s for c, s in levels[:3]) and levels[3][0] > levels[3][1], levels
        assert p["coarser"] >= need and p["beyond"][2] >= need, p["beyond"]
    elif name == "outlier":
        assert p["small4"] >= need and p["stream0"] >= need
    elif name in ("planar", "ties"):
        assert p["coarser"] >= need
    elif name == "collinear":
        assert p["small2"] >= need and p["coarser"] >= need


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", scenes.SCENES)
def test_lists_and_normals_of_every_map_point(lib, name, k):
    m, probes, positions, tree = _scene(name)
    p = run_scene(lib, m, probes, positions, tree, k, tag=f"{name} k={k}")
    _expect(name, k, p)


@pytest.mark.parametrize("k", KS)
def test_maps_of_at_most_k_plus_one_points(lib, k):
    """M = 1, 2, k and k + 1.  With M <= k the search finds M < k + 1 points: the kernel's moments are those of the
    M - 1 others divided by k (reference_covs' reading of a short list), which the reference leaves undefined (its
    k-NN query asks for more points than the map holds)."""
    for M in sorted({1, 2, k, k + 1}):
        m = scenes.tiny(M)
        probes = np.random.RandomState(M).uniform(-2, 2, (64, 3)).astype(np.float32)
        p = run_scene(lib, m, probes, ref.kernel_sort_positions(m), cKDTree(m.astype(np.float64)), k,
                      tag=f"M={M} k={k}")
        assert (p["found_lt_K"] > 0) == (M < k + 1)


_CELL_SCRIPT = r"""
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
os.environ["PLS_KD_STATS"] = "1"
import numpy as np
from scipy.spatial import cKDTree
from pylidar_slam_b200 import _lib
from oracle import kd_icp_reference as ref, kd_normals_scenes as scenes
import test_kd_normals_knn_gpu as t
for name in ("clusters", "cfg2"):
    m, probes = scenes.build(name)
    pos = ref.kernel_sort_positions(m, {cell})
    tree = cKDTree(m.astype(np.float64))
    for k in (10, 31):
        r_idx, r_pos, r_d2, amb = ref.knn_lists(m, m, k, pos, tree)
        ctx = t._context(_lib, k)
        t._insert(_lib, ctx, m)
        idx, d2, gpos = t._knn(_lib, ctx, np.concatenate([m, probes]), k)
        t.check_lists(m, pos, tree, np.concatenate([m, probes]), k, idx, d2, gpos, f"cell {cell} {{name}} k={{k}}")
        nb, nrm = np.empty_like(m), np.empty_like(m)
        ctx.call("pls_kdmap_nn_search", _lib.ptr(m), m.shape[0], _lib.ptr(nb), _lib.ptr(nrm), None)
        ctx.close()
        t.check_normals(m, np.arange(len(m))[~amb], r_idx[~amb], k, nrm[~amb], f"cell {cell} {{name}} k={{k}}")
print("ok")
"""


@pytest.mark.parametrize("cell", [0.05, 1.0])
def test_cell_target_override(cell):
    """PLS_KD_CELL (read once per process by the index build): other level-0 cell sides, other sort positions and
    block sizes, the same lists and normals."""
    env = dict(os.environ, PLS_KD_CELL=str(cell))
    out = subprocess.run([sys.executable, "-c", _CELL_SCRIPT.format(root=ROOT, cell=cell)], env=env, cwd=ROOT,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout[-3000:] + out.stderr[-3000:]
