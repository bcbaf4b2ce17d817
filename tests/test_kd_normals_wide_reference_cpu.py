"""The reference of the kd map's wide normals (32 <= k <= 255), pinned on the CPU against the UNMODIFIED reference's
KdTreeLocalMap under oracle/ref_shims.py (skipped where the reference checkout does not exist):

  * oracle knn_lists gives the (k+1)-NN lists the reference's own search gives, wherever the order is not ambiguous;
  * reference_covs over the reference's lists are its float32 moments bit for bit: its SVD of them returns the
    reference's normals bit for bit;
  * numpy's `.mean(axis=1)` over [n, k, 3, 3] still sums sequentially (not pairwise) at every such k: it equals the
    sequential float32 sum over entries 1..k divided by k, the order warp_second_moments_wide sums in.
"""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import kd_icp_reference as ref
from oracle import kd_normals_scenes as scenes
from oracle import ref_shims

pytestmark = pytest.mark.skipif(not os.path.isdir(ref_shims.REFERENCE_ROOT), reason="needs the reference checkout")

KS = [32, 33, 63, 64, 65, 127, 128, 200, 255]
CENTRES = 400
_SCENES = {}


@pytest.fixture(scope="module")
def ns():
    return ref_shims.load_reference()


def _scene(name):
    if name not in _SCENES:
        m, _ = scenes.build(name)
        rng = np.random.RandomState(len(m))
        sub = np.sort(rng.choice(len(m), min(len(m), CENTRES), replace=False))
        _SCENES[name] = (m, sub, ref.kernel_sort_positions(m), cKDTree(m.astype(np.float64)))
    return _SCENES[name]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", scenes.SCENES)
def test_wide_lists_and_moments_are_the_references(ns, name, k):
    m, sub, positions, tree = _scene(name)
    lm = ns.local_map.KdTreeLocalMap(ns.local_map.KdTreeLocalMapConfig(local_map_size=1, num_neighbors_normals=k))
    lm.init()
    lm.set_map_pointcloud(m)
    res = lm.nearest_neighbor_search(m[sub])
    nb, nrm = np.asarray(res.neighbor_points), np.asarray(res.neighbor_normals)
    assert np.array_equal(nb, m[sub])
    # the reference's own lists: its kd-tree query of the matched points (pykdtree, served by cKDTree in the shims)
    _, match = cKDTree(m).query(m[sub])
    _, lists = cKDTree(m).query(m[match], k=k + 1)
    covs = ref.reference_covs(m, match, lists, k)
    assert covs.dtype == np.float32
    assert np.array_equal(np.linalg.svd(covs)[2][:, 2, :].view(np.uint32), nrm.view(np.uint32)), (name, k)
    # sequential float32 sums in list order, one division by k
    d = m[lists[:, 1:]] - m[match][:, None, :]
    acc = np.zeros((len(match), 3, 3), np.float32)
    for j in range(k):
        acc = acc + d[:, j, :, None] * d[:, j, None, :]
    assert np.array_equal(acc / np.float32(k), covs), (name, k)
    # the oracle's lists are the reference's wherever the float32 order is not ambiguous: the same entries, except that
    # among points at exactly the same distance the kernel takes the lower sorted position and the reference's tree any
    o_idx, _, o_d2, amb = ref.knn_lists(m, m[match], k, positions, tree)
    sure = ~amb
    assert sure.mean() > 0.5, (name, k, sure.mean())
    diff = m[lists].astype(np.float64) - m[match][:, None, :].astype(np.float64)
    r_d2 = np.sort((diff * diff).sum(-1), 1)
    assert np.array_equal(o_d2[sure], r_d2[sure]), (name, k)
    same = sure & (np.sort(o_idx, 1) == np.sort(lists, 1)).all(1)
    tied = sure & ~same
    assert not tied.any() or name == "ties", (name, k, int(tied.sum()))
