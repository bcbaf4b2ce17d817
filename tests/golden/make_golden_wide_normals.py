"""Goldens of the kd map's normals from more than 31 neighbours, from the UNMODIFIED reference under
oracle/ref_shims.py.  Build container only:

    python tests/golden/make_golden_wide_normals.py -> wide_normals.npz
    python tests/golden/make_golden_wide_normals.py --check   # regenerate in memory, compare with the committed file
                                                              # bit for bit, write nothing

Cases, at num_neighbors_normals k in KS:
  wn_map, wn_queries        a synthetic map (three scans in the frame of scan 0) and queries near it
  wn_nb_<k>, wn_nrm_<k>     KdTreeLocalMap.nearest_neighbor_search (local_map.py:372-422): neighbours and normals
  wn_pose_<k>               ICPFrameToModel.get_relative_poses() [F,4,4] after process_next_frame on F frames of the
                            synthetic stream (grid-sampled scans, the kd map, point-to-plane Gauss-Newton)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import icp_oracle as orc  # noqa: E402
from oracle import ref_shims  # noqa: E402
from pylidar_slam_b200 import synthetic as syn  # noqa: E402

torch.set_num_threads(1)
ns = ref_shims.load_reference(kdtree_workers=-1)
pose = ns.pose.Pose("euler")
KS = (32, 64, 255)
H, W = 32, 512        # scans of the map and of the stream
FRAMES = 4
VOXEL = 0.4


def frame_points(k):
    """Scan k of the synthetic sequence, float32, in the frame of scan 0 (ground-truth poses)."""
    pc = syn.scan(k, H, W).astype(np.float64)
    T = syn.gt_pose(k).astype(np.float64)
    return (pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def stream_poses(k):
    proj = ns.projection.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = ns.icp.ICPFrameToModelConfig(
        local_map=ns.local_map.KdTreeLocalMapConfig(local_map_size=4, num_neighbors_normals=k),
        alignment=ns.alignment.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                                      max_iters=1)),
        max_num_alignments=8, data_key="numpy_pc")
    algo = ns.icp.ICPFrameToModel(cfg, projector=proj, pose=pose, device=torch.device("cpu"))
    algo.init()
    for f in range(FRAMES):
        s, _ = orc.grid_sample(syn.scan(f, H, W), VOXEL)
        algo.process_next_frame({"numpy_pc": np.ascontiguousarray(s, np.float32)})
    return np.asarray(algo.get_relative_poses(), np.float32)


def main():
    out = {}
    m = np.ascontiguousarray(np.concatenate([frame_points(k)[::2] for k in (0, 2, 4)]))
    rng = np.random.RandomState(5)
    q = m[rng.choice(len(m), 3000, replace=False)] + rng.normal(0, 0.05, (3000, 3)).astype(np.float32)
    out.update(wn_map=m, wn_queries=q)
    for k in KS:
        lm = ns.local_map.KdTreeLocalMap(ns.local_map.KdTreeLocalMapConfig(local_map_size=1, num_neighbors_normals=k))
        lm.init()
        lm.set_map_pointcloud(m)
        r = lm.nearest_neighbor_search(q)
        out[f"wn_nb_{k}"], out[f"wn_nrm_{k}"] = np.asarray(r.neighbor_points), np.asarray(r.neighbor_normals)
        out[f"wn_pose_{k}"] = stream_poses(k)

    path = os.path.join(HERE, "wide_normals.npz")
    if "--check" in sys.argv[1:]:
        old = np.load(path)
        bad = sorted(set(old.files) ^ set(out))
        for key in sorted(set(old.files) & set(out)):
            a, b = old[key], np.asarray(out[key])
            if a.shape != b.shape or a.dtype != b.dtype or not np.array_equal(a, b, equal_nan=a.dtype.kind in "fc"):
                bad.append(key)
        print(f"{len(out)} arrays regenerated, {len(bad)} differ from {os.path.basename(path)}", *bad[:20])
        sys.exit(1 if bad else 0)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes", {key: v.shape for key, v in out.items()})


if __name__ == "__main__":
    main()
