"""Goldens of many scans registered against one prior map, from the UNMODIFIED reference under oracle/ref_shims.py.
Build container only:

    python tests/golden/make_golden_register_scans.py -> register_scans.npz
    python tests/golden/make_golden_register_scans.py --check   # regenerate in memory, compare with the committed file
                                                                # bit for bit, write nothing

The reference has no call for several scans: ICPFrameToModel.register_new_frame (icp_odometry.py:248-299) runs once per
registration on a map set by KdTreeLocalMap.set_map_pointcloud (local_map.py:289-299), which registering leaves as it is.
  rs_cloud                     the map
  rs_scan_{s}                  three scans of different sizes (s = 0, 1, 2)
  rs_scan_of, rs_T0            six registrations, two initial estimates per scan
  rs_T, rs_params, rs_losses,  each registration's pose, parameters, losses (NaN past its iterations) and iterations
  rs_iters
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from pylidar_slam_b200 import synthetic as syn  # noqa: E402

torch.set_num_threads(1)
ns = ref_shims.load_reference(kdtree_workers=-1)
pose = ns.pose.Pose("euler")
H, W = 16, 256
MAX_ALIGN = 12


def frame_points(k):
    """Scan k of the synthetic sequence, float32, in the frame of scan 0 (ground-truth poses)."""
    pc = syn.scan(k, H, W).astype(np.float64)
    T = syn.gt_pose(k).astype(np.float64)
    return (pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def main():
    out = {}
    cloud = np.ascontiguousarray(np.concatenate([frame_points(k)[::3] for k in (0, 3, 6)]))
    scans = [np.ascontiguousarray(frame_points(k)[::step]) for k, step in ((2, 2), (4, 5), (5, 9))]
    proj = ns.projection.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = ns.icp.ICPFrameToModelConfig(
        local_map=ns.local_map.KdTreeLocalMapConfig(local_map_size=20),
        alignment=ns.alignment.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                                      max_iters=1)),
        max_num_alignments=MAX_ALIGN, data_key="numpy_pc", threshold_delta_pose=1e-4)
    algo = ns.icp.ICPFrameToModel(cfg, projector=proj, pose=pose, device=torch.device("cpu"))
    algo.init()
    algo.local_map.set_map_pointcloud(cloud)
    scan_of = np.array([0, 1, 2, 2, 0, 1], np.int32)
    offsets = np.array([[0, 0, 0, 0, 0, 0], [0.3, -0.2, 0.05, 0, 0, 0.03], [-0.4, 0.3, 0, 0.01, -0.01, -0.05],
                        [0.2, 0.5, 0.05, 0, 0, 0.06], [0.6, 0.6, 0.1, 0, 0, 0.08], [-0.3, -0.5, 0, 0, 0.01, -0.04]],
                       np.float32)
    T0s = pose.build_pose_matrix(torch.from_numpy(offsets)).numpy().astype(np.float32)
    P, Ts, L, its = [], [], [], []
    for s, T0 in zip(scan_of, T0s):
        p, T, ls = algo.register_new_frame(torch.from_numpy(scans[s]), initial_estimate=torch.from_numpy(T0).unsqueeze(0))
        P.append(np.asarray(p, np.float32).reshape(6))
        Ts.append(np.asarray(T, np.float32).reshape(4, 4))
        L.append([float(x) for x in ls] + [np.nan] * (MAX_ALIGN - len(ls)))
        its.append(len(ls))
    out.update(rs_cloud=cloud, rs_scan_of=scan_of, rs_T0=T0s, rs_params=np.stack(P), rs_T=np.stack(Ts),
               rs_losses=np.asarray(L, np.float64), rs_iters=np.asarray(its, np.int64))
    out.update({f"rs_scan_{s}": scan for s, scan in enumerate(scans)})

    path = os.path.join(HERE, "register_scans.npz")
    if "--check" in sys.argv[1:]:
        old = np.load(path)
        bad = sorted(set(old.files) ^ set(out))
        for k in sorted(set(old.files) & set(out)):
            a, b = old[k], np.asarray(out[k])
            if a.shape != b.shape or a.dtype != b.dtype or not np.array_equal(a, b, equal_nan=a.dtype.kind in "fc"):
                bad.append(k)
        print(f"{len(out)} arrays regenerated, {len(bad)} differ from {os.path.basename(path)}", *bad[:20])
        sys.exit(1 if bad else 0)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes", {k: v.shape for k, v in out.items()})
    print("iterations", its)


if __name__ == "__main__":
    main()
