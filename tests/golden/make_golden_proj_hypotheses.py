"""Goldens of registering one scan from several initial poses against a projective local map, from the UNMODIFIED
reference under oracle/ref_shims.py.  Build container only:

    python tests/golden/make_golden_proj_hypotheses.py -> proj_hypotheses.npz
    python tests/golden/make_golden_proj_hypotheses.py --check   # regenerate in memory, compare with the committed file
                                                                 # bit for bit, write nothing

The reference's ICPFrameToModel (projective_local_map of size K) has its local map updated with the vertex maps of
synthetic frames 0 .. F-1 (vmaps, with rel_poses: the identity, then the ground-truth relative poses); the scan is frame
F's points, registered with register_new_frame from each of T0s (the ground-truth relative pose and offsets from it).
T, params, losses and iterations of each registration are stored.
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
H, W, K, F, M = 32, 512, 3, 4, 12


def main():
    proj = ns.projection.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0)
    cfg = ns.icp.ICPFrameToModelConfig(
        local_map=ns.local_map.ProjectiveLocalMapConfig(local_map_size=K),
        alignment=ns.alignment.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                                      max_iters=1)),
        max_num_alignments=M, data_key="numpy_pc", threshold_delta_pose=1e-4)
    algo = ns.icp.ICPFrameToModel(cfg, projector=proj, pose=pose, device=torch.device("cpu"))
    algo.init()
    vmaps, rels = [], []
    for k in range(F):
        v = syn.vertex_map_from_scan(syn.scan(k, H, W), H, W).astype(np.float32)
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        algo.local_map.update(torch.from_numpy(rel).unsqueeze(0), new_vertex_map=torch.from_numpy(v))
        vmaps.append(v[0])
        rels.append(rel)
    scan = np.ascontiguousarray(syn.scan(F, H, W), np.float32)
    truth = pose.from_pose_matrix(torch.from_numpy(syn.gt_relative_pose(F).astype(np.float32)).unsqueeze(0))
    offsets = np.array([[0, 0, 0, 0, 0, 0], [0.2, -0.15, 0.02, 0, 0, 0.02], [-0.3, 0.25, 0, 0.005, -0.005, -0.04],
                        [0.4, 0.3, 0.03, 0, 0, 0.06]], np.float32)
    T0s = pose.build_pose_matrix(truth + torch.from_numpy(offsets)).numpy().astype(np.float32)
    P, Ts, L, its = [], [], [], []
    for T0 in T0s:
        p, T, ls = algo.register_new_frame(torch.from_numpy(scan), initial_estimate=torch.from_numpy(T0).unsqueeze(0))
        P.append(np.asarray(p, np.float32).reshape(6))
        Ts.append(np.asarray(T, np.float32).reshape(4, 4))
        L.append([float(x) for x in ls] + [np.nan] * (M - len(ls)))
        its.append(len(ls))
    out = dict(H=np.int64(H), W=np.int64(W), K=np.int64(K), M=np.int64(M), vmaps=np.stack(vmaps), rel_poses=np.stack(rels),
               scan=scan, T0s=T0s, params=np.stack(P), T=np.stack(Ts), losses=np.asarray(L, np.float64),
               iters=np.asarray(its, np.int64))

    path = os.path.join(HERE, "proj_hypotheses.npz")
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
    print(path, os.path.getsize(path), "bytes", "iterations", its)


if __name__ == "__main__":
    main()
