"""Goldens of localisation against a prior map, from the UNMODIFIED reference under oracle/ref_shims.py.  Build
container only:

    python tests/golden/make_golden_prior_map.py -> prior_map.npz
    python tests/golden/make_golden_prior_map.py --check   # regenerate in memory, compare with the committed file
                                                           # bit for bit, write nothing

Cases (KdTreeLocalMap.set_map_pointcloud, local_map.py:289-299; get_last_frame, :238-240 and :425-427):
  pm_cloud32 / pm_cloud64     a float32 and a float64 cloud set as the map
  pm_nb*_off, pm_nb*, pm_nrm* nearest_neighbor_search of pm_queries after each, normals off and on
  pm_err_*                    error type and message of: a search with normals after set_map_pointcloud(.., normals),
                              set_map_pointcloud with a torch tensor, get_last_frame right after set_map_pointcloud, the
                              projective get_last_frame before any update
  pm_ev_*                     a set cloud, then frames up to and past local_map_size = 3 (one frame of NaN rows only,
                              inserted as zero rows): map rows, frame counts and get_last_frame after every update
  pm_proj_*                   the projective map's get_last_frame after two vertex maps
  pm_reg_*                    ICPFrameToModel.register_new_frame on a set map from several initial estimates
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
H, W = 16, 256      # scans of the set clouds and of the registration
PH, PW = 8, 128      # vertex maps of the projective map
LM_SIZE = 3


def frame_points(k):
    """Scan k of the synthetic sequence, float32, in the frame of scan 0 (ground-truth poses)."""
    pc = syn.scan(k, H, W).astype(np.float64)
    T = syn.gt_pose(k).astype(np.float64)
    return (pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def caught(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 -- the type is what is pinned
        return np.array([type(e).__name__, str(e)])
    raise AssertionError("the reference did not raise")


def kd_map(size=LM_SIZE):
    lm = ns.local_map.KdTreeLocalMap(ns.local_map.KdTreeLocalMapConfig(local_map_size=size))
    lm.init()
    return lm


def main():
    out = {}
    cloud32 = np.ascontiguousarray(np.concatenate([frame_points(k)[::3] for k in (0, 3, 6)]))
    rng = np.random.RandomState(7)
    cloud64 = cloud32[::8].astype(np.float64) + rng.uniform(-1e-3, 1e-3, cloud32[::8].shape)
    q = frame_points(2)[::12] + rng.normal(0, 0.05, (len(frame_points(2)[::12]), 3)).astype(np.float32)
    out.update(pm_cloud32=cloud32, pm_cloud64=cloud64, pm_queries=q)

    # ---- set_map_pointcloud + nearest_neighbor_search, float32 and float64 clouds
    for tag, cloud in (("32", cloud32), ("64", cloud64)):
        lm = kd_map()
        lm.set_map_pointcloud(cloud)
        r = lm.nearest_neighbor_search(q, with_normals=False)
        out[f"pm_nb{tag}_off"] = np.asarray(r.neighbor_points)
        r = lm.nearest_neighbor_search(q)
        out[f"pm_nb{tag}"], out[f"pm_nrm{tag}"] = np.asarray(r.neighbor_points), np.asarray(r.neighbor_normals)

    # ---- the normals argument: stored [N,3], read at column 3 by the search
    lm = kd_map()
    lm.set_map_pointcloud(cloud32, normals=np.zeros_like(cloud32))
    out["pm_nb_given_off"] = np.asarray(lm.nearest_neighbor_search(q, with_normals=False).neighbor_points)
    out["pm_err_given_normals"] = caught(lambda: lm.nearest_neighbor_search(q))
    out["pm_err_torch_cloud"] = caught(lambda: kd_map().set_map_pointcloud(torch.from_numpy(cloud32)))
    lm = kd_map()
    lm.set_map_pointcloud(cloud32[:500])
    out["pm_err_last_after_set"] = caught(lm.get_last_frame)

    # ---- updates after a set cloud, up to and past local_map_size: the eviction slices rows off the front
    lm = kd_map()
    prior = np.ascontiguousarray(cloud32[::8])
    lm.set_map_pointcloud(prior)
    out["pm_ev_prior"] = prior
    for k in range(6):
        rel = syn.gt_relative_pose(k + 1).astype(np.float32)
        pts = np.ascontiguousarray(syn.scan(k + 1, H, W)[:: 10 + k])
        if k == 3:
            pts = np.full((40, 3), np.nan, np.float32)  # every row dropped: a frame of zero rows
        lm.update(torch.from_numpy(rel).unsqueeze(0), new_pc_data=pts)
        out[f"pm_ev_rel_{k}"], out[f"pm_ev_pts_{k}"] = rel, pts
        out[f"pm_ev_map_{k}"] = np.asarray(lm._local_map).copy()
        out[f"pm_ev_counts_{k}"] = np.asarray(lm._local_map_num_elements, dtype=np.int64)
        out[f"pm_ev_last_{k}"] = lm.get_last_frame().numpy().copy()

    # ---- the projective map's last frame
    proj = ns.projection.SphericalProjector(height=PH, width=PW, up_fov=3.0, down_fov=-24.0)
    pm = ns.local_map.ProjectiveLocalMap(ns.local_map.ProjectiveLocalMapConfig(local_map_size=LM_SIZE), projector=proj)
    pm.init()
    out["pm_err_proj_empty"] = caught(pm.get_last_frame)
    v0 = torch.from_numpy(syn.vertex_map_from_scan(syn.scan(0, PH, PW), PH, PW))
    v1 = torch.from_numpy(syn.vertex_map_from_scan(syn.scan(1, PH, PW), PH, PW))
    pm.update(torch.eye(4).unsqueeze(0), new_vertex_map=v0)
    pm.update(torch.from_numpy(syn.gt_relative_pose(1).astype(np.float32)).unsqueeze(0), new_vertex_map=v1)
    out.update(pm_proj_v0=v0[0].numpy(), pm_proj_v1=v1[0].numpy(), pm_proj_rel=syn.gt_relative_pose(1).astype(np.float32),
               pm_proj_last=pm.get_last_frame().numpy().copy())

    # ---- register_new_frame on a set map from several initial estimates
    cfg = ns.icp.ICPFrameToModelConfig(
        local_map=ns.local_map.KdTreeLocalMapConfig(local_map_size=20),
        alignment=ns.alignment.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                                      max_iters=1)),
        max_num_alignments=12, data_key="numpy_pc", threshold_delta_pose=1e-4)
    algo = ns.icp.ICPFrameToModel(cfg, projector=proj, pose=pose, device=torch.device("cpu"))
    algo.init()
    algo.local_map.set_map_pointcloud(cloud32)
    scan = frame_points(4)[::4]
    truth = torch.zeros(1, 6)
    offsets = np.array([[0, 0, 0, 0, 0, 0], [0.3, -0.2, 0.05, 0, 0, 0.03], [-0.5, 0.4, 0, 0.01, -0.01, -0.06],
                        [0.8, 0.8, 0.1, 0, 0, 0.1]], np.float32)
    T0s = pose.build_pose_matrix(truth + torch.from_numpy(offsets)).numpy().astype(np.float32)
    P, Ts, L, its = [], [], [], []
    for T0 in T0s:
        p, T, ls = algo.register_new_frame(torch.from_numpy(scan), initial_estimate=torch.from_numpy(T0).unsqueeze(0))
        P.append(np.asarray(p, np.float32).reshape(6))
        Ts.append(np.asarray(T, np.float32).reshape(4, 4))
        L.append([float(x) for x in ls] + [np.nan] * (cfg.max_num_alignments - len(ls)))
        its.append(len(ls))
    out.update(pm_reg_scan=scan, pm_reg_T0=T0s, pm_reg_params=np.stack(P), pm_reg_T=np.stack(Ts),
               pm_reg_losses=np.asarray(L, np.float64), pm_reg_iters=np.asarray(its, np.int64))

    path = os.path.join(HERE, "prior_map.npz")
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
    print(path, os.path.getsize(path), "bytes", {k: v.shape for k, v in out.items() if k.startswith("pm_reg")})
    print("iterations", its, "errors", {k: tuple(v) for k, v in out.items() if k.startswith("pm_err")})


if __name__ == "__main__":
    main()
