"""The correspondence gate of register_new_frames (pls_register_scans_gated) on the H100.

  (a) overhead: register_new_frames of B 0.3 m-sampled scans of 32 k points near the truth (within 0.5 m and 3 degrees),
      B in (1, 8, 64, 512), max_distance 1 m against inf, on the scene map and on scene_plus_2M_uniform (above
      KD_COLD_MAP_POINTS: the four-launch later iterations);
  (b) far-off hypotheses: 8 starts 5-30 m and up to 180 degrees off, gated (1 m) against ungated, time per call;
  (c) accuracy on a changed map (oracle/gated_registration_reference.changed_map_scene): final pose error gated and
      ungated.
Every shape is warmed up first; gated and ungated calls alternate within each repetition and medians are reported.
The card's name, power limit and max SM clock are read in the same run.

    python tools/gated_registration_bench.py --out profiles/h100_gated_registration.json [--reps 7]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from evaluate_poses_bench import card, scene_cloud, scans_of  # noqa: E402


def odometry(max_iters, scheme="geman_mcclure", k=10):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=64, width=2048, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=max_iters, threshold_delta_pose=1e-4, data_key="numpy_pc",
               local_map=dict(type="kdtree_local_map", local_map_size=20, num_neighbors_normals=k),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme=scheme, sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def set_map(odo, cloud):
    import pylidar_slam_b200 as b200
    b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20), ctx=odo.ctx).set_map_pointcloud(cloud)


def poses(B, seed, trans, yaw_deg):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(B):
        T[b, :3, :3] = Rotation.from_euler("z", rng.uniform(-yaw_deg, yaw_deg), degrees=True).as_matrix()
        d = rng.normal(size=2)
        T[b, :2, 3] = d / np.linalg.norm(d) * rng.uniform(*trans)
    return T


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_gated_registration.json"))
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from oracle import gated_registration_reference as gr
    res = {"card": card(), "reps": args.reps, "overhead": [], "far_off": [], "changed_map": {}}
    scene = scene_cloud()
    rng = np.random.RandomState(1)
    fill = rng.uniform([-80, -80, -2], [80, 80, 4], (2_000_000, 3)).astype(np.float32)
    maps = {"scene": scene, "scene_plus_2M_uniform": np.ascontiguousarray(np.concatenate([scene, fill]))}
    max_iters = 10
    for name, cloud in maps.items():
        odo = odometry(max_iters)
        set_map(odo, cloud)
        # (a) near the truth
        for B in (1, 8, 64, 512):
            S = min(B, 64)
            scans = scans_of(scene, S, 32768, B)
            of = np.arange(B, dtype=np.int32) % S
            T0 = poses(B, B, (0.0, 0.5), 3.0)
            for md in (np.inf, 1.0):   # warm-up of both
                odo.register_new_frames(scans, T0, of, max_distance=md)
            t = {np.inf: [], 1.0: []}
            for _ in range(args.reps):
                for md in (np.inf, 1.0):
                    dt, out = timed(lambda: odo.register_new_frames(scans, T0, of, max_distance=md))
                    t[md].append(dt)
            _, Tu, _, iu = odo.register_new_frames(scans, T0, of)
            _, Tg, _, ig = odo.register_new_frames(scans, T0, of, max_distance=1.0)
            res["overhead"].append(dict(
                map=name, B=B, ungated_ms=1e3 * float(np.median(t[np.inf])), gated_ms=1e3 * float(np.median(t[1.0])),
                ratio=float(np.median(t[1.0]) / np.median(t[np.inf])),
                mean_iters_ungated=float(np.mean(iu)), mean_iters_gated=float(np.mean(ig)),
                mean_inlier_fraction=float(np.mean(odo.last_registrations_inliers) / 32768),
                max_pose_diff_m=float(np.abs(Tu[:, :3, 3] - Tg[:, :3, 3]).max())))
            print(res["overhead"][-1], flush=True)
        # (b) far-off hypotheses of one scan
        scan = scans_of(scene, 1, 32768, 99)[0]
        T0 = poses(8, 5, (5.0, 30.0), 180.0)
        for md in (np.inf, 1.0):
            odo.register_new_frame_hypotheses(scan, T0, max_distance=md)
        t = {np.inf: [], 1.0: []}
        for _ in range(max(3, args.reps // 2)):
            for md in (np.inf, 1.0):
                dt, _ = timed(lambda: odo.register_new_frame_hypotheses(scan, T0, max_distance=md))
                t[md].append(dt)
        res["far_off"].append(dict(map=name, hypotheses=8, ungated_ms=1e3 * float(np.median(t[np.inf])),
                                   gated_ms=1e3 * float(np.median(t[1.0])),
                                   speedup=float(np.median(t[np.inf]) / np.median(t[1.0])),
                                   gated_inliers=[int(v) for v in odo.last_hypotheses_inliers]))
        print(res["far_off"][-1], flush=True)
    # (c) the changed map
    prior, scan, truth, start = gr.changed_map_scene(0)
    odo = odometry(30, scheme="default")
    set_map(odo, prior)
    for label, md in (("ungated", np.inf), ("gated_1m", 1.0)):
        _, T, _, it = odo.register_new_frames([scan], start[None], max_distance=md)
        et, er_ = gr.pose_error(T[0], truth)
        res["changed_map"][label] = dict(translation_error_m=et, rotation_error_rad=er_, iterations=int(it[0]))
    print(res["changed_map"], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
