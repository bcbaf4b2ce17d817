"""Throughput of ICPFrameToModel.evaluate_registrations (pls_kdmap_evaluate_poses) on the H100.

For each map and B in (1, 8, 64, 512): one evaluate_registrations call over B poses of 0.3 m-sampled scans of about
32 k points, against a loop of B single-pose calls and against register_new_frames with max_num_alignments = 1 at the
same B.  Every shape is warmed up first; the three variants alternate within each repetition and the medians are
reported.  The card's name, power limit and max SM clock are read in the same run.

    python tools/evaluate_poses_bench.py --out profiles/h100_evaluate_poses.json [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"not read ({e})"
    return info


def scene_cloud(frames=40):
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    parts = []
    for k in range(0, frames, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k).astype(np.float64)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.3)[0]))
    return np.ascontiguousarray(np.concatenate(parts).astype(np.float32))


def odometry(k=10):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=64, width=2048, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=1, threshold_delta_pose=1e-4, data_key="numpy_pc",
               local_map=dict(type="kdtree_local_map", local_map_size=20, num_neighbors_normals=k),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    return odo


def scans_of(cloud, S, n, seed):
    rng = np.random.RandomState(seed)
    return [np.ascontiguousarray((cloud[rng.choice(len(cloud), n, replace=False)]
                                  + rng.normal(0, 0.05, (n, 3))).astype(np.float32)) for _ in range(S)]


def poses(B, seed):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(B):
        T[b, :3, :3] = Rotation.from_euler("z", rng.uniform(-3, 3), degrees=True).as_matrix()
        T[b, :3, 3] = rng.uniform(-0.5, 0.5, 3) * [1, 1, 0.1]
    return T


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_evaluate_poses.json"))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--points", type=int, default=32768)
    a = ap.parse_args()
    import pylidar_slam_b200 as b200
    scene = scene_cloud()
    rng = np.random.RandomState(3)
    fill = rng.uniform([-80, -80, -2], [80, 80, 4], (2_000_000, 3)).astype(np.float32)
    maps = {"scene": scene, "scene_plus_2M_uniform": np.ascontiguousarray(np.concatenate([scene, fill]))}
    result = {"card": card(), "points_per_scan": a.points, "reps": a.reps, "maps": {},
              "not_measured": ["cfg4 map", "2 km map", "re-ranking value on the DESIGN section 19 experiment"]}
    for name, cloud in maps.items():
        odo = odometry()
        lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20), ctx=odo.ctx)
        lm.set_map_pointcloud(cloud)
        scans = scans_of(scene, 8, a.points, 1)
        rows = {"map_points": int(len(cloud)), "B": {}}
        for B in (1, 8, 64, 512):
            T = poses(B, B)
            of = np.arange(B, dtype=np.int32) % len(scans)
            variants = {
                "evaluate_batch": lambda: odo.evaluate_registrations(scans, T, 1.0, of),
                "evaluate_single_loop": lambda: [odo.evaluate_registrations([scans[of[b]]], T[b:b + 1], 1.0)
                                                 for b in range(B)],
                "register_new_frames_1_alignment": lambda: odo.register_new_frames(scans, T, of),
            }
            for fn in variants.values():   # warm-up of every shape
                fn()
            times = {k: [] for k in variants}
            for _ in range(a.reps):
                for k, fn in variants.items():
                    times[k].append(timed(fn))
            rows["B"][str(B)] = {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)),
                                     "per_pose_us": float(np.median(v)) * 1e3 / B} for k, v in times.items()}
            print(name, B, {k: round(float(np.median(v)), 3) for k, v in times.items()}, flush=True)
        result["maps"][name] = rows
        del odo, lm
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
