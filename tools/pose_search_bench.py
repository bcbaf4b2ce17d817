"""Correlative pose search on one GPU: pls_kdmap_pose_search time and poses scored per second, and
ICPFrameToModel.localize's success rate against a blind register_new_frame_hypotheses sweep with the same ICP budget.

Maps are those of tools/prior_map_bench.py: cfg4 (the scene plus 4.8 M uniform filler, which occupies most 0.5 m cells
of its 200 m box: a timing case only), the scene alone (0.1 m grid samples of the even frames 0-58 placed by gt_pose)
and the sparse 2 km map.  The scan is frame 7 in the sensor frame, grid-sampled at 1 m (~4 k points) or 0.3 m (~32 k).
Timing: every case warmed up once, then --reps alternating repetitions, host clock around calls that end in a device
synchronisation (median and spread).  Accuracy: priors 5-30 m and 0-180 degrees off gt_pose(7); success = within
0.1 m and 0.5 degrees.  The blind sweep registers num_candidates hypotheses (yaw steps of 360/num_candidates degrees at
the prior's position), the ICP budget localize spends on its candidates.

    python tools/pose_search_bench.py [--reps 5] [--out profiles/h100_pose_search.json]
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


def _scans():
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    pc = syn.scan(7, 64, 2048).astype(np.float32)
    return {f"{v}m": np.ascontiguousarray(b200.grid_sample(pc, v)[0]) for v in (1.0, 0.3)}


def _odometry(max_align):
    import pylidar_slam_b200 as b200
    proj = b200.SphericalProjector(height=64, width=2048, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=20),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3,
                                                                              max_iters=1)),
        max_num_alignments=max_align, threshold_delta_pose=1e-4, data_key="numpy_pc")
    o = b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0")
    o.init()
    return o


def _rz(t):
    return np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1.0]])


def _err(T, gt):
    d = np.linalg.inv(gt) @ T
    return float(np.linalg.norm(d[:3, 3])), float(np.rad2deg(abs(np.arctan2(d[1, 0], d[0, 0]))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--trials", type=int, default=12)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pose_search.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_search_bench.py needs a CUDA device"
    import pylidar_slam_b200 as b200
    from bench import device_info
    from prior_map_bench import make_maps
    from pylidar_slam_b200 import synthetic as syn
    from pylidar_slam_b200.odometry import KdTreeLocalMap, KdTreeLocalMapConfig, yaw_sweep
    maps, _ = make_maps()
    maps["scene"] = _scene(maps["cfg4"])
    scans = _scans()
    gt = syn.gt_pose(7)
    out = dict(device=device_info(0), scan_points={k: int(v.shape[0]) for k, v in scans.items()}, timing=[], accuracy=[])
    windows = [dict(yaws=72, radius=20.0, cell=0.5), dict(yaws=360, radius=50.0, cell=1.0)]
    for mname in ("cfg4", "scene", "wide2km"):
        o = _odometry(10)
        km = KdTreeLocalMap(KdTreeLocalMapConfig(), ctx=o.ctx)
        km.set_map_pointcloud(maps[mname])
        arms = []
        for w in windows:
            bases = yaw_sweep(gt, np.pi, 2 * np.pi / w["yaws"])
            half = int(np.ceil(w["radius"] / w["cell"]))
            for sname, scan in scans.items():
                arms.append((w, sname, scan, bases, half))
        for w, sname, scan, bases, half in arms:     # warm-up
            km.search_poses(scan, bases, w["cell"], (half, half), 8)
        times = {i: [] for i in range(len(arms))}
        for _ in range(args.reps):
            for i, (w, sname, scan, bases, half) in enumerate(arms):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                km.search_poses(scan, bases, w["cell"], (half, half), 8)
                times[i].append(time.perf_counter() - t0)
        for i, (w, sname, scan, bases, half) in enumerate(arms):
            med = float(np.median(times[i]))
            poses = bases.shape[0] * (2 * half + 1) ** 2
            T, sc, _ = km.search_poses(scan, bases, w["cell"], (half, half), 8)
            out["timing"].append(dict(map=mname, map_points=int(maps[mname].shape[0]), scan=sname, yaws=w["yaws"],
                                      radius_m=w["radius"], cell_m=w["cell"], poses=poses, median_ms=1e3 * med,
                                      min_ms=1e3 * min(times[i]), max_ms=1e3 * max(times[i]),
                                      poses_per_s=poses / med, top_score=int(sc[0]) if len(sc) else 0,
                                      top_error_m_deg=_err(T[0], gt) if len(sc) else None))
            print(json.dumps(out["timing"][-1]), flush=True)
        if mname == "cfg4":
            continue
        rng = np.random.RandomState(7)
        scan = scans["0.3m"]
        for trial in range(args.trials):
            dist, yaw = rng.uniform(5, 30), rng.uniform(0, 180) * rng.choice([-1, 1])
            ang = rng.uniform(-np.pi, np.pi)
            prior = gt.copy()
            prior[:3, :3] = _rz(np.deg2rad(yaw)) @ gt[:3, :3]
            prior[:2, 3] += dist * np.array([np.cos(ang), np.sin(ang)])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = o.localize(scan, prior, radius=32.0, cell_size=0.5, yaw_step=np.deg2rad(5), num_candidates=8)
            t_loc = time.perf_counter() - t0
            e = _err(res[0].T, gt) if res else (np.inf, np.inf)
            blind = yaw_sweep(prior, np.pi, 2 * np.pi / 8).astype(np.float32)
            t0 = time.perf_counter()
            _, Tb, _, _ = o.register_new_frame_hypotheses(scan, blind)
            t_blind = time.perf_counter() - t0
            sb = km.score_poses(scan, Tb.astype(np.float64), 0.5)
            eb = _err(Tb[int(np.argmax(sb))].astype(np.float64), gt)
            out["accuracy"].append(dict(map=mname, start_offset_m=dist, start_yaw_deg=yaw, localize_ms=1e3 * t_loc,
                                        localize_error_m_deg=e, localize_ok=bool(e[0] <= 0.1 and e[1] <= 0.5),
                                        blind_ms=1e3 * t_blind, blind_error_m_deg=eb,
                                        blind_ok=bool(eb[0] <= 0.1 and eb[1] <= 0.5)))
            print(json.dumps(out["accuracy"][-1]), flush=True)
    for mname in ("scene", "wide2km"):
        rows = [r for r in out["accuracy"] if r["map"] == mname]
        out[f"summary_{mname}"] = dict(localize_success=sum(r["localize_ok"] for r in rows) / len(rows),
                                       blind_success=sum(r["blind_ok"] for r in rows) / len(rows),
                                       localize_median_ms=float(np.median([r["localize_ms"] for r in rows])),
                                       blind_median_ms=float(np.median([r["blind_ms"] for r in rows])))
        print(json.dumps({mname: out[f"summary_{mname}"]}), flush=True)
    out["device_after"] = device_info(0)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)


def _scene(cfg4):
    """The scene part of the cfg4 map: everything before its 5 M - len(scene) uniform filler rows."""
    from pylidar_slam_b200 import synthetic as syn
    import pylidar_slam_b200 as b200
    parts = []
    for k in range(0, 60, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.1)[0]))
    n = sum(p.shape[0] for p in parts)
    return np.ascontiguousarray(cfg4[:n])


if __name__ == "__main__":
    main()
