"""Batched against per-scan pose search on one GPU: KdTreeLocalMap.search_poses_scans (pls_kdmap_pose_search_scans)
against a loop of search_poses (pls_kdmap_pose_search), and ICPFrameToModel.localize_scans against a loop of localize,
on the same context, outputs compared bit for bit.

Maps: cfg4, the scene and the sparse 2 km map of tools/prior_map_bench.py.  Scans: synthetic frames 0, 1, 2, ...
grid-sampled at 0.3 m (about 32 k points each), each at its own ground-truth pose, so a batch is spread along the
trajectory; each prior is its pose moved by a known offset (up to 3 m and 12 degrees, seeded).  Batch sizes S = 1, 8,
64, 256 (localize: 1, 8, 64).  Windows: 13 yaws x +-5 m at 0.5 m (a GNSS prior) and 72 yaws x +-20 m at 0.5 m;
localize over the first.
Timing: host clock around calls that end in a device synchronisation.  Each case is warmed up once, then the two arms
alternate for --reps repetitions (median, min, max).

    python tools/pose_search_scans_bench.py [--reps 5] [--out profiles/h100_pose_search_scans.json]
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

K = 8
SIZES = (1, 8, 64, 256)
LOCALIZE_SIZES = (1, 8, 64)  # a loop of 256 localize calls takes about 25 s per repetition on one map
# (name, yaw_range, yaw_step, radius m, cell m): 13 yaws = +-6 steps of 5 degrees; 72 yaws = the full circle
WINDOWS = (("13yaw_5m", np.deg2rad(30.0), np.deg2rad(5.0), 5.0, 0.5),
           ("72yaw_20m", np.pi, np.deg2rad(5.0), 20.0, 0.5))


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def _same_search(a, b):
    return all(np.array_equal(x, y) for ra, rb in zip(a, b) for x, y in zip(ra, rb)) and len(a) == len(b)


def _same_localize(a, b):
    if len(a) != len(b):
        return False
    for la, lb in zip(a, b):
        if len(la) != len(lb):
            return False
        for ca, cb in zip(la, lb):
            if (ca.score, ca.coarse_score, ca.coarse_rank, ca.iterations, ca.status) != \
                    (cb.score, cb.coarse_score, cb.coarse_rank, cb.iterations, cb.status):
                return False
            if not (np.array_equal(ca.T, cb.T) and np.array_equal(ca.T0, cb.T0)):
                return False
    return True


def _alternate(arms, reps):
    """Warm-up once per arm (its outputs kept), then the arms alternate for reps repetitions."""
    res, times = {}, {k: [] for k in arms}
    for k, fn in arms.items():
        res[k] = _timed(fn)[1]
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(_timed(fn)[0])
    row = {}
    for k in arms:
        row[f"{k}_median_ms"] = 1e3 * float(np.median(times[k]))
        row[f"{k}_min_ms"] = 1e3 * min(times[k])
        row[f"{k}_max_ms"] = 1e3 * max(times[k])
    return row, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pose_search_scans.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_search_scans_bench.py needs a CUDA device"
    import pylidar_slam_b200 as b200
    from bench import device_info
    from pose_search_bench import _odometry, _scene
    from prior_map_bench import make_maps
    from pylidar_slam_b200 import synthetic as syn
    from pylidar_slam_b200.odometry import KdTreeLocalMap, KdTreeLocalMapConfig, yaw_sweep
    maps, _ = make_maps()
    maps["scene"] = _scene(maps["cfg4"])
    S_max = max(SIZES)
    scans = [np.ascontiguousarray(b200.grid_sample(syn.scan(k, 64, 2048).astype(np.float32), 0.3)[0])
             for k in range(S_max)]
    rng = np.random.RandomState(0)
    priors = np.stack([syn.gt_pose(k).astype(np.float64) for k in range(S_max)])
    for s in range(S_max):
        th = np.deg2rad(rng.uniform(-12.0, 12.0))
        R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1.0]])
        priors[s, :3, :3] = R @ priors[s, :3, :3]
        priors[s, :2, 3] += rng.uniform(-3.0, 3.0, 2)
    out = dict(device=device_info(0), K=K, reps=args.reps, scan_points=[int(s.shape[0]) for s in scans],
               search=[], localize=[])
    for mname in ("cfg4", "scene", "wide2km"):
        o = _odometry(10)
        km = KdTreeLocalMap(KdTreeLocalMapConfig(), ctx=o.ctx)
        km.set_map_pointcloud(maps[mname])
        for wname, yaw_range, yaw_step, radius, cell in WINDOWS:
            bases = [yaw_sweep(priors[s], yaw_range, yaw_step) for s in range(S_max)]
            h = int(np.ceil(radius / cell))
            for S in SIZES:
                row = dict(map=mname, map_points=int(maps[mname].shape[0]), window=wname, S=S,
                           poses_per_scan=int(bases[0].shape[0] * (2 * h + 1) ** 2))
                arms = {"batched": lambda: km.search_poses_scans(scans[:S], bases[:S], cell, (h, h), K),
                        "loop": lambda: [km.search_poses(scans[s], bases[s], cell, (h, h), K) for s in range(S)]}
                t, res = _alternate(arms, args.reps)
                row.update(t)
                row["outputs_equal"] = bool(_same_search(res["batched"], res["loop"]))
                row["speedup"] = row["loop_median_ms"] / row["batched_median_ms"]
                out["search"].append(row)
                print(json.dumps(row), flush=True)
        wname, yaw_range, yaw_step, radius, cell = WINDOWS[0]
        for S in LOCALIZE_SIZES:
            row = dict(map=mname, window=wname, S=S, num_candidates=K)
            kw = dict(cell_size=cell, yaw_range=yaw_range, yaw_step=yaw_step, num_candidates=K)
            arms = {"batched": lambda: o.localize_scans(scans[:S], priors[:S], radius, **kw),
                    "loop": lambda: [o.localize(scans[s], priors[s], radius, **kw) for s in range(S)]}
            t, res = _alternate(arms, args.reps)
            row.update(t)
            row["outputs_equal"] = bool(_same_localize(res["batched"], res["loop"]))
            row["speedup"] = row["loop_median_ms"] / row["batched_median_ms"]
            gt = [syn.gt_pose(k).astype(np.float64) for k in range(S)]
            errs = []
            for s, cands in enumerate(res["batched"]):
                if cands:
                    d = np.linalg.inv(gt[s]) @ cands[0].T
                    errs.append(float(np.linalg.norm(d[:3, 3])))
            row["best_within_0_1m"] = int(sum(e <= 0.1 for e in errs))
            out["localize"].append(row)
            print(json.dumps(row), flush=True)
    out["all_outputs_equal"] = all(r["outputs_equal"] for r in out["search"] + out["localize"])
    out["device_after"] = device_info(0)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
