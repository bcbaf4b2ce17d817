"""Exhaustive against pruned pose search on one GPU: pls_kdmap_pose_search (K = 8, no volume) and
pls_kdmap_pose_search_pyramid on the same context, times and outputs compared bit for bit.

Maps and scans are those of tools/pose_search_bench.py (cfg4, the scene, the sparse 2 km map; frame 7 grid-sampled at
1 m and 0.3 m), the bases a yaw sweep about gt_pose(7).  Workloads:
  * the two windows of tools/pose_search_bench.py and +-200 m at 0.5 m, on the three maps, for both scans;
  * +-1000 m at 1 m and at 0.5 m with 72 yaws on the 2 km map (the exhaustive call is run where it accepts);
  * small windows of 72 yaws at 0.5 m on the scene and the 2 km map, around the crossover of _pose_search.
Timing: host clock around calls that end in a device synchronisation.  Each case is warmed up once, then the two
calls alternate for --reps repetitions (median, min, max).  A refusal (PLS_E_INVALID) is recorded with its message.

    python tools/pose_search_pyramid_bench.py [--reps 5] [--out profiles/h100_pose_search_pyramid.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

K = 8


def _call(lib, ctx, name, scan, bases, cell, half):
    T, sc = np.zeros((K, 4, 4)), np.zeros(K, np.int32)
    ix, num = np.zeros(K, np.int64), C.c_int(-1)
    args = [ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(bases), bases.shape[0], float(cell), half, half, K]
    if name == "pls_kdmap_pose_search":
        args.append(None)
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = getattr(lib.load(), name)(*args, lib.ptr(T), lib.ptr(sc), lib.ptr(ix), C.byref(num))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    if st != lib.PLS_OK:
        return None, lib.load().pls_last_error(ctx.handle).decode()
    k = num.value
    return dt, (T[:k], sc[:k], ix[:k])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_pose_search_pyramid.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_search_pyramid_bench.py needs a CUDA device"
    from bench import device_info
    from pose_search_bench import _scans, _scene
    from prior_map_bench import make_maps
    from pylidar_slam_b200 import _lib as lib
    from pylidar_slam_b200 import synthetic as syn
    from pylidar_slam_b200.odometry import yaw_sweep
    maps, _ = make_maps()
    maps["scene"] = _scene(maps["cfg4"])
    scans = _scans()
    gt = syn.gt_pose(7)
    out = dict(device=device_info(0), scan_points={k: int(v.shape[0]) for k, v in scans.items()}, K=K, reps=args.reps,
               cases=[])
    cases = []
    for mname in ("cfg4", "scene", "wide2km"):
        for yaws, radius, cell in ((72, 20.0, 0.5), (360, 50.0, 1.0), (72, 200.0, 0.5)):
            for sname in scans:
                cases.append((mname, sname, yaws, radius, cell))
    for cell in (1.0, 0.5):
        for sname in scans:
            cases.append(("wide2km", sname, 72, 1000.0, cell))
    for mname in ("scene", "wide2km"):
        for half in (8, 32, 64, 128, 256, 320):
            cases.append((mname, "1.0m", 72, half * 0.5, 0.5))
    ctxs = {}
    for mname in ("cfg4", "scene", "wide2km"):
        ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=20)
        pts = np.ascontiguousarray(maps[mname], np.float32)
        ctx.call("pls_kdmap_set_points", lib.ptr(pts), 0, pts.shape[0])
        ctxs[mname] = ctx
    for mname, sname, yaws, radius, cell in cases:
        ctx, scan = ctxs[mname], scans[sname]
        bases = np.ascontiguousarray(yaw_sweep(gt, np.pi, 2 * np.pi / yaws))
        half = int(np.ceil(radius / cell))
        poses = yaws * (2 * half + 1) ** 2
        row = dict(map=mname, map_points=int(maps[mname].shape[0]), scan=sname, yaws=yaws, radius_m=radius, cell_m=cell,
                   poses=poses)
        times = {"exhaustive": [], "pyramid": []}
        res = {}
        names = {"exhaustive": "pls_kdmap_pose_search", "pyramid": "pls_kdmap_pose_search_pyramid"}
        for arm, name in names.items():  # warm-up, and the arm's outputs
            dt, r = _call(lib, ctx, name, scan, bases, cell, half)
            res[arm] = r
            if dt is None:
                row[f"{arm}_refused"] = r
        live = [arm for arm in names if f"{arm}_refused" not in row]
        for _ in range(args.reps):
            for arm in live:
                dt, r = _call(lib, ctx, names[arm], scan, bases, cell, half)
                times[arm].append(dt)
        for arm in live:
            row[f"{arm}_median_ms"] = 1e3 * float(np.median(times[arm]))
            row[f"{arm}_min_ms"] = 1e3 * min(times[arm])
            row[f"{arm}_max_ms"] = 1e3 * max(times[arm])
            row[f"{arm}_runs"] = len(times[arm])
        if len(live) == 2:
            row["outputs_equal"] = bool(all(np.array_equal(a, b) for a, b in zip(res["exhaustive"], res["pyramid"])))
            row["speedup"] = row["exhaustive_median_ms"] / row["pyramid_median_ms"]
        if "pyramid" in live:
            T, sc, _ = res["pyramid"]
            row["top_score"] = int(sc[0]) if len(sc) else 0
        out["cases"].append(row)
        print(json.dumps(row), flush=True)
    out["all_outputs_equal"] = all(r.get("outputs_equal", True) for r in out["cases"])
    out["device_after"] = device_info(0)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
