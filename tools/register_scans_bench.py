"""Many scans localised against one prior map on one GPU: S distinct scans, one initial estimate each, registered in one
pls_register_scans call against a loop of S pls_register_frame calls.

Maps: those of tools/prior_map_bench.py, the cfg4 map (BASELINE config 4: 5 M points, above KD_COLD_MAP_POINTS, so
later ICP iterations take the batched four-launch path) and a 2 km-wide sparse map of 1 M points.  Scan s is the 0.3 m
grid sample of synthetic 64x2048 scan s placed on the map, its estimate a few metres and degrees off (geman_mcclure 0.3,
<= 10 alignments, threshold_delta_pose 1e-4).  A static map keeps its normals across calls, so two cases are timed:
  * cold: the first call after the map was set, which computes the normals its matches need;
  * warm: a repeated call on the same scans, whose normals are cached.
Each case times both arms alternating, --reps times after a warm-up (host clock around calls that end in a device
synchronisation; median and every sample listed).  The outputs of the two arms are checked bit for bit.  The card's name,
power limit and SM clocks are read in the same run.

    python tools/register_scans_bench.py [--scans 1,8,32,64] [--reps 5] [--out profiles/h100_register_scans.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

MAX_ALIGN = 10


def make_scans(S):
    from scipy.spatial.transform import Rotation
    from pylidar_slam_b200 import synthetic as syn
    import pylidar_slam_b200 as b200
    rng = np.random.RandomState(S)
    scans, T0 = [], np.tile(np.eye(4, dtype=np.float32), (S, 1, 1))
    for s in range(S):
        pc = syn.scan(s, 64, 2048).astype(np.float64)
        T = syn.gt_pose(s).astype(np.float64)
        scans.append(np.ascontiguousarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.3)[0]))
        T0[s, :3, :3] = Rotation.from_euler("z", rng.uniform(-5, 5), degrees=True).as_matrix()
        T0[s, :3, 3] = rng.uniform(-1.5, 1.5, 3) * [1, 1, 0.1]
    return scans, T0


def sm_clocks():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"sm_mhz": float(out[0]), "sm_max_mhz": float(out[1])}
    except Exception:
        return {"sm_mhz": None, "sm_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", default="1,8,32,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_register_scans.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "register_scans_bench.py needs a CUDA device"
    from bench import device_info
    from prior_map_bench import make_maps
    from pylidar_slam_b200 import _lib
    lib = _lib.load()
    maps, _ = make_maps()
    ctx = _lib.Context(local_map_type=_lib.MAP_KDTREE, local_map_size=20, scheme=_lib.SCHEMES["geman_mcclure"],
                       sigma=0.3, max_num_alignments=MAX_ALIGN, gn_max_iters=1, threshold_delta_pose=1e-4)
    result = dict(device=device_info(), max_num_alignments=MAX_ALIGN, reps=args.reps, maps={})

    def set_map(cloud):
        ctx.call("pls_kdmap_set_points", _lib.ptr(cloud), 0, cloud.shape[0])

    def one_call(scans, T0):
        S = len(scans)
        addr = np.array([_lib.ptr(s) for s in scans], np.uint64)
        rows = np.array([s.shape[0] for s in scans], np.int64)
        out = (np.zeros((S, 16), np.float32), np.zeros((S, 6), np.float32), np.zeros((S, MAX_ALIGN), np.float32),
               np.zeros(S, np.int32), np.zeros(S, np.int32))
        ctx.call("pls_register_scans", _lib.ptr(addr), _lib.ptr(rows), S, None, _lib.ptr(T0), S, *[_lib.ptr(o) for o in out])
        return out

    def loop(scans, T0):
        S = len(scans)
        out = (np.zeros((S, 16), np.float32), np.zeros((S, 6), np.float32), np.zeros((S, MAX_ALIGN), np.float32),
               np.zeros(S, np.int32))
        for s in range(S):
            it = C.c_int(0)
            st = lib.pls_register_frame(ctx.handle, _lib.ptr(scans[s]), scans[s].shape[0], _lib.ptr(T0[s]),
                                        _lib.ptr(out[0][s]), _lib.ptr(out[1][s]), _lib.ptr(out[2][s]), C.byref(it))
            assert st in (_lib.PLS_OK, _lib.PLS_E_SINGULAR), st
            out[3][s] = it.value
        return out

    def timed(fn, *a):
        ctx.call("pls_synchronize")
        t0 = time.perf_counter()
        r = fn(*a)
        ctx.call("pls_synchronize")
        return (time.perf_counter() - t0) * 1e3, r

    def same(a, b, what):
        for k in range(4):
            assert a[k].tobytes() == b[k].reshape(a[k].shape).tobytes(), (what, k)

    def stats(t):
        t = sorted(t)
        return dict(median=t[len(t) // 2], all=t)

    all_scans, all_T0 = make_scans(max(int(s) for s in args.scans.split(",")))
    for name, cloud in maps.items():
        entry = dict(points=int(cloud.shape[0]), scans={})
        for S in [int(s) for s in args.scans.split(",")]:
            scans, T0 = all_scans[:S], np.ascontiguousarray(all_T0[:S])
            set_map(cloud)
            a = one_call(scans, T0)
            same(a, loop(scans, T0), (name, S))   # warm-up of both arms, and the bit-for-bit check
            cold = dict(call=[], loop=[])
            warm = dict(call=[], loop=[])
            for _ in range(args.reps):   # alternating arms; a cold sample re-sets the map first (untimed)
                set_map(cloud)
                t, r = timed(one_call, scans, T0)
                cold["call"].append(t)
                same(a, r, (name, S, "cold call"))
                set_map(cloud)
                t, r = timed(loop, scans, T0)
                cold["loop"].append(t)
                same(a, r, (name, S, "cold loop"))
                warm["call"].append(timed(one_call, scans, T0)[0])
                warm["loop"].append(timed(loop, scans, T0)[0])
            row = dict(scan_points=[int(s.shape[0]) for s in scans], iterations=a[3].tolist())
            for case, d in (("cold", cold), ("warm", warm)):
                c, l = stats(d["call"]), stats(d["loop"])
                row[case] = dict(one_call_ms=c, loop_ms=l, speedup=l["median"] / c["median"])
                print(f"{name} S={S} {case}: one call {c['median']:.2f} ms, loop {l['median']:.2f} ms, "
                      f"x{l['median'] / c['median']:.2f}", flush=True)
            entry["scans"][str(S)] = row
        result["maps"][name] = entry
    result["clocks_after"] = sm_clocks()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "maps"}))


if __name__ == "__main__":
    main()
