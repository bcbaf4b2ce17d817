"""Localisation against a prior map on one GPU: set_map_pointcloud time, and B hypotheses of one scan registered in one
pls_register_hypotheses call against a loop of B pls_register_frame calls.

Maps: the cfg4 map (BASELINE config 4: 5 M points, above KD_COLD_MAP_POINTS, so later ICP iterations take the batched
four-launch path) and a 2 km-wide sparse map of 1 M points (coarsened level-0 cells).  The scan is the 0.3 m grid sample
of one synthetic 64x2048 scan placed on the map; hypotheses are a yaw sweep with position offsets of up to 2 m
(geman_mcclure 0.3, <= 10 alignments, threshold_delta_pose 1e-4).  Every arm is warmed up once, then timed over
--reps alternating repetitions (host clock around calls that end in a device synchronisation; median and spread
listed).  The outputs of the two arms are checked bit for bit.

    python tools/prior_map_bench.py [--batches 1,8,32,64] [--reps 5] [--out profiles/h100_prior_map.json]
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

MAX_ALIGN = 10


def make_maps():
    from pylidar_slam_b200 import synthetic as syn
    import pylidar_slam_b200 as b200
    parts = []
    for k in range(0, 60, 2):
        pc = syn.scan(k, 64, 2048).astype(np.float64)
        T = syn.gt_pose(k).astype(np.float64)
        parts.append(np.asarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.1)[0]))
    scene = np.concatenate(parts).astype(np.float32)
    rng = np.random.RandomState(0)
    fill = rng.uniform([-100, -100, -2], [100, 100, 6], (5_000_000 - len(scene), 3)).astype(np.float32)
    cfg4 = np.ascontiguousarray(np.concatenate([scene, fill]))
    local = scene[:200_000]
    wide = np.ascontiguousarray(np.concatenate([local, rng.uniform([-1000, -1000, -5], [1000, 1000, 15],
                                                                   (1_000_000 - len(local), 3)).astype(np.float32)]))
    pc = syn.scan(7, 64, 2048).astype(np.float64)
    T = syn.gt_pose(7).astype(np.float64)
    scan = np.ascontiguousarray(b200.grid_sample((pc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), 0.3)[0])
    return dict(cfg4=cfg4, wide2km=wide), scan


def hypotheses(B):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(B)
    T0 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(B):
        T0[b, :3, :3] = Rotation.from_euler("z", -10.0 + 20.0 * b / max(B - 1, 1), degrees=True).as_matrix()
        T0[b, :3, 3] = rng.uniform(-2, 2, 3) * [1, 1, 0.1]
    return T0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_prior_map.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "prior_map_bench.py needs a CUDA device"
    from bench import device_info
    from pylidar_slam_b200 import _lib
    lib = _lib.load()
    maps, scan = make_maps()
    ctx = _lib.Context(local_map_type=_lib.MAP_KDTREE, local_map_size=20, scheme=_lib.SCHEMES["geman_mcclure"],
                       sigma=0.3, max_num_alignments=MAX_ALIGN, gn_max_iters=1, threshold_delta_pose=1e-4)
    n = scan.shape[0]
    result = dict(device=device_info(), scan_points=int(n), max_num_alignments=MAX_ALIGN, reps=args.reps, maps={})

    def set_map(cloud):
        ctx.call("pls_kdmap_set_points", _lib.ptr(cloud), 0, cloud.shape[0])

    def one_call(T0):
        B = T0.shape[0]
        out = (np.zeros((B, 16), np.float32), np.zeros((B, 6), np.float32), np.zeros((B, MAX_ALIGN), np.float32),
               np.zeros(B, np.int32), np.zeros(B, np.int32))
        ctx.call("pls_register_hypotheses", _lib.ptr(scan), n, _lib.ptr(T0), B, *[_lib.ptr(o) for o in out])
        return out

    def loop(T0):
        B = T0.shape[0]
        out = (np.zeros((B, 16), np.float32), np.zeros((B, 6), np.float32), np.zeros((B, MAX_ALIGN), np.float32),
               np.zeros(B, np.int32))
        for b in range(B):
            it = C.c_int(0)
            st = lib.pls_register_frame(ctx.handle, _lib.ptr(scan), n, _lib.ptr(T0[b]), _lib.ptr(out[0][b]),
                                        _lib.ptr(out[1][b]), _lib.ptr(out[2][b]), C.byref(it))
            assert st in (_lib.PLS_OK, _lib.PLS_E_SINGULAR), st
            out[3][b] = it.value
        return out

    def timed(fn, *a):
        ctx.call("pls_synchronize")
        t0 = time.perf_counter()
        r = fn(*a)
        ctx.call("pls_synchronize")
        return (time.perf_counter() - t0) * 1e3, r

    for name, cloud in maps.items():
        set_map(cloud)  # warm-up: buffers sized
        set_ms = sorted(timed(set_map, cloud)[0] for _ in range(args.reps))
        entry = dict(points=int(cloud.shape[0]), set_map_ms=dict(median=set_ms[len(set_ms) // 2], all=set_ms), batches={})
        for B in [int(b) for b in args.batches.split(",")]:
            T0 = hypotheses(B)
            a = one_call(T0)
            b = loop(T0)   # warm-up of both arms, and the bit-for-bit check
            for k in range(4):
                assert a[k].tobytes() == b[k].reshape(a[k].shape).tobytes(), (name, B, k)
            t_call, t_loop = [], []
            for _ in range(args.reps):   # alternating
                t_call.append(timed(one_call, T0)[0])
                t_loop.append(timed(loop, T0)[0])
            t_call.sort()
            t_loop.sort()
            med_c, med_l = t_call[len(t_call) // 2], t_loop[len(t_loop) // 2]
            entry["batches"][str(B)] = dict(one_call_ms=med_c, loop_ms=med_l, speedup=med_l / med_c, one_call_all=t_call,
                                            loop_all=t_loop, iterations=a[3].tolist())
            print(f"{name} B={B}: one call {med_c:.2f} ms, loop {med_l:.2f} ms, x{med_l / med_c:.2f}", flush=True)
        result["maps"][name] = entry
        print(f"{name}: set_map_pointcloud {entry['set_map_ms']['median']:.1f} ms for {cloud.shape[0]} points", flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "maps"}))


if __name__ == "__main__":
    main()
