"""B pose hypotheses of one scan on a projective local map: one pls_register_hypotheses call against a loop of B
pls_register_frame calls, on one GPU.

Models: the projective odometry run over 26 synthetic frames at 64x720 and at 128x2048, local_map_size K = 20 (the
model holds 20 frames).  The scan is the 27th frame; hypotheses are a +-10 degree yaw sweep with offsets up to 2 m
(geman_mcclure 0.3, <= 10 alignments, threshold_delta_pose 1e-4).  Every arm is warmed up, then timed over --reps
alternating repetitions with a host clock around calls that end in a device synchronisation (median and all listed);
the two arms are checked bit for bit.  A separate profiled pass (torch.profiler, CUDA activity) gives the device time
of the correspondence kernels over the call, next to the model bytes the kernels ask for, computed from the shapes:
one pass per executed hypothesis-iteration in both arms (one CTA reads a tile for one hypothesis); what differs is how
many of those passes L2 serves, which the kernel times show and the bytes do not.

    python tools/proj_hypotheses_bench.py [--batches 1,8,32,64] [--reps 5] [--out profiles/h100_proj_hypotheses.json]
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAX_ALIGN = 10
K = 20
SHAPES = [(64, 720), (128, 2048)]
WARM_FRAMES = 26


def hypotheses(B):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(B)
    T0 = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(B):
        T0[b, :3, :3] = Rotation.from_euler("z", -10.0 + 20.0 * b / max(B - 1, 1), degrees=True).as_matrix()
        T0[b, :3, 3] = rng.uniform(-2, 2, 3) * [1, 1, 0.1]
    return T0


def build_model(_lib, H, W):
    from pylidar_slam_b200 import synthetic as syn
    lib = _lib.load()
    ctx = _lib.Context(local_map_type=_lib.MAP_PROJECTIVE, height=H, width=W, local_map_size=K,
                       scheme=_lib.SCHEMES["geman_mcclure"], sigma=0.3, max_num_alignments=MAX_ALIGN, gn_max_iters=1,
                       threshold_delta_pose=1e-4, threshold_trans=0.0, threshold_rot=0.0)
    init = None
    for k in range(WARM_FRAMES):
        pts = np.ascontiguousarray(syn.scan(k, H, W), np.float32)
        pose, params, info, has = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
        st = lib.pls_process_frame(ctx.handle, _lib.ptr(pts), _lib.INPUT_NDARRAY, pts.shape[0], _lib.ptr(init),
                                   _lib.ptr(pose), _lib.ptr(params), C.byref(has), _lib.ptr(info))
        assert st == _lib.PLS_OK, st
        if has.value:
            init = pose.reshape(4, 4).copy()
    # the pending update of the last frame is enqueued by the next call: one query makes the model complete
    nf = C.c_int(0)
    ctx.call("pls_projmap_num_frames", C.byref(nf))
    scan = np.ascontiguousarray(syn.scan(WARM_FRAMES, H, W), np.float32)
    return ctx, scan, nf.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_proj_hypotheses.json"))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "proj_hypotheses_bench.py needs a CUDA device"
    from bench import device_info
    from pylidar_slam_b200 import _lib
    lib = _lib.load()
    result = dict(device=device_info(), max_num_alignments=MAX_ALIGN, local_map_size=K, reps=args.reps, shapes={})
    for H, W in SHAPES:
        ctx, scan, frames = build_model(_lib, H, W)
        n = scan.shape[0]

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

        hw = H * W
        model_bytes = hw * frames * 12          # the K vertex rows of every pixel, read once per pass
        entry = dict(H=H, W=W, model_frames=frames, scan_points=int(n), model_bytes_per_pass=model_bytes, batches={})
        for B in [int(b) for b in args.batches.split(",")]:
            T0 = hypotheses(B)
            a = one_call(T0)
            b = loop(T0)   # warm-up of both arms, and the bit-for-bit check
            for k in range(4):
                assert a[k].tobytes() == b[k].reshape(a[k].shape).tobytes(), (H, W, B, k)
            t_call, t_loop = [], []
            for _ in range(args.reps):   # alternating
                t_call.append(timed(one_call, T0)[0])
                t_loop.append(timed(loop, T0)[0])
            t_call.sort()
            t_loop.sort()
            med_c, med_l = t_call[len(t_call) // 2], t_loop[len(t_loop) // 2]
            # profiled pass: device time of the correspondence kernels per executed hypothesis-iteration sum
            from torch.profiler import ProfilerActivity, profile
            kern = {}
            for arm, fn in (("one_call", one_call), ("loop", loop)):
                ctx.call("pls_synchronize")
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn(T0)
                    ctx.call("pls_synchronize")
                tot = {}
                for ev in prof.key_averages():
                    m = re.search(r"(proj_icp\w*_kernel|query_\w*_kernel|icp_step\w*_kernel)(<\d+>)?", ev.key)
                    if m:
                        t = tot.setdefault(m.group(0), dict(us=0.0, count=0))
                        t["us"] += getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                        t["count"] += ev.count
                kern[arm] = tot
            iters = a[3]
            max_it = int(iters.max())
            # model bytes the correspondence kernels ask for over the call: one pass per hypothesis still iterating,
            # in both arms
            live = [int((iters > i).sum()) for i in range(max_it)]
            bytes_call = bytes_loop = sum(live) * model_bytes
            entry["batches"][str(B)] = dict(one_call_ms=med_c, loop_ms=med_l, speedup=med_l / med_c, one_call_all=t_call,
                                            loop_all=t_loop, iterations=iters.tolist(), model_bytes_one_call=bytes_call,
                                            model_bytes_loop=bytes_loop, kernels=kern)
            corr = {arm: sum(v["us"] for k, v in kern[arm].items() if k.startswith("proj_icp")) / 1e3 for arm in kern}
            entry["batches"][str(B)]["correspondence_kernel_ms"] = corr
            print(f"{H}x{W} B={B}: one call {med_c:.2f} ms, loop {med_l:.2f} ms, x{med_l / med_c:.2f}; "
                  f"correspondence kernels {corr['one_call']:.2f} / {corr['loop']:.2f} ms; "
                  f"model bytes {bytes_call / 1e6:.0f} / {bytes_loop / 1e6:.0f} MB", flush=True)
        result["shapes"][f"{H}x{W}"] = entry
        ctx.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k != "shapes"}))


if __name__ == "__main__":
    main()
