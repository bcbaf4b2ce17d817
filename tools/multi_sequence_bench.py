"""Aggregate frames/s of B independent odometry sequences on one GPU: sequential, threaded and batched.

The cfg2 workload with bench.py's constants (64x2048 synthetic scans, grid sample 0.3, kd map of 20 frames,
geman_mcclure 0.3, <= 10 alignments, constant-velocity initialisation), raw scans resident in HBM; sequence i starts
at synthetic frame 200 i.  For each B the three arms run alternately in one process, each on fresh contexts:

  sequential  one host thread calls pls_process_frame_grid_sample on each context in turn (what a user can do without
              pls_process_frames);
  threaded    B persistent host threads, each driving its own context through every step (ctypes releases the GIL
              during a call);
  batched     one pls_process_frames(voxel = 0.3) call per step.

An arm warms up W steps and times K steps, closed after every context is synchronised; frames/s = B K / time, the
median of 3 passes (every pass listed).  Launches per step come from pls_launch_count (its counter is not atomic, so the
threaded arm's count may come out low).  The poses of all three arms are checked bit for bit, sequence by sequence.
A further batched pass per B sets PLS_BATCH_TRACE for its timed steps: the per-step split of a batched call into its
input stage and its batched ICP (CUDA events on the lead context's stream), its epilogue (host clock), and the host
time of the whole call, with the number of extra ICP rounds (pls_process_frames's per-call trace; median per step).

    python tools/multi_sequence_bench.py [--batches 1,2,4,8,16] [--steps 100] [--warmup 24] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, VOXEL, MAX_ALIGN, LM_SIZE, SIGMA = 64, 2048, 0.3, 10, 20, 0.3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,4,8,16")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "multi_sequence_bench.py needs a CUDA device"
    from bench import device_info
    from pylidar_slam_b200 import _lib
    from pylidar_slam_b200 import synthetic as syn
    lib = _lib.load()
    batches = [int(b) for b in args.batches.split(",")]
    Bmax, steps = max(batches), args.warmup + args.steps
    dev = torch.device("cuda", 0)
    scans = torch.from_numpy(np.stack([syn.scan(200 * i + k, H, W) for i in range(Bmax) for k in range(steps)])).to(dev)
    scans = scans.reshape(Bmax, steps, -1, 3)
    n_raw = scans.shape[2]
    torch.cuda.synchronize()

    def contexts(B):
        cs = [_lib.Context(local_map_type=_lib.MAP_KDTREE, height=H, width=W, local_map_size=LM_SIZE,
                           scheme=_lib.SCHEMES["geman_mcclure"], sigma=SIGMA, max_num_alignments=MAX_ALIGN, gn_max_iters=1)
              for _ in range(B)]
        for c in cs:
            c.call("pls_odometry_init")
        return cs

    def run_arm(B, arm, trace=None):
        cs = contexts(B)
        poses = np.zeros((B, steps, 16), np.float32)
        prev = [None] * B
        handles = (C.c_void_p * B)(*[c.handle.value for c in cs])
        layouts = (C.c_int * B)(*([_lib.INPUT_TENSOR | _lib.PTR_DEVICE] * B))
        n = (C.c_int64 * B)(*([n_raw] * B))
        pk, prm = np.zeros((B, 16), np.float32), np.zeros((B, 6), np.float32)
        has, info, status = np.zeros(B, np.int32), np.zeros((B, 12)), np.zeros(B, np.int32)

        outs = [(np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)) for _ in range(B)]
        out_args = [(_lib.ptr(p), _lib.ptr(pr), C.byref(h), _lib.ptr(inf)) for p, pr, inf, h in outs]

        def one(i, k):
            cs[i].call("pls_process_frame_grid_sample", scans[i, k].data_ptr(), n_raw, VOXEL, _lib.INPUT_TENSOR,
                       _lib.ptr(prev[i]), *out_args[i])
            poses[i, k] = outs[i][0]
            if outs[i][3].value:
                prev[i] = outs[i][0].reshape(4, 4).copy()

        if arm == "threaded":   # one thread per sequence for the whole run; the main thread only opens the window
            bar = threading.Barrier(B + 1)

            def worker(i):
                for k in range(args.warmup):
                    one(i, k)
                cs[i].call("pls_synchronize")
                bar.wait()
                bar.wait()
                for k in range(args.warmup, steps):
                    one(i, k)
                cs[i].call("pls_synchronize")

            ts = [threading.Thread(target=worker, args=(i,)) for i in range(B)]
            for t in ts:
                t.start()
            bar.wait()
            l0 = C.c_int64(0)
            lib.pls_launch_count(C.byref(l0))
            t0 = time.perf_counter()
            bar.wait()
            for t in ts:
                t.join()
            t = time.perf_counter() - t0
            l1 = C.c_int64(0)
            lib.pls_launch_count(C.byref(l1))
            for c in cs:
                c.close()
            return B * args.steps / t, (l1.value - l0.value) / args.steps, poses

        def step(k):
            if arm == "sequential":
                for i in range(B):
                    one(i, k)
            else:
                data = (C.c_void_p * B)(*[scans[i, k].data_ptr() for i in range(B)])
                inits = (C.c_void_p * B)(*[None if prev[i] is None else _lib.ptr(prev[i]) for i in range(B)])
                st = cs[0].process_frames(handles, B, data, layouts, n, VOXEL, inits, _lib.ptr(pk), _lib.ptr(prm),
                                          _lib.ptr(has), _lib.ptr(info), _lib.ptr(status))
                assert st == _lib.PLS_OK, (st, lib.pls_last_error(cs[0].handle))
                for i in range(B):
                    poses[i, k] = pk[i]
                    if has[i]:
                        prev[i] = pk[i].reshape(4, 4).copy()

        for k in range(args.warmup):
            step(k)
        for c in cs:
            c.call("pls_synchronize")
        l0 = C.c_int64(0)
        lib.pls_launch_count(C.byref(l0))
        if trace:
            os.environ["PLS_BATCH_TRACE"] = trace
        t0 = time.perf_counter()
        for k in range(args.warmup, steps):
            step(k)
        for c in cs:
            c.call("pls_synchronize")
        t = time.perf_counter() - t0
        os.environ.pop("PLS_BATCH_TRACE", None)
        l1 = C.c_int64(0)
        lib.pls_launch_count(C.byref(l1))
        for c in cs:
            c.close()
        return B * args.steps / t, (l1.value - l0.value) / args.steps, poses

    rows = []
    for B in batches:
        res = {arm: [] for arm in ("sequential", "threaded", "batched")}
        launches, poses = {}, {}
        for _ in range(args.passes):
            for arm in res:
                fps, lps, ps = run_arm(B, arm)
                res[arm].append(fps)
                launches[arm] = lps
                poses[arm] = ps
        identical = all(poses[a].tobytes() == poses["sequential"].tobytes() for a in poses)
        row = {"B": B, "identical_poses": identical}
        for arm, v in res.items():
            row[arm] = {"frames_per_s": float(np.median(v)), "passes": [float(x) for x in v], "launches_per_step": launches[arm]}
        row["batched_over_sequential"] = row["batched"]["frames_per_s"] / row["sequential"]["frames_per_s"]
        row["batched_over_threaded"] = row["batched"]["frames_per_s"] / row["threaded"]["frames_per_s"]
        path = os.path.join(tempfile.mkdtemp(), "trace.jsonl")
        fps, _, ps = run_arm(B, "batched", trace=path)
        lines = [json.loads(line) for line in open(path)]
        assert len(lines) == args.steps and ps.tobytes() == poses["batched"].tobytes()
        row["phases_per_step"] = {"frames_per_s_traced": fps, **{
            key: float(np.median([ln[key] for ln in lines])) for key in ("input_ms", "icp_ms", "epilogue_ms", "call_ms")},
            "extra_rounds_per_step": float(np.mean([ln["extra_rounds"] for ln in lines]))}
        print(json.dumps(row), flush=True)
        rows.append(row)
    result = {"workload": "cfg2 x B sequences (bench.py constants), raw scans in HBM, sequence i from frame 200 i",
              "steps": args.steps, "warmup": args.warmup, "device": device_info(0), "rows": rows}
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result["device"]))


if __name__ == "__main__":
    main()
