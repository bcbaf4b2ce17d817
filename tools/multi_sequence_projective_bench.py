"""Aggregate frames/s of B independent projective-map odometry sequences on one GPU: sequential, threaded and batched.

The workload the reference's own benchmark sweeps (projective local map, data_key=vertex_map, the KITTI projector's
64x720 frames), on the synthetic stream: vertex maps resident in HBM, local map of K frames, geman_mcclure sigma 0.3,
<= 10 alignments, constant-velocity initialisation; sequence i starts at synthetic frame 200 i.  For each B the three
arms run alternately in one process, each on fresh contexts:

  sequential  one host thread calls pls_process_frame on each context in turn;
  threaded    B persistent host threads, each driving its own context through every step (ctypes releases the GIL);
  batched     one pls_process_frames call per step.

An arm warms up W steps and times K steps, closed after every context is synchronised; frames/s = B K / time, the median
of 3 passes (every pass listed).  The poses of the three arms are checked bit for bit.  A further batched pass per B
sets PLS_BATCH_TRACE for its timed steps: the per-step split of a batched call into its input stage, its batched ICP
(CUDA events on the lead context's stream), its epilogue (host clock) and the host time of the whole call.

Sections (--sections): `kitti` (--height x --width, --k, every B of --batches), `cfg3` (128x2048, K = 20, B = 1 and 4)
and `sweep` (8 sequences of --height x --width with K in {10, 20, 30} and three schemes, one heterogeneous batch).

    python tools/multi_sequence_projective_bench.py [--sections kitti,cfg3,sweep] [--batches 1,2,4,8,16]
        [--height 64] [--width 720] [--k 20] [--steps 100] [--warmup 24] [--out FILE]
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

MAX_ALIGN, SIGMA = 10, 0.3
SWEEP = [(10, "geman_mcclure"), (20, "cauchy"), (30, "huber"), (10, "cauchy"), (20, "huber"), (30, "geman_mcclure"),
         (20, "geman_mcclure"), (10, "huber")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="kitti,cfg3,sweep")
    ap.add_argument("--batches", default="1,2,4,8,16")
    ap.add_argument("--height", type=int, default=64)
    ap.add_argument("--width", type=int, default=720)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "multi_sequence_projective_bench.py needs a CUDA device"
    from bench import device_info
    from pylidar_slam_b200 import _lib
    from pylidar_slam_b200 import synthetic as syn
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    steps = args.warmup + args.steps
    _maps = {}

    def vertex_maps(H, W, B):
        """[B][steps] device vertex maps, sequence i from synthetic frame 200 i."""
        key = (H, W)
        have = _maps.get(key)
        if have is None or have.shape[0] < B:
            have = torch.from_numpy(np.stack([syn.vertex_map_from_scan(syn.scan(200 * i + k, H, W), H, W)[0]
                                              for i in range(B) for k in range(steps)])).to(dev).reshape(B, steps, 3, H, W)
            _maps[key] = have
            torch.cuda.synchronize()
        return have

    def run_arm(H, W, seqs, arm, trace=None):
        """seqs: [(K, scheme name)] per sequence.  Returns (frames/s, poses)."""
        B = len(seqs)
        vms = vertex_maps(H, W, B)
        cs = [_lib.Context(local_map_type=_lib.MAP_PROJECTIVE, height=H, width=W, local_map_size=k,
                           scheme=_lib.SCHEMES[s], sigma=SIGMA, max_num_alignments=MAX_ALIGN, gn_max_iters=1)
              for k, s in seqs]
        for c in cs:
            c.call("pls_odometry_init")
        poses = np.zeros((B, steps, 16), np.float32)
        prev = [None] * B
        handles = (C.c_void_p * B)(*[c.handle.value for c in cs])
        layouts = (C.c_int * B)(*([_lib.INPUT_VERTEX_MAP] * B))
        n = (C.c_int64 * B)(*([0] * B))
        pk, prm = np.zeros((B, 16), np.float32), np.zeros((B, 6), np.float32)
        has, info, status = np.zeros(B, np.int32), np.zeros((B, 12)), np.zeros(B, np.int32)
        outs = [(np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)) for _ in range(B)]
        out_args = [(_lib.ptr(p), _lib.ptr(pr), C.byref(h), _lib.ptr(inf)) for p, pr, inf, h in outs]

        def one(i, k):
            cs[i].call("pls_process_frame", vms[i, k].data_ptr(), _lib.INPUT_VERTEX_MAP, 0, _lib.ptr(prev[i]), *out_args[i])
            poses[i, k] = outs[i][0]
            if outs[i][3].value:
                prev[i] = outs[i][0].reshape(4, 4).copy()

        def close():
            for c in cs:
                c.close()

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
            t0 = time.perf_counter()
            bar.wait()
            for t in ts:
                t.join()
            t = time.perf_counter() - t0
            close()
            return B * args.steps / t, poses

        def step(k):
            if arm == "sequential":
                for i in range(B):
                    one(i, k)
                return
            data = (C.c_void_p * B)(*[vms[i, k].data_ptr() for i in range(B)])
            inits = (C.c_void_p * B)(*[None if prev[i] is None else _lib.ptr(prev[i]) for i in range(B)])
            st = cs[0].process_frames(handles, B, data, layouts, n, 0.0, inits, _lib.ptr(pk), _lib.ptr(prm),
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
        if trace:
            os.environ["PLS_BATCH_TRACE"] = trace
        t0 = time.perf_counter()
        for k in range(args.warmup, steps):
            step(k)
        for c in cs:
            c.call("pls_synchronize")
        t = time.perf_counter() - t0
        os.environ.pop("PLS_BATCH_TRACE", None)
        close()
        return B * args.steps / t, poses

    def row(H, W, seqs, label):
        B = len(seqs)
        res = {arm: [] for arm in ("sequential", "threaded", "batched")}
        poses = {}
        for _ in range(args.passes):
            for arm in res:
                fps, ps = run_arm(H, W, seqs, arm)
                res[arm].append(fps)
                poses[arm] = ps
        out = {"section": label, "B": B, "shape": [H, W], "sequences": [{"K": k, "scheme": s} for k, s in seqs],
               "identical_poses": all(poses[a].tobytes() == poses["sequential"].tobytes() for a in poses)}
        for arm, v in res.items():
            out[arm] = {"frames_per_s": float(np.median(v)), "passes": [float(x) for x in v]}
        out["batched_over_sequential"] = out["batched"]["frames_per_s"] / out["sequential"]["frames_per_s"]
        out["batched_over_threaded"] = out["batched"]["frames_per_s"] / out["threaded"]["frames_per_s"]
        path = os.path.join(tempfile.mkdtemp(), "trace.jsonl")
        fps, ps = run_arm(H, W, seqs, "batched", trace=path)
        lines = [json.loads(line) for line in open(path)]
        assert len(lines) == args.steps and ps.tobytes() == poses["batched"].tobytes()
        out["phases_per_step"] = {"frames_per_s_traced": fps, **{
            key: float(np.median([ln[key] for ln in lines])) for key in ("input_ms", "icp_ms", "epilogue_ms", "call_ms")},
            "extra_rounds_per_step": float(np.mean([ln["extra_rounds"] for ln in lines]))}
        print(json.dumps(out), flush=True)
        return out

    rows = []
    sections = args.sections.split(",")
    if "kitti" in sections:
        for B in [int(b) for b in args.batches.split(",")]:
            rows.append(row(args.height, args.width, [(args.k, "geman_mcclure")] * B, "kitti"))
    if "cfg3" in sections:
        for B in (1, 4):
            rows.append(row(128, 2048, [(20, "geman_mcclure")] * B, "cfg3"))
    if "sweep" in sections:
        rows.append(row(args.height, args.width, SWEEP, "sweep"))
    result = {"workload": "B projective-map sequences, vertex maps in HBM (data_key=vertex_map), geman_mcclure sigma 0.3 "
                          "unless listed, <= 10 alignments, sequence i from synthetic frame 200 i",
              "steps": args.steps, "warmup": args.warmup, "passes": args.passes,
              "resident_mb_env": os.environ.get("PLS_PROJ_RESIDENT_MB"), "device": device_info(0), "rows": rows}
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result["device"]))


if __name__ == "__main__":
    main()
