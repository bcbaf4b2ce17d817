"""Per-frame GPU timeline of the cfg2 frame call (pls_process_frame_grid_sample on the kd map): where the main stream
waits before its first ICP kernel, and the gaps between the kernels of both streams.

    python tools/frame_timeline.py [--frames 64] [--warmup 24]

Same workload, stream set-up and warm-up as bench.py's `value`.  The kernel and copy records come from torch.profiler
(CUPTI activity records of every kernel, copy and memset of the process, on both of the library's streams); they need no
change to the library.  Tracing adds host time per launch, so the host-bound intervals read longer than in an untraced
run: the host phases are therefore taken from a second, untraced pass with PLS_HOST_TRACE=1 (printed by the library to
stderr every 64 frames).

Per frame, the median over the timed frames of:
  grid sample      first grid-sample kernel start -> grid-sample selection end (main stream)
  gs kernels       the summed device time of the grid-sample kernels and memsets in that span (the rest of the span
                   is launch latency and idle time between them), then each op's own median below the table
  input stage      grid-sample selection end -> frame_begin_kernel end (main stream)
  map branch       first map-update op start -> kd_finalize_kernel end (map stream; the previous frame's map update)
  map ready -> ICP kd_finalize_kernel end -> first ICP kernel start: the main stream's idle time after the map is ready
  input -> ICP     frame_begin_kernel end -> first ICP kernel start
  ICP              first ICP kernel start -> last ICP kernel end
  ICP -> next      last ICP kernel end -> the next frame's first op (the pose sync and the next call's host work)
  frame            first op of a frame -> first op of the next frame
and the median gap from one op's end to the next op's start on each stream inside a frame, with the op counts.
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import tempfile

os.environ.setdefault("PLS_HOST_TRACE", "1")  # read when the library loads
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import pylidar_slam_b200 as b200
from pylidar_slam_b200 import _lib, synthetic as syn

H, W, VOXEL = 64, 2048, 0.3


def make_algo(dev, stream):
    cfg = b200.ICPFrameToModelConfig(local_map=b200.KdTreeLocalMapConfig(local_map_size=20),
                                     alignment=b200.GaussNewtonPointToPlaneConfig(
                                         gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
                                     max_num_alignments=10, data_key="input_data")
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0),
                                device=dev, stream=stream.cuda_stream)
    algo.init()
    return algo


def run_frames(algo, dscans, n_raw, first, last):
    ctx = algo.ctx
    pose, params, info, has = np.zeros((4, 4), np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    prev = getattr(algo, "_timeline_prev", None)
    for k in range(first, last):
        ctx.call("pls_process_frame_grid_sample", dscans[k].data_ptr(), n_raw, VOXEL, _lib.INPUT_TENSOR, _lib.ptr(prev),
                 _lib.ptr(pose), _lib.ptr(params), C.byref(has), _lib.ptr(info))
        if has.value:
            prev = pose.copy()
    algo._timeline_prev = prev
    ctx.call("pls_synchronize")


def ops_of(trace):
    ops = []
    for e in trace["traceEvents"]:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        ops.append({"name": e["name"], "cat": e["cat"], "t0": float(e["ts"]), "t1": float(e["ts"]) + float(e["dur"]),
                    "stream": e.get("args", {}).get("stream")})
    ops.sort(key=lambda o: o["t0"])
    return ops


def has(o, s):
    return s in o["name"]


def analyse(ops):
    main_s = {o["stream"] for o in ops if has(o, "frame_begin_kernel")}
    map_s = {o["stream"] for o in ops if has(o, "kd_finalize_kernel")}
    assert len(main_s) == 1 and len(map_s) == 1, (main_s, map_s)
    main_s, map_s = main_s.pop(), map_s.pop()
    main = [o for o in ops if o["stream"] == main_s]
    mapq = [o for o in ops if o["stream"] == map_s]
    # a frame on the main stream starts at its grid sample's first kernel (the bucket path's gs_hash_bins_kernel, or
    # voxel_hash_kernel in front of the radix sort) and its sample ends with the selection
    starts = [i for i, o in enumerate(main) if has(o, "voxel_hash_kernel") or has(o, "gs_hash_bins_kernel")]
    rows, gaps_main, gaps_map, n_main, n_map, gs_ops = [], [], [], [], [], {}
    prev_icp0 = None
    for a, b in zip(starts[:-1], starts[1:]):
        fr = main[a:b]
        nxt = main[b]
        ib = [i for i, o in enumerate(fr) if has(o, "frame_begin_kernel")]
        if len(ib) != 1:
            continue
        ib = ib[0]
        sel = [o for o in fr[:ib] if has(o, "GridSampleSelect") or has(o, "gs_bucket_select_kernel")]
        gs_end = max(o["t1"] for o in sel)
        gs = [o for o in fr[:ib] if o["t1"] <= gs_end]
        for o in gs:
            m = re.search(r"(\w+_kernel)", o["name"]) if o["cat"] == "kernel" else None
            short = m.group(1) if m else o["cat"]
            gs_ops.setdefault(short, []).append(o["t1"] - o["t0"])
        icp = fr[ib + 1:]
        icp_k = [o for o in icp if o["cat"] == "kernel"]
        if not icp_k:
            continue
        t_icp0 = icp_k[0]["t0"]
        t_icp1 = max(o["t1"] for o in icp_k)
        # the map update this frame's ICP waited for: the map-stream ops between the previous frame's ICP and this one's
        upd = [o for o in mapq if prev_icp0 is not None and prev_icp0 < o["t0"] < t_icp0]
        prev_icp0 = t_icp0
        fin = [o for o in upd if has(o, "kd_finalize_kernel")]
        row = {"grid sample": gs_end - fr[0]["t0"], "gs kernels": sum(o["t1"] - o["t0"] for o in gs),
               "input stage": fr[ib]["t1"] - gs_end,
               "input -> ICP": t_icp0 - fr[ib]["t1"], "ICP": t_icp1 - t_icp0, "ICP -> next": nxt["t0"] - t_icp1,
               "frame": nxt["t0"] - fr[0]["t0"]}
        if fin:
            row["map branch"] = fin[-1]["t1"] - upd[0]["t0"]
            row["map ready -> ICP"] = t_icp0 - fin[-1]["t1"]
            row["map end - input end"] = fin[-1]["t1"] - fr[ib]["t1"]
            gaps_map += [q["t0"] - p["t1"] for p, q in zip(upd[:-1], upd[1:])]
            n_map.append(len(upd))
        rows.append(row)
        seq = fr[:ib + 1]
        gaps_main += [q["t0"] - p["t1"] for p, q in zip(seq[:-1], seq[1:])]
        gaps_main += [q["t0"] - p["t1"] for p, q in zip(icp[:-1], icp[1:])]
        n_main.append(len(fr))
    return rows, gaps_main, gaps_map, n_main, n_map, gs_ops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=24)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    p = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        smi = f"nvidia-smi unavailable: {e}"
    print(f"# device: {p.name}; nvidia-smi: {smi}")
    F = args.warmup + 1 + args.frames
    scans = [syn.scan(k, H, W) for k in range(F)]
    n_raw = scans[0].shape[0]
    dscans = torch.from_numpy(np.stack(scans)).to(dev)
    stream = torch.cuda.Stream(dev)

    # pass 1, untraced: the library's host trace (stderr) over the timed frames
    print("# pass 1 (untraced): PLS_HOST_TRACE lines follow on stderr", flush=True)
    algo = make_algo(dev, stream)
    run_frames(algo, dscans, n_raw, 0, args.warmup + 1)
    run_frames(algo, dscans, n_raw, args.warmup + 1, F)
    sys.stderr.flush()

    # pass 2, traced: the GPU timeline of the timed frames
    algo = make_algo(dev, stream)
    run_frames(algo, dscans, n_raw, 0, args.warmup + 1)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_frames(algo, dscans, n_raw, args.warmup + 1, F)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "t.pt.trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    rows, gm, gp, nm, np_, gs_ops = analyse(ops_of(trace))
    print(f"# pass 2 (torch.profiler): {len(rows)} frames of {args.frames} timed; medians in microseconds")
    keys = ["grid sample", "gs kernels", "input stage", "map branch", "map end - input end", "map ready -> ICP", "input -> ICP", "ICP",
            "ICP -> next", "frame"]
    for k in keys:
        v = [r[k] for r in rows if k in r]
        if v:
            print(f"{k:22s} median {np.median(v):8.1f}   p10 {np.percentile(v, 10):8.1f}   p90 {np.percentile(v, 90):8.1f}")
    print(f"main stream: {np.median(nm):.1f} ops per frame, median gap between consecutive ops {np.median(gm):.2f} us "
          f"(input chain and ICP chain)")
    for name, v in gs_ops.items():
        print(f"  grid-sample op {name:34s} {len(v) / len(rows):4.1f} per frame, median {np.median(v):7.2f} us")
    if gp:
        print(f"map stream:  {np.median(np_):.1f} ops per update, median gap between consecutive ops {np.median(gp):.2f} us")


if __name__ == "__main__":
    main()
