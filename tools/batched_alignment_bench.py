"""Batched alignment vs a loop of single alignments, on the GPU (point-to-plane, float32, geman_mcclure 0.3).

For each shape (B, N) and max_iters in {1, 5} (norm_stop 0, so every iteration runs in both arms):
  * batch: one pls_align_p2plane_batch call on the B correspondence sets;
  * loop:  B pls_align_p2plane calls, one per set.
The arms alternate; each is the median of three timed passes after a warm-up, host clock around calls that end in
their own synchronisation.  Inputs are resident on the device, except for the `host` shape, whose arrays are pageable
host memory (so both arms include the PCIe transfer).  At max_iters = 1 the script checks that both arms agree bit
for bit.  Bytes per iteration are counted by formula (inputs 36 B + loss 4 B per point, 240 B per block partial
written and read) and set against the H100 SXM data sheet's 3.35 TB/s of HBM3 -- a whole-call rate, not a kernel's.

With --base CHECKOUT, the single call at B = 1 is also timed with the parent checkout's library, in separate processes
alternating with this build's (three rounds), to show the B = 1 path did not regress.

    python tools/batched_alignment_bench.py --out profiles/h100_batched_alignment.json [--base path/to/parent]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1, 65536, "device"), (16, 65536, "device"), (256, 4096, "device"), (4096, 256, "device"),
          (256, 4096, "host")]
DATASHEET_HBM = 3.35e12  # B/s, H100 SXM data sheet
GN_THREADS, NUM_SMS = 256, 132


def blocks_per_element(n):
    return max(1, min((n + GN_THREADS - 1) // GN_THREADS, 2 * NUM_SMS))


def bytes_per_iteration(B, n):
    return B * (n * 40 + blocks_per_element(n) * 480)


def make_inputs(B, n, where, seed=0):
    import torch
    g = torch.Generator().manual_seed(seed)
    tgt = torch.rand(B, n, 3, generator=g) * 40 - 20
    nrm = torch.randn(B, n, 3, generator=g)
    nrm /= nrm.norm(dim=-1, keepdim=True)
    ref = tgt + 0.05 * torch.randn(B, n, 3, generator=g) + torch.randn(B, 1, 3, generator=g) * 0.05
    if where == "device":
        return [t.contiguous().cuda() for t in (ref, tgt, nrm)]
    return [np.ascontiguousarray(t.numpy()) for t in (ref, tgt, nrm)]


def _addr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _out(B, n, where):
    import torch
    if where == "device":
        return [torch.empty(s, device="cuda") for s in ((B, 16), (B, 6), (B, n))]
    return [np.empty(s, np.float32) for s in ((B, 16), (B, 6), (B, n))]


def arms(lib, h, B, n, where, iters):
    ref, tgt, nrm = make_inputs(B, n, where)
    ob, ol = _out(B, n, where), _out(B, n, where)
    it = C.c_int(0)
    stride3, stride16, stride6, stride_n = n * 3 * 4, 16 * 4, 6 * 4, n * 4

    def batch():
        st = lib.pls_align_p2plane_batch(h, _addr(ref), _addr(tgt), _addr(nrm), B, n, 0, 5, 0.3, iters, 0.0, None,
                                         _addr(ob[0]), _addr(ob[1]), _addr(ob[2]), C.byref(it))
        assert st == 0, st

    def loop():
        r0, t0, n0 = _addr(ref), _addr(tgt), _addr(nrm)
        d0, x0, l0 = _addr(ol[0]), _addr(ol[1]), _addr(ol[2])
        for b in range(B):
            st = lib.pls_align_p2plane(h, r0 + b * stride3, t0 + b * stride3, n0 + b * stride3, n, 0, 5, 0.3, iters,
                                       0.0, None, d0 + b * stride16, x0 + b * stride6, l0 + b * stride_n)
            assert st == 0, st

    return batch, loop, ob, ol


def timed(fn, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps * 1e3


def reps_for(fn, target_s=0.15, cap=200):
    t0 = time.perf_counter()
    fn()
    dt = time.perf_counter() - t0
    return int(max(1, min(cap, target_s / max(dt, 1e-6))))


def measure(lib, h):
    import torch
    rows = []
    for B, n, where in SHAPES:
        for iters in (1, 5):
            batch, loop, ob, ol = arms(lib, h, B, n, where, iters)
            for _ in range(3):          # warm-up: module load, staging buffers sized
                batch()
                loop()
            torch.cuda.synchronize()
            rb, rl = reps_for(batch), reps_for(loop)
            tb, tl = [], []
            for _ in range(3):          # alternate the arms
                tb.append(timed(batch, rb))
                tl.append(timed(loop, rl))
            same = None
            if iters == 1:
                same = all(np.array_equal(np.asarray(a.cpu() if hasattr(a, "cpu") else a),
                                          np.asarray(b.cpu() if hasattr(b, "cpu") else b)) for a, b in zip(ob, ol))
                assert same, (B, n, where)
            mb, ml = statistics.median(tb), statistics.median(tl)
            bpi = bytes_per_iteration(B, n)
            rows.append(dict(B=B, N=n, inputs=where, max_iters=iters, batch_ms=round(mb, 4), loop_ms=round(ml, 4),
                             batch_passes_ms=[round(v, 4) for v in tb], loop_passes_ms=[round(v, 4) for v in tl],
                             speedup=round(ml / mb, 3), batch_alignments_per_s=round(B / mb * 1e3, 1),
                             loop_alignments_per_s=round(B / ml * 1e3, 1), bytes_per_iteration=bpi,
                             batch_share_of_datasheet_hbm=round(bpi * iters / (mb * 1e-3) / DATASHEET_HBM, 4),
                             bit_identical_at_one_iteration=same))
            print(json.dumps(rows[-1]), flush=True)
            del batch, loop, ob, ol
            torch.cuda.empty_cache()
    return rows


def single_b1(reps_rounds=3):
    """Median of three passes of pls_align_p2plane at N = 65536 on device inputs, max_iters 1 and 5 (this process's
    package, i.e. whichever checkout is first on sys.path)."""
    import torch
    from pylidar_slam_b200 import _lib
    ctx = _lib.Context()
    out = {}
    for iters in (1, 5):
        ref, tgt, nrm = make_inputs(1, 65536, "device")
        d, x, l = _out(1, 65536, "device")

        def one():
            st = ctx.lib.pls_align_p2plane(ctx.handle, _addr(ref), _addr(tgt), _addr(nrm), 65536, 0, 5, 0.3, iters, 0.0,
                                           None, _addr(d), _addr(x), _addr(l))
            assert st == 0
        for _ in range(5):
            one()
        torch.cuda.synchronize()
        r = reps_for(one)
        out[f"max_iters_{iters}_ms"] = round(statistics.median(timed(one, r) for _ in range(reps_rounds)), 4)
    ctx.close()
    return out


def gpu_identity():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"not read ({e})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--base", default=None, help="parent checkout with its library built")
    ap.add_argument("--single-b1", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--root", default=ROOT, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.single_b1:
        sys.path.insert(0, a.root)
        print(json.dumps(single_b1()))
        return 0
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from pylidar_slam_b200 import _lib
    ctx = _lib.Context()
    result = {"what": "pls_align_p2plane_batch (one call) vs a loop of pls_align_p2plane calls; point-to-plane, "
                      "float32, geman_mcclure 0.3, norm_stop 0; median of 3 alternating passes after warm-up",
              **gpu_identity(), "rows": measure(ctx.lib, ctx.handle)}
    ctx.close()
    if a.base:
        rounds = []
        for _ in range(3):
            for label, root in (("parent", os.path.abspath(a.base)), ("this", ROOT)):
                env = {k: v for k, v in os.environ.items() if k != "PLS_LIB_PATH"}
                o = subprocess.run([sys.executable, os.path.abspath(__file__), "--single-b1", "--root", root],
                                   capture_output=True, text=True, env=env, cwd=root, check=True).stdout
                rounds.append({"build": label, **json.loads(o.strip().splitlines()[-1])})
        result["single_call_b1_n65536_parent_vs_this"] = rounds
        for k in ("max_iters_1_ms", "max_iters_5_ms"):
            for label in ("parent", "this"):
                v = [r[k] for r in rounds if r["build"] == label]
                result.setdefault("single_call_b1_summary", {})[f"{label}_{k}"] = {"median": statistics.median(v),
                                                                                   "min": min(v), "max": max(v)}
    print(json.dumps({k: v for k, v in result.items() if k != "rows"}, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
