"""Development helper: where the time of the kd residual-and-solve phase goes, per ICP iteration of the cfg2 frame.

Builds the library with -DPLS_KD_SPLIT into a scratch directory (the default build compiles no stamp) and runs the
frames of tools/kd_profile.py.  kd_residual_kernel (a frame's first iteration) and kd_icp_refine_kernel (each later
one) then write %globaltimer stamps per block: start, start of the residual phase, the block's last thread done with
its loads / its fp64 accumulation, block partial stored, ticket taken; the last block also: rows summed, solve done,
pose written.  kd_normals_warp_kernel stamps its end, so the gap before the first iteration's kernel is seen too.
Prints the median over frames of each interval, in microseconds.  Two passes: without CUDA events, and with the
events of profile slots 10 and 11 (what tools/kd_profile.py reports), so that both can be set side by side.

    python tools/kd_residual_split.py [--src REPO] [--lib PATH] [--frames 44]
"""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITERS, BLOCKS, STAMPS = 8, 8 * 132, 12  # KD_SPLIT_ITERS, KD_SPLIT_BLOCKS, KD_SPLIT_STAMPS
WORDS = (ITERS + 1) * BLOCKS * 2 * STAMPS


def build(src_root, out_dir):
    import importlib.util
    spec = importlib.util.spec_from_file_location("_pls_build", os.path.join(src_root, "pylidar_slam_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    csrc = os.path.join(src_root, "pylidar_slam_b200", "csrc")
    srcs = sorted(f for f in os.listdir(csrc) if f.endswith(".cu"))
    procs, objs = [], []
    for s in srcs:
        obj = os.path.join(out_dir, s[:-3] + ".o")
        procs.append(subprocess.Popen([b.NVCC, *b.FLAGS, "-DPLS_KD_SPLIT", "-c", os.path.join(csrc, s), "-o", obj]))
        objs.append(obj)
    if any(p.wait() for p in procs):
        raise SystemExit("nvcc failed")
    lib = os.path.join(out_dir, "libplslam_b200_split.so")
    subprocess.check_call([b.NVCC, "-shared", "-o", lib, *objs, *b.GENCODE, "-ldl"])
    return lib


def med(v):
    v = sorted(v)
    return v[len(v) // 2] if v else float("nan")


def analyse(rec, normals_end):
    """rec: [ITERS + 1][BLOCKS][2 * STAMPS] u64 of one frame -> {kind: {interval: us}} (kind: first / later<i> / noop)."""
    import numpy as np
    out, prev_end = {}, normals_end
    for slot in range(ITERS + 1):
        r = rec[slot]
        live = r[:, 0] != 0
        if not live.any():
            continue
        g = r[live, :STAMPS].astype(np.int64)
        c = r[live, STAMPS:].astype(np.int64)
        t0 = int(g[:, 0].min())
        d = {"gap before (previous kernel's end -> first block start)": (t0 - prev_end) / 1e3 if prev_end else float("nan"),
             "block starts spread (first -> last block start)": (g[:, 0].max() - t0) / 1e3}
        if slot == ITERS:
            out["noop"] = d
            continue
        us = lambda a, b: float(np.median(g[:, b] - g[:, a])) / 1e3  # noqa: E731  (median over blocks)
        mx = lambda a, b: float(np.max(g[:, b] - g[:, a])) / 1e3  # noqa: E731  (slowest block)
        names = ["start -> residual phase start", "residual phase start -> loads done", "loads done -> accumulation done",
                 "accumulation done -> partial stored (shuffle reduce)", "partial stored -> ticket taken (fence + atomic)"]
        for i, nm in enumerate(names):
            d["per block: " + nm] = us(i, i + 1)
        for i, nm in enumerate(names):
            d["slowest block: " + nm] = mx(i, i + 1)
        late = int(np.argmax(g[:, 5]))  # the block whose ticket came last
        for i, nm in enumerate(names):
            d["block with the last ticket: " + nm] = (g[late, i + 1] - g[late, i]) / 1e3
        d["blocks whose ticket came more than 10 us after the first block start"] = float(np.sum(g[:, 5] - t0 > 10000))
        sm = g[:, 11] - 1
        _, inv, cnt = np.unique(sm, return_inverse=True, return_counts=True)
        d["blocks on an SM that runs another block of the launch"] = float(np.sum(cnt[inv] > 1))
        d["block with the last ticket: blocks of the launch on its SM"] = float(cnt[inv[late]])
        d["block with the last ticket: blockIdx.x (of gridDim.x - 1)"] = float(np.nonzero(live)[0][late])
        d["gridDim.x - 1"] = float(len(g) - 1)
        if slot > 0:  # stamps 9 / 10 of kd_icp_refine_kernel are counts: re-searched queries, normals computed
            slow = int(np.argmax(g[:, 1] - g[:, 0]))
            d["re-searched queries per block (median)"] = float(np.median(g[:, 9]))
            d["re-searched queries per block (max)"] = float(np.max(g[:, 9]))
            d["normals computed per block (median)"] = float(np.median(g[:, 10]))
            d["normals computed per block (max)"] = float(np.max(g[:, 10]))
            d["block with the longest search phase: re-searched queries"] = float(g[slow, 9])
            d["block with the longest search phase: normals computed"] = float(g[slow, 10])
        d["first block start -> last block's start of residual phase"] = (g[:, 1].max() - t0) / 1e3
        d["first block start -> last ticket taken"] = (g[:, 5].max() - t0) / 1e3
        last = np.nonzero(g[:, 6])[0]
        if len(last):
            L, cl = g[last[0]], c[last[0]]
            d["last block: ticket -> rows summed"] = (L[6] - L[5]) / 1e3
            d["last block: rows summed -> solve done"] = (L[7] - L[6]) / 1e3 if L[7] else float("nan")
            d["last block: solve done -> pose written"] = (L[8] - L[7]) / 1e3 if L[7] and L[8] else float("nan")
            d["last block: rows summed -> pose written"] = (L[8] - L[6]) / 1e3 if L[8] else float("nan")
            d["last block: rows summed -> solve done (SM cycles)"] = float(cl[7] - cl[6]) if L[7] else float("nan")
            d["last block: solve done -> pose written (SM cycles)"] = float(cl[8] - cl[7]) if L[7] and L[8] else float("nan")
            d["TOTAL first block start -> pose written"] = (L[8] - t0) / 1e3 if L[8] else float("nan")
            prev_end = int(L[8]) if L[8] else int(L[6])
        out["first" if slot == 0 else f"later{slot}"] = d
    return out


def run(lib, frames, warm, events):
    import ctypes as C
    import numpy as np
    import torch
    os.environ["PLS_LIB_PATH"] = lib
    sys.path.insert(0, ROOT)
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import _lib, synthetic as syn
    H, W = 64, 2048
    scans = [syn.scan(k, H, W) for k in range(frames)]
    dev = torch.device("cuda", 0)
    dscans = torch.from_numpy(np.stack(scans)).to(dev)
    cfg = b200.ICPFrameToModelConfig(local_map=b200.KdTreeLocalMapConfig(local_map_size=20),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
        max_num_alignments=10, data_key="input_data")
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0), device=dev)
    algo.init()
    ctx = algo.ctx
    fn = ctx.lib.pls_debug_kd_split
    fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p, C.c_int64], C.c_int
    buf = np.zeros(WORDS + 1, np.uint64)
    pose, params, info, has = np.zeros((4, 4), np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    prev, per_frame, iters = None, [], 0
    for k in range(frames):
        if k == warm:
            ctx.call("pls_synchronize")
            if events:
                for s in (10, 11):
                    ctx.profile(s)
                    ctx.call("pls_profile_enable", s, 1)
        ctx.call("pls_process_frame_grid_sample", dscans[k].data_ptr(), scans[k].shape[0], 0.3, _lib.INPUT_TENSOR, _lib.ptr(prev),
                 _lib.ptr(pose), _lib.ptr(params), C.byref(has), _lib.ptr(info))
        if has.value:
            prev = pose.copy()
        _lib.check(ctx.handle, fn(ctx.handle, buf.ctypes.data, WORDS + 1))
        if k >= warm:
            iters += int(info[0])
            rec = buf[:WORDS].reshape(ITERS + 1, BLOCKS, 2 * STAMPS)
            per_frame.append(analyse(rec, int(buf[WORDS])))
    n = frames - warm
    ev = {s: 1e3 * ctx.profile(s)[0] / n for s in (10, 11)} if events else None
    return per_frame, iters / n, ev


def report(per_frame, iters, ev, title):
    print(f"## {title}: {len(per_frame)} frames, {iters:.2f} ICP iterations per frame")
    if ev:
        print(f"CUDA events: slot 10 (first iteration's kd_residual_kernel) {ev[10]:.1f} us/frame, "
              f"slot 11 (later iterations, no-op launches included) {ev[11]:.1f} us/frame")
    kinds = sorted({k for f in per_frame for k in f}, key=lambda k: (k != "first", k == "noop", k))
    for kind in kinds:
        rows = [f[kind] for f in per_frame if kind in f]
        print(f"# {kind}: {len(rows)} launches in {len(per_frame)} frames (medians over launches, us unless stated)")
        for key in rows[0]:
            print(f"  {key:70s} {med([r[key] for r in rows]):9.2f}")
    later = [sum(f[k]["TOTAL first block start -> pose written"] + max(f[k]["gap before (previous kernel's end -> first block start)"], 0)
                 for k in f if k.startswith("later")) for f in per_frame]
    print(f"# per frame: later iterations, gap + start -> pose written, summed: median {med(later):.2f} us")
    noop = [f["noop"]["gap before (previous kernel's end -> first block start)"] + f["noop"]["block starts spread (first -> last block start)"]
            for f in per_frame if "noop" in f]
    if noop:
        print(f"# per frame with a no-op launch ({len(noop)} of {len(per_frame)}): gap + block starts spread, median {med(noop):.2f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=ROOT, help="repository whose sources are built (default: this one)")
    ap.add_argument("--lib", help="an already built -DPLS_KD_SPLIT library")
    ap.add_argument("--frames", type=int, default=44)
    ap.add_argument("--warmup", type=int, default=24)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="kd_split_") as tmp:
        lib = a.lib or build(os.path.abspath(a.src), tmp)
        import torch
        print(f"# {torch.cuda.get_device_name(0)}; library {os.path.basename(lib)} built from {os.path.basename(os.path.abspath(a.src))}")
        for events in (False, True):
            pf, it, ev = run(lib, a.frames, a.warmup, events)
            report(pf, it, ev, "with CUDA events of slots 10 and 11" if events else "no CUDA events")


if __name__ == "__main__":
    main()
