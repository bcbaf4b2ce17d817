"""The cost of the kd map's normals as num_neighbors_normals grows, on the cfg2 workload (bench.py's constants:
synthetic 64x2048 scans grid-sampled at 0.3 m, a 20-frame kd map, point-to-plane GN geman_mcclure 0.3, <= 10
alignments, constant-velocity initialisation).  Per k:

  * fps                 frames per second of ICPFrameToModel.process_next_frame over --frames frames after --warmup,
                        host clock around calls that return the pose (each ends in a device synchronisation);
  * normals_ms          device time of the normals launches per frame (CUDA events of profile slot 9), and
    normals_per_frame   normals computed per frame (PLS_KD_STATS: one (k+1)-NN search per normal), both from a
                        separate run with the events and the counters on;
  * later_iter_ms       the time of one ICP iteration after a frame's first: on the map the stream holds after 20
                        frames, pls_register_frame of the next frame's samples with max_num_alignments = 6 and 1
                        (threshold_delta_pose 0, the index rebuilt before each call so that no normal is cached),
                        (t6 - t1) / 5, median of --reps.  k <= 31 runs them in kd_icp_refine_kernel, larger k in the
                        four launches verify / 1-NN / normals / residual.

    python tools/kd_wide_normals_bench.py [--ks 10,31,32,64,127,255] [--out profiles/h100_kd_wide_normals.json]
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
import bench  # noqa: E402  (the workload's constants)

PROFILE_NORMALS = 9


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def frames(n):
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    return [np.ascontiguousarray(b200.grid_sample(syn.scan(f, bench.H, bench.W), bench.VOXEL)[0]) for f in range(n)]


def make_algo(k, stats):
    """A cfg2 odometry at k; stats: its map counts the (k+1)-NN searches (PLS_KD_STATS is read when a map is set up)."""
    import pylidar_slam_b200 as b200
    if not stats:
        os.environ.pop("PLS_KD_STATS", None)
    else:
        os.environ["PLS_KD_STATS"] = "1"
    proj = b200.SphericalProjector(height=bench.H, width=bench.W, up_fov=3.0, down_fov=-24.0)
    cfg = b200.ICPFrameToModelConfig(
        local_map=b200.KdTreeLocalMapConfig(local_map_size=bench.LM_SIZE, num_neighbors_normals=k),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme=bench.SCHEME, sigma=bench.SIGMA,
                                                                              max_iters=1)),
        max_num_alignments=bench.MAX_ALIGN, data_key="numpy_pc")
    algo = b200.ICPFrameToModel(cfg, projector=proj, device="cuda:0")
    algo.init()
    return algo


def run_stream(algo, fr, warm, on_timed=None):
    prev, iters = None, 0
    t0 = None
    for i, s in enumerate(fr):
        if i == warm:
            if on_timed:
                on_timed()
            t0 = time.perf_counter()
        d = {"numpy_pc": s, "init_rpose": prev}
        algo.process_next_frame(d)
        if "odometry_pose" in d:
            prev = d["odometry_pose"].astype(np.float64)
        if i >= warm:
            iters += int(algo.last_info[0])
    return time.perf_counter() - t0, iters


def later_iteration_ms(k, m, q, T0, reps):
    from pylidar_slam_b200 import _lib as lib
    os.environ.pop("PLS_KD_STATS", None)
    out = {}
    for j in (1, 6):
        ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=1, num_neighbors_normals=k,
                          scheme=lib.SCHEMES[bench.SCHEME], sigma=bench.SIGMA, gn_max_iters=1, max_num_alignments=j,
                          threshold_delta_pose=0.0)
        T, params, losses, it = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(j, np.float32), C.c_int(0)
        ts = []
        for r in range(reps + 1):
            ctx.call("pls_kdmap_update_points", lib.ptr(np.eye(4, dtype=np.float32)), lib.ptr(m), m.shape[0])
            t = time.perf_counter()
            ctx.call("pls_register_frame", lib.ptr(q), q.shape[0], lib.ptr(T0.reshape(16)), lib.ptr(T), lib.ptr(params),
                     lib.ptr(losses), C.byref(it))
            if r:
                ts.append(time.perf_counter() - t)
        ctx.close()
        out[j] = float(np.median(ts)) * 1e3
    return (out[6] - out[1]) / 5, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="10,31,32,64,127,255")
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_kd_wide_normals.json"))
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import _lib as lib, synthetic as syn
    fr = frames(a.warmup + a.frames)
    # the map the stream holds after 20 frames and the next frame's samples, 0.3 m / 1 degree off its true pose
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=bench.LM_SIZE))
    lm.init()
    for f in range(20):
        rel = np.eye(4, dtype=np.float32) if f == 0 else syn.gt_relative_pose(f).astype(np.float32)
        lm.update(rel[None], new_pc_data=fr[f] if f < len(fr) else frames(f + 1)[f])
    m = np.ascontiguousarray(lm.points())
    lm.ctx.close()
    q = fr[20] if len(fr) > 20 else frames(21)[20]
    from scipy.spatial.transform import Rotation
    P = np.eye(4)
    P[:3, :3] = Rotation.from_rotvec(np.radians(1.0) * np.array([0.0, 0.6, 0.8])).as_matrix()
    P[:3, 3] = [0.3, 0.0, 0.0]
    T0 = np.ascontiguousarray((syn.gt_relative_pose(20).astype(np.float64) @ P).astype(np.float32))
    rows = []
    for k in [int(x) for x in a.ks.split(",")]:
        algo = make_algo(k, stats=False)
        secs, iters = run_stream(algo, fr, a.warmup)
        algo.ctx.close()
        algo = make_algo(k, stats=True)
        marks = {}

        def start():
            algo.ctx.call("pls_profile_enable", PROFILE_NORMALS, 1)
            algo.ctx.profile(PROFILE_NORMALS)
            st = np.zeros(16, np.uint64)
            algo.ctx.call("pls_kdmap_stats", lib.ptr(st))
            marks["stats"] = st.astype(np.int64)
        run_stream(algo, fr, a.warmup, start)
        nms, nlaunch, _ = algo.ctx.profile(PROFILE_NORMALS)
        st = np.zeros(16, np.uint64)
        algo.ctx.call("pls_kdmap_stats", lib.ptr(st))
        normals = int(st.astype(np.int64)[4] - marks["stats"][4])
        algo.ctx.close()
        later, parts = later_iteration_ms(k, m, q, T0, a.reps)
        row = dict(k=k, fps=a.frames / secs, ms_per_frame=secs * 1e3 / a.frames, icp_iters_per_frame=iters / a.frames,
                   normals_ms_per_frame=nms / a.frames, normals_launches_per_frame=nlaunch / a.frames,
                   normals_per_frame=normals / a.frames, later_iter_ms=later, register_ms_1_and_6_iters=parts,
                   later_path="kd_icp_refine_kernel" if k <= 31 else "four launches (kd_normals_wide_kernel)")
        print(json.dumps(row), flush=True)
        rows.append(row)
    res = dict(tool="tools/kd_wide_normals_bench.py", card=card(), map_points=int(m.shape[0]), queries=int(q.shape[0]),
               frames=a.frames, warmup=a.warmup, reps=a.reps, rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print("card:", res["card"], "->", a.out)


if __name__ == "__main__":
    main()
