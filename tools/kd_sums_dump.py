"""Development helper: the 30 fp64 accumulators and the pose of every kd ICP iteration, to compare two builds bit for bit.

On the cfg2-shaped scene of tests/test_kd_icp_iterations_gpu.py (a 20-frame kd map, the next frame's grid samples as
queries), register calls with max_num_alignments = 1..J on fresh contexts; after each, pls_kdmap_last_correspondences
reads back the accumulators of its last iteration (kd_residual_kernel for j = 1, kd_icp_refine_kernel after), and the
call returns the pose.  Three starting poses and three weight schemes.

    PLS_LIB_PATH=<build A>/libplslam_b200.so python tools/kd_sums_dump.py --out a.npz
    PLS_LIB_PATH=<build B>/libplslam_b200.so python tools/kd_sums_dump.py --out b.npz
    python tools/kd_sums_dump.py --compare a.npz b.npz
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dump(out, iters):
    sys.path.insert(0, ROOT)
    from scipy.spatial.transform import Rotation
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import _lib as lib, synthetic as syn
    lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=20))
    lm.init()
    for k in range(20):
        rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
        s, _ = b200.grid_sample(syn.scan(k, 64, 2048), 0.3)
        lm.update(rel[None], new_pc_data=s)
    m = np.ascontiguousarray(lm.points())
    lm.ctx.close()
    q, _ = b200.grid_sample(syn.scan(20, 64, 2048), 0.3)
    q = np.ascontiguousarray(q)
    T_gt = syn.gt_relative_pose(20)
    res = {}
    for seed, (metres, degrees) in enumerate([(0.3, 1.0), (0.1, 0.3), (0.6, 2.0)]):
        rng = np.random.RandomState(seed)
        axis, d = rng.randn(3), rng.randn(3)
        P = np.eye(4)
        P[:3, :3] = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(degrees)).as_matrix()
        P[:3, 3] = d / np.linalg.norm(d) * metres
        T0 = (np.asarray(T_gt, np.float64) @ P).astype(np.float32)
        for scheme in ("geman_mcclure", "default", "cauchy"):
            for j in range(1, iters + 1):
                ctx = lib.Context(local_map_type=lib.MAP_KDTREE, local_map_size=1, num_neighbors_normals=10,
                                  scheme=lib.SCHEMES[scheme], sigma=0.3, gn_max_iters=1, max_num_alignments=j,
                                  threshold_delta_pose=0.0)
                ctx.call("pls_kdmap_update_points", lib.ptr(np.eye(4, dtype=np.float32)), lib.ptr(m), m.shape[0])
                T, params, losses, it = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(j, np.float32), C.c_int(0)
                ctx.call("pls_register_frame", lib.ptr(q), q.shape[0], lib.ptr(T0.reshape(16)), lib.ptr(T), lib.ptr(params),
                         lib.ptr(losses), C.byref(it))
                sums = np.empty(30, np.float64)
                ctx.call("pls_kdmap_last_correspondences", q.shape[0], None, None, None, None, lib.ptr(sums))
                ctx.close()
                key = f"{seed}_{scheme}_{j}"
                res[key + "_sums"], res[key + "_T"], res[key + "_params"], res[key + "_losses"] = sums, T, params, losses
    np.savez(out, **res)
    print(f"wrote {len(res) // 4} iterations' accumulators and poses to {out}")


def compare(a, b):
    A, B = np.load(a), np.load(b)
    assert sorted(A.files) == sorted(B.files), "different runs"
    diff = [k for k in sorted(A.files) if A[k].tobytes() != B[k].tobytes()]
    n = len(A.files) // 4
    print(f"{n} iterations (accumulators, pose, parameters, losses): "
          + ("identical bit for bit" if not diff else f"{len(diff)} arrays differ: {diff[:10]}"))
    return 1 if diff else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--compare", nargs=2)
    a = ap.parse_args()
    if a.compare:
        return compare(*a.compare)
    dump(a.out, a.iters)
    return 0


if __name__ == "__main__":
    sys.exit(main())
