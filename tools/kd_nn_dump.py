"""Development helper: KdTreeLocalMap.nearest_neighbor_search (points and normals) on a cfg2-sized map -- 20 frames of
the synthetic 64x2048 stream, grid-sampled at 0.3 -- queried with the next frame's samples, saved to an .npz; or two
such files compared bit for bit.  Checks that a change of the kd search kernels leaves their results unchanged.

    python tools/kd_nn_dump.py [--root TREE] OUT.npz     (TREE: the checkout whose built package is used)
    python tools/kd_nn_dump.py --compare A.npz B.npz
"""
import argparse
import os
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
ap.add_argument("out", nargs="?")
args = ap.parse_args()

if args.compare:
    a, b = (np.load(f) for f in args.compare)
    same = True
    for k in sorted(a.files):
        eq = a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes()
        same &= eq
        print(f"{k}: {a[k].shape} {'identical' if eq else 'DIFFERENT'}")
    print("identical" if same else "DIFFERENT")
    sys.exit(0 if same else 1)

sys.path.insert(0, os.path.abspath(args.root))
import pylidar_slam_b200 as b200  # noqa: E402
from pylidar_slam_b200 import synthetic as syn  # noqa: E402

H, W, FRAMES, VOXEL = 64, 2048, 20, 0.3
lm = b200.KdTreeLocalMap(b200.KdTreeLocalMapConfig(local_map_size=FRAMES))
lm.init()
for k in range(FRAMES):
    s, _ = b200.grid_sample(syn.scan(k, H, W), VOXEL)
    rel = np.eye(4, dtype=np.float32) if k == 0 else syn.gt_relative_pose(k).astype(np.float32)
    lm.update(rel[None], new_pc_data=np.ascontiguousarray(s, dtype=np.float32))
q, _ = b200.grid_sample(syn.scan(FRAMES, H, W), VOXEL)
q = np.ascontiguousarray(q, dtype=np.float32)
res = lm.nearest_neighbor_search(q)
np.savez(args.out, queries=q, points=res.neighbor_points, normals=res.neighbor_normals)
print(f"map {lm.num_points()} points, {q.shape[0]} queries -> {args.out} (package from {b200.__file__})")
