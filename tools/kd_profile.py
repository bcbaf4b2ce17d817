"""Development helper: in-pipeline (L2-warm) CUDA-event times of the single kernels of the cfg2 frame
(profile slots 6..15), one slot per pass so that the event records of one kernel do not perturb another.
Slot 0 covers every ICP iteration; 7 / 9 / 10 are the three kernels of a frame's first iteration, 11 the one kernel of
each later iteration."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import pylidar_slam_b200 as b200
from pylidar_slam_b200 import _lib, synthetic as syn

H, W, F, WARM = 64, 2048, 44, 24
scans = [syn.scan(k, H, W) for k in range(F)]
dev = torch.device("cuda", 0)
dscans = torch.from_numpy(np.stack(scans)).to(dev)
names = {0: "icp iteration (all)", 3: "index build", 4: "grid sample", 7: "nn search", 9: "normals", 10: "residual+solve",
         11: "later iteration"}
for slot in (int(a) for a in (sys.argv[1:] or ["0", "3", "4", "7", "9", "10", "11"])):
    cfg = b200.ICPFrameToModelConfig(local_map=b200.KdTreeLocalMapConfig(local_map_size=20),
        alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)),
        max_num_alignments=10, data_key="input_data")
    algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0), device=dev)
    algo.init()
    ctx = algo.ctx
    pose, params, info, has = np.zeros((4, 4), np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    prev, iters = None, 0
    for k in range(F):
        if k == WARM:
            ctx.call("pls_synchronize")
            ctx.call("pls_profile_enable", slot, 1)
        ctx.call("pls_process_frame_grid_sample", dscans[k].data_ptr(), scans[k].shape[0], 0.3, _lib.INPUT_TENSOR, _lib.ptr(prev),
                 _lib.ptr(pose), _lib.ptr(params), C.byref(has), _lib.ptr(info))
        if has.value:
            prev = pose.copy()
        if k >= WARM:
            iters += int(info[0])
    ms, n, _ = ctx.profile(slot)
    frames = F - WARM
    print(f"slot {slot:2d} {names.get(slot, ''):22s} {1e3 * ms / frames:8.1f} us/frame  {n} scopes  ({iters / frames:.2f} iterations/frame)")
