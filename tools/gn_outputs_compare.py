"""Compares the stand-alone alignments of two builds of libplslam_b200.so bit for bit (GPU).

Each build runs in a subprocess of its own, importing its own package, and dumps:
  * pls_align_p2plane / pls_align_p2point at the point counts of tests/test_next_rows_edges_gpu.py (GN_SIZES), every
    scheme, float32 and float64, one step and four steps (norm_stop 1e-9), with and without an initial estimate:
    dT, x, loss and the status;
  * the poses of the ICP loop with several Gauss-Newton steps per alignment (the tests/golden/icp_gn.npz
    configurations: kd map 3 steps, projective map 2 steps), which calls pls_align_p2plane once per step.

    python tools/gn_outputs_compare.py --base path/to/parent/checkout [--out compare.log]

The parent checkout needs its pylidar_slam_b200 package with the library built, and its oracle/.
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GN_SIZES = [1, 2, 255, 256, 257, 67583, 67584, 67585, 300007]
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]


def _data(n):
    """tests/test_next_rows_edges_gpu.py _gn_data."""
    from oracle import next_rows_reference as nrr
    rs = np.random.RandomState(n % 100003)
    tgt = rs.uniform(-20, 20, (n, 3))
    T = nrr.build_pose([0.05, -0.03, 0.02, 0.004, -0.003, 0.005])
    ref = tgt @ T[:3, :3].T + T[:3, 3] + rs.normal(0, 0.05, (n, 3))
    nrm = rs.normal(0, 1, (n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return ref, tgt, nrm


def dump(path, root):
    sys.path.insert(0, root)
    import torch
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import _lib
    from pylidar_slam_b200 import synthetic as syn
    ctx = _lib.Context()
    lib = ctx.lib
    out = {}
    p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    x0 = np.array([0.01, -0.02, 0.015, 0.002, -0.001, 0.003])
    for n in GN_SIZES:
        ref64, tgt64, nrm64 = _data(n)
        for dt in (np.float32, np.float64):
            ref, tgt, nrm = (np.ascontiguousarray(a, dt) for a in (ref64, tgt64, nrm64))
            for cost in ("plane", "point"):
                for sch in SCHEMES:
                    for iters in (1, 4):
                        for init in (None, np.ascontiguousarray(x0, dt)):
                            dT, x, loss = np.zeros(16, dt), np.zeros(6, dt), np.zeros(n, dt)
                            common = (int(dt == np.float64), _lib.SCHEMES[sch], 0.3, iters, 1e-9, p(init), p(dT), p(x),
                                      p(loss))
                            if cost == "plane":
                                st = lib.pls_align_p2plane(ctx.handle, p(ref), p(tgt), p(nrm), n, *common)
                            else:
                                st = lib.pls_align_p2point(ctx.handle, p(ref), p(tgt), n, *common)
                            key = f"{cost}_{sch}_{np.dtype(dt).name}_n{n}_it{iters}_{'x0' if init is not None else 'zero'}"
                            out[key + "_status"] = np.array(st)
                            if st == _lib.PLS_OK or st == _lib.PLS_W_TINY_RESIDUAL:
                                out[key + "_dT"], out[key + "_x"], out[key + "_loss"] = dT, x, loss
    H, W = 32, 512
    for name, lm, key, gn_iters in (("kd_gn3", "kdtree", "numpy_pc", 3), ("proj_gn2", "projective", "vertex_map", 2)):
        lmc = b200.KdTreeLocalMapConfig(local_map_size=4) if lm == "kdtree" else b200.ProjectiveLocalMapConfig(local_map_size=4)
        cfg = b200.ICPFrameToModelConfig(
            local_map=lmc, alignment=b200.GaussNewtonPointToPlaneConfig(gauss_newton_config=dict(
                scheme="geman_mcclure", sigma=0.3, max_iters=gn_iters, norm_stop_criterion=1e-9)),
            max_num_alignments=5, data_key=key, threshold_delta_pose=0.0)
        algo = b200.ICPFrameToModel(cfg, projector=b200.SphericalProjector(height=H, width=W, up_fov=3.0, down_fov=-24.0),
                                    pose=b200.Pose("euler"), device="cuda:0")
        algo.init()
        prev, poses = None, []
        for k in range(6):
            pc = syn.scan(k, H, W)
            if key == "numpy_pc":
                dd = {"numpy_pc": b200.grid_sample(pc, 0.4)[0]}
            else:
                dd = {"vertex_map": torch.from_numpy(syn.vertex_map_from_scan(pc, H, W))}
            dd["init_rpose"] = prev
            algo.process_next_frame(dd)
            if "odometry_pose" in dd:
                poses.append(dd["odometry_pose"].copy())
                prev = dd["odometry_pose"].astype(np.float64)
        out[f"icp_{name}_poses"] = np.stack(poses)
    ctx.close()
    np.savez(path, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="checkout of the parent commit, library built")
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", help=argparse.SUPPRESS)
    ap.add_argument("--root", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.dump:
        dump(a.dump, a.root)
        return 0
    tmp = tempfile.mkdtemp(prefix="gn_compare_")
    files = {}
    for label, root in (("base", os.path.abspath(a.base)), ("new", ROOT)):
        env = {k: v for k, v in os.environ.items() if k != "PLS_LIB_PATH"}
        files[label] = os.path.join(tmp, f"{label}.npz")
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", files[label], "--root", root], env=env,
                              cwd=root)
    base, new = np.load(files["base"]), np.load(files["new"])
    lines = []
    bad = 0
    if set(base.files) != set(new.files):
        bad += 1
        lines.append(f"KEYS DIFFER: {sorted(set(base.files) ^ set(new.files))[:10]}")
    keys = sorted(set(base.files) & set(new.files))
    for k in keys:
        if not np.array_equal(base[k], new[k], equal_nan=True) or base[k].dtype != new[k].dtype:
            bad += 1
            lines.append(f"DIFFERS {k} max|d| = {np.abs(base[k].astype(np.float64) - new[k].astype(np.float64)).max()}")
    n_align = sum(k.endswith("_status") for k in keys)
    n_err = sum(k.endswith("_status") and int(base[k]) not in (0, 4) for k in keys)
    lines.append(f"{n_align} single-entry-point alignments ({n_err} ending in the reference's RuntimeError, status "
                 f"compared), {sum(k.startswith('icp_') for k in keys)} ICP pose sequences; {len(keys)} arrays compared, "
                 f"{bad} differ")
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
