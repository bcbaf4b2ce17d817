"""The eigenvalue-thresholded solve of register_new_frames (pls_register_scans_degeneracy) on the H100.

  (a) whole-call time: register_new_frames of B 0.3 m-sampled scans of 32 768 rows near the truth (within 0.5 m and 3
      degrees) on the scene map, B in (1, 8, 64, 512), max_distance 1 m, with min_eigenvalue 1e-3 against without it,
      with the iteration counts and degenerate counts of both;
  (b) the tunnel and flat-field scenes (oracle/degeneracy_reference.py): the final pose errors along and across the
      degenerate directions, with and without the threshold.
Every shape is warmed up first; the two calls alternate within each repetition and medians are reported.  The
eigen-solve runs inside the last block of each iteration's correspondence kernel, so its own time per iteration
cannot be separated from a whole call: it is reported as not measured, beside the whole-call difference.  The card's
name, power limit and max SM clock are read in the same run.

    python tools/degeneracy_bench.py --out profiles/h100_degeneracy.json [--reps 7]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from evaluate_poses_bench import card, scene_cloud, scans_of  # noqa: E402
from gated_registration_bench import odometry, poses, set_map, timed  # noqa: E402

THRESHOLD = 1e-3
GATE = 1.0
AXES = ["x", "y", "z", "roll", "pitch", "yaw"]


def scene_errors(odo, m, s, truth, start, thr, degenerate_axes):
    """Final pose errors of the plain and the thresholded call: along the degenerate directions against the start
    (what the threshold holds), across them against the truth."""
    from oracle import degeneracy_reference as dr
    out = {}
    for label, e in (("plain", 0.0), ("thresholded", thr)):
        _, T, _, it = odo.register_new_frames([s], start[None], max_distance=GATE, min_eigenvalue=e)
        p, p0, pt = dr.euler(T[0]), dr.euler(start), dr.euler(truth)
        across = [i for i in range(6) if i not in degenerate_axes]
        out[label] = dict(
            status=int(odo.last_registrations_status[0]), iterations=int(it[0]),
            degenerate=None if e == 0 else int(odo.last_registrations_degenerate[0]),
            along_from_start={AXES[i]: float(p[i] - p0[i]) for i in degenerate_axes},
            along_from_truth={AXES[i]: float(p[i] - pt[i]) for i in degenerate_axes},
            across_translation_error_m=float(np.abs(p[[i for i in across if i < 3]] -
                                                    pt[[i for i in across if i < 3]]).max()),
            across_rotation_error_rad=float(np.abs(p[[i for i in across if i >= 3]] -
                                                   pt[[i for i in across if i >= 3]]).max()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_degeneracy.json"))
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    from oracle import degeneracy_reference as dr
    res = {"card": card(), "reps": args.reps, "threshold": THRESHOLD, "max_distance": GATE, "calls": [],
           "eigen_solve_per_iteration": "not measured: it runs in the tail of each iteration's last block and cannot "
                                        "be separated from the whole call",
           "scenes": {}}
    scene = scene_cloud()
    odo = odometry(10)
    set_map(odo, scene)
    for B in (1, 8, 64, 512):
        S = min(B, 64)
        scans = scans_of(scene, S, 32768, B)
        of = np.arange(B, dtype=np.int32) % S
        T0 = poses(B, B, (0.0, 0.5), 3.0)
        for e in (0.0, THRESHOLD):   # warm-up of both
            odo.register_new_frames(scans, T0, of, max_distance=GATE, min_eigenvalue=e)
        t = {0.0: [], THRESHOLD: []}
        for _ in range(args.reps):
            for e in (0.0, THRESHOLD):
                dt, _ = timed(lambda: odo.register_new_frames(scans, T0, of, max_distance=GATE, min_eigenvalue=e))
                t[e].append(dt)
        _, Tp, _, ip = odo.register_new_frames(scans, T0, of, max_distance=GATE)
        _, Td, _, idg = odo.register_new_frames(scans, T0, of, max_distance=GATE, min_eigenvalue=THRESHOLD)
        plain, thr = float(np.median(t[0.0])), float(np.median(t[THRESHOLD]))
        res["calls"].append(dict(
            map="scene", B=B, rows=32768, plain_ms=1e3 * plain, thresholded_ms=1e3 * thr, ratio=thr / plain,
            plain_ms_spread=[1e3 * float(min(t[0.0])), 1e3 * float(max(t[0.0]))],
            thresholded_ms_spread=[1e3 * float(min(t[THRESHOLD])), 1e3 * float(max(t[THRESHOLD]))],
            mean_iters_plain=float(np.mean(ip)), mean_iters_thresholded=float(np.mean(idg)),
            whole_call_difference_per_iteration_us=1e6 * (thr - plain) / float(np.max(idg)),
            registrations_with_degenerate_directions=int(np.sum(odo.last_registrations_degenerate > 0)),
            min_eigenvalue_over_n=float(odo.last_registrations_eigenvalues[:, 0].min()),
            max_pose_diff_m=float(np.abs(Tp[:, :3, 3] - Td[:, :3, 3]).max())))
        print(res["calls"][-1], flush=True)
    for name, scene_fn, thr, axes in (("tunnel", dr.tunnel_scene, dr.TUNNEL_MIN_EIGENVALUE, [0]),
                                      ("flat_field", dr.flat_field_scene, dr.FLAT_MIN_EIGENVALUE, [0, 1, 5])):
        m, s, truth, start = scene_fn()
        so = odometry(30, scheme="default")
        set_map(so, m)
        res["scenes"][name] = dict(min_eigenvalue=thr, **scene_errors(so, m, s, truth, start, thr, axes))
        print(name, res["scenes"][name], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
