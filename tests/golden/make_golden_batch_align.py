"""Goldens of the two Gauss-Newton alignments on BATCHES of correspondence sets (B > 1 in one call), from the
UNMODIFIED reference under oracle/ref_shims.py.  Build container only:

    python tests/golden/make_golden_batch_align.py -> batch_align.npz
    python tests/golden/make_golden_batch_align.py --check   # regenerate in memory, compare with the committed file
                                                             # bit for bit, write nothing

GaussNewton.compute (slam/common/optimization.py:296-344) couples the elements of a batch: the tiny-residual guard and
the stop test take norms over the whole batch, and one singular element fails the call.  Cases (`cost` is plane or
point, `dt` f32 or f64):
  ba_sch_*       one step, both costs x the seven schemes x both dtypes, B = 3, 4, 5 (scheme by scheme)
  ba_multi_*     up to 8 iterations (max_iters = k for k = 1..8) on elements whose own alignments would converge
                 at different iterations; ba_multi_*_single_x: each element aligned on its own (max_iters = 8)
  ba_x0_*        initial estimates as [B,6] parameters and as [B,4,4] float32 matrices
  ba_zero_*      one element with zero residuals beside live ones (raises where its weights or Jacobian vanish)
  ba_allzero_*   every residual zero: the warning, x unchanged, loss = r^2
  ba_degen_*     one element whose target points all lie at the origin: the reference raises
"""
import logging
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

torch.set_num_threads(1)
ns = ref_shims.load_reference(kdtree_workers=-1)
pose = ns.pose.Pose("euler")
SCHEMES = ["default", "huber", "exp", "neighborhood", "geman_mcclure", "square_geman_mcclure", "cauchy"]
DTYPES = {"f32": torch.float32, "f64": torch.float64}
SCALE = torch.tensor([0.05, 0.05, 0.05, 0.005, 0.005, 0.005], dtype=torch.float64)


class _Warnings(logging.Handler):
    count = 0

    def emit(self, record):
        if "residual norm is lower" in record.getMessage():
            _Warnings.count += 1


logging.getLogger().addHandler(_Warnings())


def scene(B, N, seed, pose_scale, noise):
    """[B,N,3] target points, unit reference normals, per-element poses (pose_scale[b] x SCALE) and reference points."""
    g = torch.Generator().manual_seed(seed)
    tgt = torch.randn(B, N, 3, generator=g, dtype=torch.float64) * 10.0
    nrm = torch.randn(B, N, 3, generator=g, dtype=torch.float64)
    nrm /= nrm.norm(dim=-1, keepdim=True)
    xs = torch.randn(B, 6, generator=g, dtype=torch.float64) * SCALE * torch.as_tensor(pose_scale, dtype=torch.float64)[:, None]
    ref = pose.apply_transformation(tgt, xs) + torch.as_tensor(noise, dtype=torch.float64)[:, None, None] * \
        torch.randn(B, N, 3, generator=g, dtype=torch.float64)
    return tgt, nrm, ref


def aligner(cost, **gn):
    if cost == "plane":
        return ns.alignment.GaussNewtonPointToPlaneAlignment(
            ns.alignment.GaussNewtonPointToPlaneConfig(gauss_newton_config=gn), pose=pose)
    return ns.alignment.GaussNewtonPointToPointAlignment(ns.alignment.GNPointToPointConfig(gauss_newton_config=gn), pose=pose)


def run(cost, ref, tgt, nrm, x0=None, **gn):
    """(dT, x, loss, raised, warned) of one reference call."""
    al = aligner(cost, **gn)
    before = _Warnings.count
    try:
        if cost == "plane":
            dT, x, loss = al.align(ref, tgt, nrm, initial_estimate=x0)
        else:
            dT, x, loss = al.align(ref, tgt, initial_estimate=x0)
    except RuntimeError as e:
        assert "Invalid Jacobian" in str(e), e
        return None, None, None, True, False
    return dT.detach().numpy(), x.detach().numpy(), loss.detach().numpy(), False, _Warnings.count > before


out = {}
# ---- one step: both costs x seven schemes x both dtypes at B = 3..5
tgt, nrm, ref = scene(5, 400, 11, [1.0, 2.0, 0.5, 1.5, 3.0], [0.01, 0.02, 0.005, 0.01, 0.03])
out.update(ba_sch_tgt=tgt.numpy(), ba_sch_nrm=nrm.numpy(), ba_sch_ref=ref.numpy())
for i, sch in enumerate(SCHEMES):
    B = 3 + i % 3
    for dn, dt in DTYPES.items():
        for cost in ("plane", "point"):
            dT, x, loss, raised, warned = run(cost, ref[:B].to(dt), tgt[:B].to(dt), nrm[:B].to(dt), scheme=sch, sigma=0.3,
                                              max_iters=1)
            assert not raised and not warned
            out[f"ba_sch_{cost}_{sch}_{dn}_dT"], out[f"ba_sch_{cost}_{sch}_{dn}_x"] = dT, x
            out[f"ba_sch_{cost}_{sch}_{dn}_loss"] = loss

# ---- several iterations: elements 0 and 2 near noise-free, small poses (their own alignments converge within a few
# steps), 1 and 3 noisy, large poses.  Not noise-free: the robust weight sqrt(cost(r)) / max(|r|, 1e-4) vanishes with r,
# and with it det H -- one such element would make the whole batch raise.
for cost in ("plane", "point"):
    tgt, nrm, ref = scene(4, 500, 12, [0.5, 6.0, 2.0, 4.0], [0.003, 0.05, 0.003, 0.02])
    out.update({f"ba_multi_{cost}_tgt": tgt.numpy(), f"ba_multi_{cost}_nrm": nrm.numpy(), f"ba_multi_{cost}_ref": ref.numpy()})
    for dn, dt in DTYPES.items():
        xs = []
        for k in range(1, 9):
            dT, x, loss, raised, warned = run(cost, ref.to(dt), tgt.to(dt), nrm.to(dt), scheme="geman_mcclure", sigma=0.3,
                                              max_iters=k, norm_stop_criterion=1e-6)
            assert not raised and not warned, (cost, dn, k)
            xs.append(x)
        out[f"ba_multi_{cost}_{dn}_x"] = np.stack(xs)
        out[f"ba_multi_{cost}_{dn}_dT"], out[f"ba_multi_{cost}_{dn}_loss"] = dT, loss   # of max_iters = 8
        single = [run(cost, ref[b:b + 1].to(dt), tgt[b:b + 1].to(dt), nrm[b:b + 1].to(dt), scheme="geman_mcclure",
                      sigma=0.3, max_iters=8, norm_stop_criterion=1e-6)[1][0] for b in range(4)]
        out[f"ba_multi_{cost}_{dn}_single_x"] = np.stack(single)

# ---- initial estimates: [B,6] parameters and [B,4,4] float32 matrices
tgt, nrm, ref = scene(3, 300, 13, [1.0, 2.0, 3.0], [0.01, 0.01, 0.01])
g = torch.Generator().manual_seed(14)
x0 = (torch.randn(3, 6, generator=g, dtype=torch.float64) * SCALE).to(torch.float32)
mats = pose.build_pose_matrix(x0)
out.update(ba_x0_tgt=tgt.numpy(), ba_x0_nrm=nrm.numpy(), ba_x0_ref=ref.numpy(), ba_x0_x0=x0.numpy(), ba_x0_mats=mats.numpy())
for cost in ("plane", "point"):
    for form, init in (("vec", x0), ("mat", mats)):
        dT, x, loss, raised, warned = run(cost, ref.float(), tgt.float(), nrm.float(), x0=init, scheme="huber", sigma=0.3,
                                          max_iters=3, norm_stop_criterion=1e-9)
        assert not raised and not warned
        out[f"ba_x0_{cost}_{form}_dT"], out[f"ba_x0_{cost}_{form}_x"], out[f"ba_x0_{cost}_{form}_loss"] = dT, x, loss

# ---- one zero-residual element beside live ones: no warning.  With unit weights it is solved (dx = 0) with the others;
# a robust weight is 0 at r = 0 (and the point-to-point Jacobian r dr/dx is 0), so its H is singular and the call raises
tgt, nrm, ref = scene(3, 300, 15, [1.0, 1.0, 1.0], [0.01, 0.01, 0.01])
ref[1] = tgt[1]
out.update(ba_zero_tgt=tgt.numpy(), ba_zero_nrm=nrm.numpy(), ba_zero_ref=ref.numpy())
for dn, dt in DTYPES.items():
    for sch in ("default", "geman_mcclure"):
        dT, x, loss, raised, warned = run("plane", ref.to(dt), tgt.to(dt), nrm.to(dt), scheme=sch, sigma=0.3, max_iters=2,
                                          norm_stop_criterion=1e-9)
        assert not warned
        out[f"ba_zero_plane_{sch}_{dn}_raises"] = np.array(raised)
        if not raised:
            out[f"ba_zero_plane_{sch}_{dn}_dT"], out[f"ba_zero_plane_{sch}_{dn}_x"] = dT, x
            out[f"ba_zero_plane_{sch}_{dn}_loss"] = loss
    out[f"ba_zero_point_{dn}_raises"] = np.array(run("point", ref.to(dt), tgt.to(dt), None, scheme="default", max_iters=2)[3])

# ---- every residual zero: the warning, x unchanged, loss = r^2 = 0
out["ba_allzero_tgt"] = tgt.numpy()
for dn, dt in DTYPES.items():
    for cost in ("plane", "point"):
        dT, x, loss, raised, warned = run(cost, tgt.to(dt), tgt.to(dt), nrm.to(dt), scheme="huber", sigma=0.3, max_iters=3)
        assert not raised and warned
        out[f"ba_allzero_{cost}_{dn}_dT"], out[f"ba_allzero_{cost}_{dn}_x"] = dT, x
        out[f"ba_allzero_{cost}_{dn}_loss"] = loss
        out[f"ba_allzero_{cost}_{dn}_warned"] = np.array(warned)

# ---- one degenerate element (all its target points at the origin): the whole call raises
tgt, nrm, ref = scene(3, 300, 16, [1.0, 1.0, 1.0], [0.01, 0.01, 0.01])
tgt[2] = 0.0   # J = [n or d, (dR_k 0) . (n or d)] = [., 0, 0, 0]: det H = 0 exactly, in float32 as in float64
out.update(ba_degen_tgt=tgt.numpy(), ba_degen_nrm=nrm.numpy(), ba_degen_ref=ref.numpy())
for dn, dt in DTYPES.items():
    for cost in ("plane", "point"):
        out[f"ba_degen_{cost}_{dn}_raises"] = np.array(run(cost, ref.to(dt), tgt.to(dt), nrm.to(dt), scheme="default",
                                                           max_iters=1)[3])

PATH = os.path.join(HERE, "batch_align.npz")
if "--check" in sys.argv[1:]:
    old = np.load(PATH)
    bad = sorted(set(old.files) ^ set(out))
    for k in sorted(set(old.files) & set(out)):
        a, b = old[k], np.asarray(out[k])
        if a.shape != b.shape or a.dtype != b.dtype or not np.array_equal(a, b, equal_nan=a.dtype.kind in "fc"):
            bad.append(k)
    print(f"{len(out)} arrays regenerated, {len(bad)} differ from {os.path.basename(PATH)}", *bad[:20])
    sys.exit(1 if bad else 0)
np.savez_compressed(PATH, **out)
print(len(out), "arrays;", "multi plane f64 x per iteration, element 0:", out["ba_multi_plane_f64_x"][:, 0, 0])
