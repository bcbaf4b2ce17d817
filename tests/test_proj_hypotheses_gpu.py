"""pls_register_hypotheses / ICPFrameToModel.register_new_frame_hypotheses on projective local maps.

The models are built by running the projective odometry (pls_process_frame) over synthetic frames.  The scan is the
newest frame of the model: hypothesis 0 starts on it at the identity (the tiny-residual guard), hypothesis 1 starts 40 m
and 120 degrees away (it diverges or is singular), the others are a yaw sweep of +-10 degrees with offsets up to 2 m.
  * B hypotheses in one call give, per hypothesis, the bits of pls_register_frame with that T0 on the same context (T,
    params, losses, iterations, singular status), and pls_last_icp_sums afterwards is that of a single call with the
    last T0: B = 1, 2, 63, 64, 65 at 64x720 and 128x2048 with K = 20, at K = 1 and 3, on an off-TMA shape (30x100) and
    with PLS_PROJ_NO_TMA (in a subprocess).
  * The map is not changed (model bytes, frame count), and the next frame is bit-identical to a twin context's; a call
    enqueued while a key frame's model rebuild is pending equals single calls after the same update.
  * Refusals leave the context unchanged; one more ICP iteration adds the same launches at B = 1, 8 and 64.
  * Poses agree with the unmodified reference's register_new_frame (tests/golden/proj_hypotheses.npz) within the
    projective 32x512 tolerance of tests/test_gpu_parity.py.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "proj_hypotheses.npz")


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


def _lib_mod():
    from pylidar_slam_b200 import _lib
    return _lib


def make_ctx(lib, H=64, W=720, K=20, **kw):
    args = dict(local_map_type=lib.MAP_PROJECTIVE, height=H, width=W, local_map_size=K,
                scheme=lib.SCHEMES["geman_mcclure"], sigma=0.3, max_num_alignments=10, gn_max_iters=1)
    args.update(kw)
    return lib.Context(**args)


def process(lib, ctx, k, init):
    """pls_process_frame of synthetic frame k (float32 rows on the host): (status, outputs)."""
    from pylidar_slam_b200 import synthetic as syn
    H, W = int(ctx.cfg.height), int(ctx.cfg.width)
    pts = np.ascontiguousarray(syn.scan(k, H, W), np.float32)
    pose, params, info, has = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(12), C.c_int(0)
    st = lib.load().pls_process_frame(ctx.handle, lib.ptr(pts), lib.INPUT_NDARRAY, pts.shape[0], lib.ptr(init),
                                      lib.ptr(pose), lib.ptr(params), C.byref(has), lib.ptr(info))
    return st, dict(pose=pose, params=params, has=np.int32(has.value), info=info)


def warm(lib, ctx, frames, stop_on_keyframe=False):
    """Frames 0 .. frames-1 through the odometry; returns the next frame's index and initial pose."""
    init = None
    k = 0
    while k < frames:
        st, out = process(lib, ctx, k, init)
        assert st == lib.PLS_OK, (k, st)
        if out["has"]:
            init = out["pose"].reshape(4, 4).copy()
        k += 1
        if stop_on_keyframe and k > 3 and out["info"][7] == 1.0:
            break
    return k, init


def newest_frame(lib, ctx):
    H, W = int(ctx.cfg.height), int(ctx.cfg.width)
    vm = np.zeros((3, H, W), np.float32)
    ctx.call("pls_projmap_last_frame", lib.ptr(vm))
    pts = vm.reshape(3, -1).T
    return np.ascontiguousarray(pts[np.abs(pts).max(1) > 0])


def hypotheses(B, seed=0):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    T0s = np.tile(np.eye(4, dtype=np.float32), (B, 1, 1))
    for b in range(1, B):
        far = b == 1
        yaw = 120.0 if far else -10.0 + 20.0 * (b - 2) / max(B - 3, 1)
        T0s[b, :3, :3] = Rotation.from_euler("z", yaw, degrees=True).as_matrix()
        T0s[b, :3, 3] = [40.0, -30.0, 2.0] if far else rng.uniform(-2.0, 2.0, 3) * [1, 1, 0.1]
    return T0s


def call_hypotheses(lib, ctx, scan, T0s):
    B, M = T0s.shape[0], int(ctx.cfg.max_num_alignments)
    T0 = np.ascontiguousarray(T0s, np.float32)
    out = dict(T=np.zeros((B, 16), np.float32), params=np.zeros((B, 6), np.float32),
               losses=np.zeros((B, M), np.float32), iters=np.zeros(B, np.int32), status=np.zeros(B, np.int32))
    rc = lib.load().pls_register_hypotheses(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(T0), B, lib.ptr(out["T"]),
                                            lib.ptr(out["params"]), lib.ptr(out["losses"]), lib.ptr(out["iters"]),
                                            lib.ptr(out["status"]))
    return rc, out


def single(lib, ctx, scan, T0):
    M = int(ctx.cfg.max_num_alignments)
    T, p, losses, iters = np.zeros(16, np.float32), np.zeros(6, np.float32), np.zeros(M, np.float32), C.c_int(0)
    st = lib.load().pls_register_frame(ctx.handle, lib.ptr(scan), scan.shape[0], lib.ptr(np.ascontiguousarray(T0)),
                                       lib.ptr(T), lib.ptr(p), lib.ptr(losses), C.byref(iters))
    return st, T, p, losses, iters.value


def last_sums(lib, ctx):
    sums, iters = np.zeros(30, np.float64), C.c_int(-1)
    st = lib.load().pls_last_icp_sums(ctx.handle, lib.ptr(sums), C.byref(iters))
    return st, sums, iters.value


def model(lib, ctx):
    k = C.c_int(0)
    ctx.call("pls_projmap_num_frames", C.byref(k))
    H, W = int(ctx.cfg.height), int(ctx.cfg.width)
    vm, nm = np.zeros((k.value, 3, H, W), np.float32), np.zeros((k.value, 3, H, W), np.float32)
    if k.value:
        ctx.call("pls_projmap_model", lib.ptr(vm), lib.ptr(nm))
    return k.value, vm.tobytes(), nm.tobytes()


def check_against_singles(lib, ctx, scan, T0s, out, tag=""):
    """Every hypothesis against its own pls_register_frame on ctx, then the last sums against the last single call's."""
    hyp_sums = last_sums(lib, ctx)
    B = T0s.shape[0]
    for b in range(B):
        st, T1, p1, l1, it1 = single(lib, ctx, scan, T0s[b])
        assert (st == lib.PLS_E_SINGULAR) == (out["status"][b] == lib.PLS_E_SINGULAR), (tag, b, st, out["status"][b])
        assert T1.tobytes() == out["T"][b].tobytes(), (tag, b)
        assert p1.tobytes() == out["params"][b].tobytes(), (tag, b)
        assert it1 == out["iters"][b], (tag, b, it1, out["iters"][b])
        assert l1[:it1].tobytes() == out["losses"][b, :it1].tobytes(), (tag, b)
    one_sums = last_sums(lib, ctx)
    assert hyp_sums[0] == one_sums[0] == lib.PLS_OK
    assert hyp_sums[1].tobytes() == one_sums[1].tobytes() and hyp_sums[2] == one_sums[2], tag


# shapes: (H, W, K, warm-up frames)
SHAPES = {"64x720_K20": (64, 720, 20, 26), "128x2048_K20": (128, 2048, 20, 26), "64x720_K1": (64, 720, 1, 4),
          "64x720_K3": (64, 720, 3, 6), "30x100_off_tma": (30, 100, 3, 6)}
_warm_ctx = {}


def warmed(lib, name):
    if name not in _warm_ctx:
        H, W, K, frames = SHAPES[name]
        ctx = make_ctx(lib, H, W, K)
        warm(lib, ctx, frames)
        _warm_ctx[name] = ctx
    return _warm_ctx[name]


def _bit_identity(lib, ctx, B, tag):
    scan = newest_frame(lib, ctx)
    T0s = hypotheses(B, seed=B)
    before = model(lib, ctx)
    rc, out = call_hypotheses(lib, ctx, scan, T0s)
    assert rc == lib.PLS_OK, (tag, rc)
    assert model(lib, ctx) == before, tag
    check_against_singles(lib, ctx, scan, T0s, out, tag)
    assert out["status"][0] == lib.PLS_W_TINY_RESIDUAL, (tag, out["status"][0])
    if B > 1:
        M = int(ctx.cfg.max_num_alignments)
        assert out["status"][1] == lib.PLS_E_SINGULAR or out["iters"][1] == M or \
            np.linalg.norm(out["T"][1].reshape(4, 4)[:3, 3]) > 5.0, (tag, out["status"][1], out["iters"][1])
    if B > 2:
        assert (out["status"][2:] == lib.PLS_OK).any(), tag   # the sweep converges somewhere
    return out


@pytest.mark.parametrize("B", [1, 2, 63, 64, 65])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_bit_identical_to_single_calls(lib, shape, B):
    _bit_identity(lib, warmed(lib, shape), B, (shape, B))


def _no_tma_body():
    lib = _lib_mod()
    ctx = make_ctx(lib, 64, 720, 20)
    warm(lib, ctx, 24)
    for B in (2, 65):
        _bit_identity(lib, ctx, B, ("no_tma", B))
    ctx.close()


def test_without_tma_in_a_subprocess():
    env = dict(os.environ, PLS_PROJ_NO_TMA="1", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_proj_hypotheses_gpu as t; t._no_tma_body(); print('no-tma ok')"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "no-tma ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_next_frame_equals_a_twin_context(lib):
    a, b = make_ctx(lib), make_ctx(lib)
    k, init = warm(lib, a, 22)
    warm(lib, b, 22)
    scan = newest_frame(lib, a)
    rc, _ = call_hypotheses(lib, a, scan, hypotheses(9, seed=1))
    assert rc == lib.PLS_OK
    assert model(lib, a) == model(lib, b)
    for j in range(3):
        sa, oa = process(lib, a, k + j, init)
        sb, ob = process(lib, b, k + j, init)
        assert sa == sb == lib.PLS_OK
        for key in oa:
            assert oa[key].tobytes() == ob[key].tobytes(), (j, key)
        ra, rb = last_sums(lib, a), last_sums(lib, b)
        assert ra[1].tobytes() == rb[1].tobytes() and ra[2] == rb[2], j
        init = oa["pose"].reshape(4, 4).copy()
    assert model(lib, a) == model(lib, b)
    a.close()
    b.close()


def test_pending_model_rebuild_is_waited_for(lib):
    """Straight after a key frame (its model rebuild still pending on the map stream) the hypotheses see the rebuilt
    model, exactly as single calls made after the same frame on a twin context do."""
    a, b = make_ctx(lib), make_ctx(lib)
    k, _ = warm(lib, a, 40, stop_on_keyframe=True)
    warm(lib, b, k)
    from pylidar_slam_b200 import synthetic as syn
    scan = np.ascontiguousarray(syn.scan(k - 1, 64, 720), np.float32)
    T0s = hypotheses(6, seed=2)
    T0s[0] = np.eye(4, dtype=np.float32)
    rc, out = call_hypotheses(lib, a, scan, T0s)
    assert rc == lib.PLS_OK
    n_a = model(lib, a)
    for j in range(T0s.shape[0]):
        st, T1, p1, l1, it1 = single(lib, b, scan, T0s[j])
        assert (st == lib.PLS_E_SINGULAR) == (out["status"][j] == lib.PLS_E_SINGULAR), j
        assert T1.tobytes() == out["T"][j].tobytes() and p1.tobytes() == out["params"][j].tobytes(), j
        assert it1 == out["iters"][j] and l1[:it1].tobytes() == out["losses"][j, :it1].tobytes(), j
    assert n_a == model(lib, b)
    a.close()
    b.close()


def test_refusals_leave_the_context_unchanged(lib):
    ctx = warmed(lib, "64x720_K3")
    scan = newest_frame(lib, ctx)
    single(lib, ctx, scan, np.eye(4, dtype=np.float32))
    before, sums = model(lib, ctx), last_sums(lib, ctx)
    T0s = hypotheses(3)
    for args in [(scan, scan.shape[0], T0s, 0), (scan, 0, T0s, 3)]:
        s, n, T, B = args
        out = np.zeros((max(B, 1), 64), np.float32)
        rc = lib.load().pls_register_hypotheses(ctx.handle, lib.ptr(s), n, lib.ptr(np.ascontiguousarray(T)), B,
                                                lib.ptr(out), None, None, None, None)
        assert rc == lib.PLS_E_INVALID, args[1:]
    assert model(lib, ctx) == before
    after = last_sums(lib, ctx)
    assert after[1].tobytes() == sums[1].tobytes() and after[2] == sums[2]
    gn2 = make_ctx(lib, 64, 720, 3, gn_max_iters=2)
    fresh = make_ctx(lib, 64, 720, 3)
    for c, why in ((gn2, "max_iters == 1"), (fresh, "search before any update")):
        rc, _ = call_hypotheses(lib, c, scan, T0s)
        assert rc == lib.PLS_E_INVALID
        assert why in lib.load().pls_last_error(c.handle).decode()
        assert last_sums(lib, c)[0] == lib.PLS_E_STATE
    gn2.close()
    fresh.close()


def test_later_iteration_launches_do_not_grow_with_B(lib):
    """threshold_delta_pose = 0: every hypothesis runs max_num_alignments iterations.  On the TMA path one more
    iteration is the z-buffer, resolve, correspondence and step launches, whatever B."""
    counts = {}
    for M in (3, 4):
        ctx = make_ctx(lib, 64, 720, 20, max_num_alignments=M, threshold_delta_pose=0.0)
        warm(lib, ctx, 8)
        scan = newest_frame(lib, ctx)
        for B in (1, 8, 64):
            before = ctx.launch_count()
            rc, _ = call_hypotheses(lib, ctx, scan, hypotheses(B, seed=5))
            assert rc == lib.PLS_OK
            counts[B, M] = ctx.launch_count() - before
        ctx.close()
    for B in (1, 8, 64):
        assert counts[B, 4] - counts[B, 3] == 4, counts
        assert counts[B, 3] == counts[1, 3], counts


def test_python_mirror_on_a_projective_odometry(lib):
    import pylidar_slam_b200 as b200
    from pylidar_slam_b200 import synthetic as syn
    proj = b200.SphericalProjector(height=64, width=720, up_fov=3.0, down_fov=-24.0)
    cfg = dict(algorithm="icp_F2M", max_num_alignments=10, data_key="numpy_pc",
               local_map=dict(type="projective_local_map", local_map_size=5),
               alignment=dict(mode="point_to_plane_gauss_newton",
                              gauss_newton_config=dict(scheme="geman_mcclure", sigma=0.3, max_iters=1)))
    odo = b200.ICPFrameToModel(cfg, projector=proj)
    odo.init()
    for k in range(6):
        odo.process_next_frame({"numpy_pc": syn.scan(k, 64, 720)})
    import torch
    scan = syn.scan(6, 64, 720)
    T0s = hypotheses(5, seed=3)
    params, T, losses, iters = odo.register_new_frame_hypotheses(scan, torch.from_numpy(T0s))
    for b in range(5):
        p1, T1, l1 = odo.register_new_frame(scan, T0s[b])
        assert T1.tobytes() == T[b].tobytes() and p1.tobytes() == params[b].tobytes(), b
        assert np.asarray(l1, np.float32).tobytes() == np.asarray(losses[b], np.float32).tobytes(), b


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="no reference data")
def test_poses_against_the_reference():
    """The unmodified reference's register_new_frame on its ProjectiveLocalMap from several T0, against one call, with
    the projective 32x512 tolerance of tests/test_gpu_parity.py: relaxed_tolerance's translation and 1e-5 rad."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conftest import pose_errors
    from test_gpu_parity import relaxed_tolerance
    lib = _lib_mod()
    g = np.load(GOLDEN)
    H, W = int(g["H"]), int(g["W"])
    ctx = make_ctx(lib, H, W, int(g["K"]), max_num_alignments=int(g["M"]))
    rel = g["rel_poses"]
    for k in range(g["vmaps"].shape[0]):
        ctx.call("pls_projmap_update", lib.ptr(np.ascontiguousarray(rel[k])), lib.ptr(np.ascontiguousarray(g["vmaps"][k])))
    rc, out = call_hypotheses(lib, ctx, np.ascontiguousarray(g["scan"]), g["T0s"])
    assert rc == lib.PLS_OK
    tol = relaxed_tolerance("proj_vmap_32x512", 6e-4)
    errs = [pose_errors(out["T"][b], g["T"][b]) for b in range(g["T0s"].shape[0])]
    print("reference pose errors (relative translation, rad):", errs)
    for b, (dt, ang) in enumerate(errs):
        assert dt <= tol and ang <= 1e-5, (b, errs)
    ctx.close()
