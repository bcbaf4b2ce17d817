"""Grid sample, voxel statistics and the kd frame input at the edges of the device primitives under them.

Every frame runs through the single-pass selection (select_device.cuh), the flag scan and the LSD radix sort
(primitives.cu).  They go wrong, if at all, at their edges, so the tests sit there:

  * sizes: one element, a tile (2048) minus one / exactly / plus one, two tiles likewise, SEL_MAX_N (one resident wave
    of selection tiles, 1 081 344) minus one / exactly / plus one, and far beyond it, where the grid sample and the kd
    frame input take the scan path instead of the selection;
  * hashes: distinct voxels with one int64 hash, hashes that wrap the int64 range, the bounds of the 40-bit compact
    sort keys and the first hash beyond them, coordinates exactly on a voxel half;
  * the 10-bit selection epoch: the status words are cleared only when it wraps, every 1023 selections;
  * reused scratch: one context across all sizes, ascending and descending.

References are exact (float64 division, round-half-even, int64 hashes that wrap, a stable sort) and the comparisons are
bit for bit wherever the operation is exact.  The edges below are checked against the CUDA sources by
test_select_scan_sort_edges_cpu.py.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import icp_oracle as orc

pytestmark = pytest.mark.gpu

TILE = 2048                          # SEL_TILE (select_device.cuh) = SCAN_TILE = SORT_TILE (primitives.cu)
NUM_SMS = 132                        # kNumSMs (internal.cuh)
SEL_MAX_N = TILE * 4 * NUM_SMS       # 1 081 344: the largest selection launch (four resident tiles per SM)
EPOCH_CYCLE = 2 ** 10 - 1            # selections per clear of the status words (10-bit epoch, 0 is never used)
COMPACT = 2 ** 39                    # hashes in [-COMPACT, COMPACT) sort on 40-bit keys, others repeat on 64-bit keys
SIZES = [1, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, SEL_MAX_N - 1, SEL_MAX_N, SEL_MAX_N + 1,
         2 * SEL_MAX_N + 7, TILE * TILE]
HX, HY, HZ = orc.HASH_PX, orc.HASH_PY, orc.HASH_PZ
VOXEL = 0.3


@pytest.fixture(scope="module")
def lib():
    from pylidar_slam_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------------------ clouds
_lidar = {}


def _lidar_scan():
    """One 128 x 32768 synthetic scan: 4 194 304 points, the largest size."""
    if "scan" not in _lidar:
        from pylidar_slam_b200 import synthetic as syn
        _lidar["scan"] = syn.scan(7, 128, 32768)
    return _lidar["scan"]


def _lattice(m, rng):
    """m distinct voxel coordinates with distinct hashes (a box of side < 2 * 82: no two of its points are a nonzero
    solution of HX x + HY y + HZ z = 0 apart), in random order."""
    s = int(np.ceil(m ** (1 / 3))) // 2 + 1
    g = np.arange(-s, s)
    box = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    return box[rng.permutation(box.shape[0])[:m]]


def cloud(kind, n, dtype):
    """n points: 'one' all in one voxel, 'own' every point alone in its voxel, 'lidar' a subset of a synthetic scan in
    scan order (voxel VOXEL)."""
    rng = np.random.RandomState(n + (7 if dtype == np.float64 else 0))
    if kind == "one":
        return (rng.uniform(-0.45, 0.45, (n, 3)) * VOXEL).astype(dtype)
    if kind == "own":
        return ((_lattice(n, rng) + rng.uniform(-0.4, 0.4, (n, 3))) * VOXEL).astype(dtype)
    full = _lidar_scan()
    rows = full if n == full.shape[0] else full[np.sort(rng.permutation(full.shape[0])[:n])]
    return rows if dtype == np.float32 else rows.astype(np.float64) * (1.0 + 1e-9)


OCCUPANCY = [1, 2, 31, 32, 33, 63, 64, 65, 100, 257]   # around the 32 lanes of the warp that reduces a voxel


def buckets(n, dtype):
    """n points in voxels holding OCCUPANCY points each (cycled; the last one truncated), rows in random order."""
    rng = np.random.RandomState(n + 3)
    reps = np.resize(OCCUPANCY, n)
    reps = reps[:np.searchsorted(np.cumsum(reps), n) + 1]
    c = np.repeat(_lattice(reps.shape[0], rng), reps, axis=0)[:n]
    return ((c + rng.uniform(-0.4, 0.4, (n, 3))) * VOXEL).astype(dtype)[rng.permutation(n)]


# ------------------------------------------------------------------------------------------------------- hash cases
def egcd(a, b):
    """(g, u, v) with a u + b v = g = gcd(a, b)."""
    if b == 0:
        return a, 1, 0
    g, u, v = egcd(b, a % b)
    return g, v, u - (a // b) * v


def solve_hash(value, span=20000):
    """Integer voxel coordinates (x, y, z) with HX x + HY y + HZ z == value exactly (Python integers, no wrap), the
    largest |coordinate| as small as a search over z near value / HZ finds.  x = (value - HZ z) / HX modulo HY, centred,
    from the extended Euclidean algorithm; the three constants are pairwise coprime."""
    g, u, _ = egcd(HX, HY)
    assert g == 1 and egcd(HX, HZ)[0] == 1 and egcd(HY, HZ)[0] == 1
    inv = u % HY
    best = None
    for z in range(value // HZ - span, value // HZ + span + 1):
        r = value - HZ * z
        x = (r * inv) % HY
        x = x - HY if x > HY // 2 else x
        y = (r - HX * x) // HY
        size = max(abs(x), abs(y), abs(z))
        if best is None or size < best[0]:
            best = (size, (x, y, z))
    x, y, z = best[1]
    assert HX * x + HY * y + HZ * z == value
    return best[1]


def int64_wrap(v):
    """The two's-complement int64 value of an integer (numba's int64 arithmetic wraps like this)."""
    return (v + 2 ** 63) % 2 ** 64 - 2 ** 63


def hash_cases():
    """name -> voxel coordinates (a list of triples).  The true value of every hash is HX x + HY y + HZ z."""
    a = solve_hash(987654321)
    return {
        "compact_min": [solve_hash(-COMPACT)],             # the compact keys' lowest hash
        "compact_max": [solve_hash(COMPACT - 1)],          # ... and highest
        "first_repeat": [solve_hash(COMPACT)],             # the first hash that sends the call to 64-bit keys
        "first_repeat_below": [solve_hash(-COMPACT - 1)],
        "wrap_up": [solve_hash(2 ** 63 + 12345)],          # beyond int64.max: a negative hash
        "wrap_down": [solve_hash(-2 ** 63 - 777)],         # below int64.min: a positive hash
        "collision": [a, (a[0] + HY, a[1] - HX, a[2])],    # two voxels, one true hash value
        "collision_wrap": [(0, 0, 0), solve_hash(2 ** 64)],  # two voxels whose true hashes are 2^64 apart
    }


HASH_VOXEL = 0.5
OFFSETS = np.array([[0.0, 0.0, 0.0], [0.25, -0.25, 0.125], [-0.25, 0.125, -0.25]])   # within the voxel, exact in binary


def case_points(coords, dtype):
    """Three points in each voxel of `coords` (voxel HASH_VOXEL), exact in dtype when |coordinate| < 2^20."""
    c = np.asarray(coords, np.float64)
    return ((c[:, None, :] + OFFSETS[None]) * HASH_VOXEL).reshape(-1, 3).astype(dtype)


def float32_carries(coords):
    return max(abs(v) for t in coords for v in t) < 2 ** 20


def half_points(dtype):
    """Points whose p / voxel is exactly k + 1/2 in float64 (round-half-even decides), negative k included: voxel 0.25
    in either dtype, and voxel 0.3 in float64 where the quotient comes out exact."""
    k = np.arange(-8, 8) + 0.5
    g = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    out = [(g * 0.25).astype(dtype), 0.25]
    if dtype == np.float64:
        p = g * 0.3
        exact = (p / 0.3 == g).all(1)
        out += [p[exact], 0.3]
    return out


# ----------------------------------------------------------------------------------------------------------- calls
def launches(ctx):
    return ctx.launch_count()


def grid_sample(lib, ctx, pts, voxel):
    """pls_grid_sample (device output, copied back by the library)."""
    n = pts.shape[0]
    out, idx, count = np.empty_like(pts), np.empty(n, np.int64), C.c_int64(0)
    ctx.call("pls_grid_sample", lib.ptr(pts), int(pts.dtype == np.float64), n, float(voxel), lib.ptr(out), lib.ptr(idx),
             C.byref(count))
    return out[:count.value], idx[:count.value]


def grid_sample_staged(lib, ctx, pts, voxel):
    """pls_grid_sample_staged into the library's mapped pinned staging (copy_counted_to_host_kernel)."""
    hx, hi, dx, count = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int64(0)
    ctx.call("pls_grid_sample_staged", lib.ptr(pts), int(pts.dtype == np.float64), pts.shape[0], float(voxel), C.byref(hx),
             C.byref(hi), C.byref(dx), C.byref(count))
    S = count.value
    return lib.host_view(hx.value, (S, 3), pts.dtype).copy(), lib.host_view(hi.value, (S,), np.int64).copy()


def check_sample(got, pts, ref_idx, tag):
    s, i = got
    assert i.shape == ref_idx.shape and np.array_equal(i, ref_idx), (tag, i.shape, ref_idx.shape)
    assert s.dtype == pts.dtype and s.tobytes() == pts[ref_idx].tobytes(), tag


# ----------------------------------------------------------------------------------------------- 1. grid sample
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_grid_sample_at_every_size_edge(lib, dtype):
    """Three clouds at every size, through both entry points, ascending then descending on one context (its scratch
    and status words come from a larger earlier call on the way down); bit-exact.  The call leaves the selection for
    head flags + scan + gather exactly above SEL_MAX_N."""
    ctx = lib.Context()
    refs, extra, tails = {}, {}, 0
    for n in SIZES + SIZES[::-1]:
        for kind in ("one", "own", "lidar"):
            pts = cloud(kind, n, dtype)
            if (kind, n) not in refs:
                refs[kind, n] = orc.grid_sample(pts, VOXEL)[1]
                if kind == "one":
                    assert refs[kind, n].tolist() == [0]
                if kind == "own":
                    assert refs[kind, n].shape[0] == n
            ref = refs[kind, n]
            before = launches(ctx)
            check_sample(grid_sample(lib, ctx, pts, VOXEL), pts, ref, (kind, n, "device"))
            extra.setdefault(n, launches(ctx) - before)
            check_sample(grid_sample_staged(lib, ctx, pts, VOXEL), pts, ref, (kind, n, "staged"))
            # byte sizes off the 16-byte vectors of the counted host copy
            tails += (ref.shape[0] * 3 * pts.itemsize) % 16 != 0 and (ref.shape[0] * 8) % 16 != 0
    assert tails >= 4
    small = extra[1]
    assert all((extra[n] > small) == (n > SEL_MAX_N) for n in SIZES), extra
    ctx.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_grid_sample_hash_edges(lib, dtype):
    """Constructed voxel coordinates hit the hash each was built for; inside a filler cloud they come out as the
    reference's samples, bit-exact, and the call repeats on 64-bit keys exactly when a hash leaves [-2^39, 2^39)."""
    ctx = lib.Context()
    rng = np.random.RandomState(21)
    filler = (rng.randn(3000, 3) * 20.0).astype(dtype)
    base = {}
    for api in (grid_sample, grid_sample_staged):
        before = launches(ctx)
        api(lib, ctx, filler, HASH_VOXEL)
        base[api] = launches(ctx) - before
    ran = 0
    for name, coords in hash_cases().items():
        if dtype == np.float32 and not float32_carries(coords):
            continue
        ran += 1
        pts_case = case_points(coords, dtype)
        assert np.array_equal(orc.voxel_coords(pts_case, HASH_VOXEL), np.repeat(np.array(coords), 3, axis=0)), name
        want = [int64_wrap(HX * x + HY * y + HZ * z) for x, y, z in coords]
        assert orc.voxel_hashes(np.array(coords, np.int64)).tolist() == want, name
        pts = np.concatenate([filler, pts_case])[rng.permutation(filler.shape[0] + pts_case.shape[0])]
        h = orc.voxel_hashes(orc.voxel_coords(pts, HASH_VOXEL))
        repeat = bool(h.min() < -COMPACT or h.max() >= COMPACT)
        assert repeat == (name not in ("compact_min", "compact_max", "collision", "collision_wrap")), name
        s_ref, i_ref = orc.grid_sample(pts, HASH_VOXEL)
        if name.startswith("collision"):
            assert len(set(want)) == 1 and (h == want[0]).sum() == 6    # six points, two voxels, one sample
        for api in (grid_sample, grid_sample_staged):
            before = launches(ctx)
            check_sample(api(lib, ctx, pts, HASH_VOXEL), pts, i_ref, (name, api.__name__))
            assert (launches(ctx) - before > base[api]) == repeat, (name, api.__name__)
    assert ran == (8 if dtype == np.float64 else 4)
    for pts, voxel in zip(*[iter(half_points(dtype))] * 2):
        c = orc.voxel_coords(pts, voxel)
        assert (c % 2 == 0).all() and (c < 0).any()          # round-half-even, on both sides of zero
        s_ref, i_ref = orc.grid_sample(pts, voxel)
        for api in (grid_sample, grid_sample_staged):
            check_sample(api(lib, ctx, pts, voxel), pts, i_ref, ("half", voxel))
        np.testing.assert_array_equal(lib_voxelise(lib, ctx, pts, voxel), c)
    ctx.close()


def lib_voxelise(lib, ctx, pts, voxel):
    coords, hashes = np.empty((pts.shape[0], 3), np.int64), np.empty(pts.shape[0], np.int64)
    ctx.call("pls_voxel_hash", lib.ptr(pts), int(pts.dtype == np.float64), pts.shape[0], float(voxel), lib.ptr(coords),
             lib.ptr(hashes))
    assert np.array_equal(hashes, orc.voxel_hashes(coords))
    return coords


# ------------------------------------------------------------------------------------------- 2. voxel statistics
def voxel_stats_ref(pts, voxel):
    """Voxelization in float64: coordinates, hashes, voxel ids / sizes (ascending hash), means and un-normalised scatter
    matrices, with per voxel sum |x| and sum (|x| + |mean|)(|x| + |mean|)^T for the error bounds."""
    coords = orc.voxel_coords(pts, voxel)
    h = orc.voxel_hashes(coords)
    _, ids, cnt = np.unique(h, return_inverse=True, return_counts=True)
    ids = ids.reshape(-1)
    x = pts.astype(np.float64)

    def vsum(w):
        return np.bincount(ids, weights=w, minlength=cnt.shape[0])

    mean = np.stack([vsum(x[:, a]) for a in range(3)], 1) / cnt[:, None]
    d, ax = x - mean[ids], np.abs(x) + np.abs(mean[ids])
    cov, mag = np.empty((cnt.shape[0], 3, 3)), np.empty((cnt.shape[0], 3, 3))
    for a in range(3):
        for b in range(a, 3):
            cov[:, a, b] = cov[:, b, a] = vsum(d[:, a] * d[:, b])
            mag[:, a, b] = mag[:, b, a] = vsum(ax[:, a] * ax[:, b])
    abs_sum = np.stack([vsum(np.abs(x[:, a])) for a in range(3)], 1)
    return dict(coords=coords, hashes=h, ids=ids, sizes=cnt, means=mean, covs=cov, abs_sum=abs_sum, mag=mag)


def check_voxel_stats(got, ref, dtype, tag):
    coords, hashes, sizes, means, covs, ids = got
    for key, g in (("coords", coords), ("hashes", hashes), ("ids", ids), ("sizes", sizes)):
        assert np.array_equal(g, ref[key]), (tag, key)
    assert means.dtype == dtype and covs.dtype == dtype, tag
    # A float64 sum of n terms is off by at most n eps sum |term| (either side: twice); the mean divides that by n.
    # The scatter matrix sums n products of differences, each factor bounded by |x| + |mean|, and moves by n dm dm^T
    # with the mean.  The outputs are then rounded once to the cloud's dtype.
    e64, e = np.finfo(np.float64).eps, np.finfo(dtype).eps
    n = ref["sizes"].astype(np.float64)
    dm = 2 * n[:, None] * e64 * ref["abs_sum"] / n[:, None]
    tol_m = e * np.abs(ref["means"]) + dm
    err_m = np.abs(means.astype(np.float64) - ref["means"])
    assert (err_m <= tol_m).all(), (tag, "means", float((err_m / tol_m).max()))
    tol_c = e * np.abs(ref["covs"]) + 4 * n[:, None, None] * e64 * ref["mag"] + n[:, None, None] * dm[:, :, None] * dm[:, None, :]
    err_c = np.abs(covs.astype(np.float64) - ref["covs"])
    assert (err_c <= tol_c).all(), (tag, "covs", float((err_c / np.maximum(tol_c, 1e-300)).max()))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_voxel_statistics_at_every_size_edge(lib, dtype):
    """Voxels of 1 to 257 points (32, just under and just over one and two warp strides) and the LiDAR cloud at every
    size, one context.

    Keep the call order: sizes largest first, and each size ending on the few-voxel cloud.  It is there so that a scan
    that fails to write the voxel count (as in a mutation that skips the total when n is a multiple of 2048) leaves a
    stale count no larger than the next call's point count, and the kernels and copies sized by that count stay within
    their buffers: such a bug then shows up as wrong values, never as an out-of-bounds access."""
    import pylidar_slam_b200 as b200
    ctx = lib.Context()
    seen = set()
    for n in SIZES[::-1]:
        for kind in ("lidar", "buckets"):
            pts = buckets(n, dtype) if kind == "buckets" else cloud("lidar", n, dtype)
            ref = voxel_stats_ref(pts, VOXEL)
            seen.update(ref["sizes"].tolist())
            check_voxel_stats(b200.voxel_statistics(pts, VOXEL, ctx=ctx), ref, dtype, (kind, n))
    assert {1, 31, 32, 33, 63, 64, 65, 257} <= seen and max(seen) > 257
    ctx.close()


# ----------------------------------------------------------------------------------------------- 3. epoch wrap
# A context's n-th selection runs with epoch (n - 1) % 1023 + 1, and every launch overwrites the status words of its own
# tiles.  A word of the earlier cycle that carries the epoch of a launch (and so reads as published to it) survives only
# if no launch in between covered that tile.  So: a multi-tile "mark" launch with epoch m, then single-tile selections
# only, until the launch with epoch m in the next cycle, a multi-tile "check" whose tiles 1 ... find the mark's words
# in front of them.  Were the words not cleared at the wrap, a check tile that polls its predecessor before it has
# published would take the mark's inclusive prefix for its own.
def wrap_schedule(first_mark, checks):
    """Kinds of a fresh context's selections 1, 2, ...: 'mark' at selection first_mark, 'check' EPOCH_CYCLE later (the
    same epoch, one cycle on), the next 'mark' right after it; 'single' (one tile) everywhere else."""
    kinds, n = {}, first_mark
    for _ in range(checks):
        kinds[n], kinds[n + EPOCH_CYCLE] = "mark", "check"
        n += EPOCH_CYCLE + 1
    last = max(kinds)
    return [kinds.get(i, "single") for i in range(1, last + 1)]


def inclusive_tile_counts(pts, voxel):
    """What a grid sample's tiles publish: the number of samples in tiles 0 ... t, per t."""
    h = np.sort(orc.voxel_hashes(orc.voxel_coords(pts, voxel)))
    heads = np.ones(h.shape[0], bool)
    heads[1:] = h[1:] != h[:-1]
    return np.cumsum(np.add.reduceat(heads, np.arange(0, h.shape[0], TILE)))


def test_selection_epoch_wraps_with_stale_status_words(lib):
    """Five wraps of one context's selection epoch with grid samples: a SEL_MAX_N-point mark before each wrap, a
    600 000-point check after it, single-tile samples in between.  The check's tiles publish other counts than the mark's
    (asserted), so a mark word taken as published changes the sample count or order.  Every result against the
    reference."""
    import torch
    import pylidar_slam_b200 as b200
    rng = np.random.RandomState(31)
    clouds = {}
    for kind, n, scale in (("single", 1500, 1.0), ("mark", SEL_MAX_N, 14.0), ("check", 600000, 10.0)):
        pts = (rng.randn(n, 3) * np.array([scale, scale, scale / 8])).astype(np.float32)
        ref = orc.grid_sample(pts, VOXEL)[1]
        clouds[kind] = (torch.from_numpy(pts).cuda(), torch.from_numpy(ref).cuda(), inclusive_tile_counts(pts, VOXEL))
    assert clouds["single"][0].shape[0] <= TILE
    mark, check = clouds["mark"][2], clouds["check"][2]
    assert (mark[:check.shape[0]] != check).all()
    schedule = wrap_schedule(100, 5)
    assert len(schedule) >= 2100 and schedule.count("check") == 5
    ctx = lib.Context()
    for i, kind in enumerate(schedule, start=1):
        pts, ref, _ = clouds[kind]
        s, idx = b200.grid_sample(pts, VOXEL, ctx=ctx)
        assert torch.equal(idx, ref) and torch.equal(s, pts[ref]), (i, kind)
    ctx.close()


def test_fused_frame_input_after_epoch_wraps_with_stale_status_words(lib):
    """The same schedule on a kd context whose checks are frames through the fused frame input (tensor layout, pixel
    queries; its only selection) and whose marks are 20-tile grid samples.  The frames' 2048-row tiles alternate between
    valid rows and NaN rows: a NaN tile is done with its rows long before the valid tile in front of it (projection,
    z-buffer read) publishes, so it polls that tile's word while the word still holds the mark's.  A twin context runs the
    frames alone; every frame gives the same bits on both."""
    from pylidar_slam_b200 import synthetic as syn
    from test_multi_sequence_gpu import Frame, make_ctx, readback, same, single
    a, b = make_ctx(lib, height=32, width=512), make_ctx(lib, height=32, width=512)
    rng = np.random.RandomState(43)
    samples = {"single": (rng.randn(1500, 3) * 10).astype(np.float32), "mark": (rng.randn(40000, 3) * 10).astype(np.float32)}
    refs = {kind: orc.grid_sample(pts, VOXEL)[1] for kind, pts in samples.items()}

    def frame(k):
        rows = syn.scan(k, 64, 512).reshape(16, TILE, 3)
        rows[1::2] = np.nan
        return Frame(lib, "tensor", np.ascontiguousarray(rows.reshape(-1, 3)))

    prev, k = [None, None], 0

    def step():                     # frame k on both contexts; frame 0 makes no selection (it only builds the map)
        nonlocal k
        f, outs = frame(k), []
        for j, ctx in enumerate((a, b)):
            st, out = single(lib, ctx, f, 0.0, prev[j])
            assert st == lib.PLS_OK and int(out["info"][5]) == 8 * TILE, (k, j)
            if out["has"]:
                prev[j] = out["pose"].reshape(4, 4).copy()
            outs.append(out)
        same(outs[0], outs[1], k)
        if k > 0:
            nq = int(outs[0]["info"][2])
            (sa, ra), (sb, rb) = readback(lib, a, nq), readback(lib, b, nq)
            assert sa == sb == lib.PLS_OK, k
            same(ra, rb, (k, "correspondences"))
        k += 1

    step()
    schedule = wrap_schedule(50, 4)
    for i, kind in enumerate(schedule, start=1):
        if kind == "check":
            step()
        else:
            assert np.array_equal(grid_sample(lib, a, samples[kind], VOXEL)[1], refs[kind]), (i, kind)
    assert k == 5
    a.close()
    b.close()


def test_epoch_wrap_in_mid_sequence(lib):
    """Two contexts run one 40-frame kd sequence (grid sample + fused frame input: two selections a frame); one of them
    first makes enough throwaway selections that its epoch wraps, and its status words are cleared, near frame 20.
    Every frame: the same bits."""
    from pylidar_slam_b200 import synthetic as syn
    from test_multi_sequence_gpu import Frame, make_ctx, readback, same, single
    a, b = make_ctx(lib, height=32, width=512), make_ctx(lib, height=32, width=512)
    throwaway = (np.random.RandomState(41).randn(5000, 3) * 10).astype(np.float32)
    ref = orc.grid_sample(throwaway, VOXEL)[1]
    for _ in range(EPOCH_CYCLE - 40):
        assert np.array_equal(grid_sample(lib, b, throwaway, VOXEL)[1], ref)
    prev = [None, None]
    for k in range(40):
        frame = Frame(lib, "tensor", syn.scan(k, 32, 512))
        outs = []
        for j, ctx in enumerate((a, b)):
            st, out = single(lib, ctx, frame, VOXEL, prev[j])
            assert st == lib.PLS_OK, (k, j)
            if out["has"]:
                prev[j] = out["pose"].reshape(4, 4).copy()
            outs.append(out)
        same(outs[0], outs[1], k)
        if k > 0:
            nq = int(outs[0]["info"][2])
            (sa, ra), (sb, rb) = readback(lib, a, nq), readback(lib, b, nq)
            assert sa == sb == lib.PLS_OK, k
            same(ra, rb, (k, "correspondences"))
    a.close()
    b.close()


# ----------------------------------------------------------------------------------- 4. kd frame input, one wave
def big_frame(k, n, nan_every=97):
    """n rows of a dense synthetic scan (128 x 8448 = SEL_MAX_N rows, plus rows of a second scan), every nan_every-th
    row NaN in one or all coordinates."""
    from pylidar_slam_b200 import synthetic as syn
    rows = syn.scan(k, 128, 8448)
    if n > rows.shape[0]:
        rows = np.concatenate([rows, syn.scan(k, 8, 1024)[:n - rows.shape[0]]])
    rows = np.ascontiguousarray(rows[:n])
    bad = np.arange(3, n, nan_every)
    rows[bad[::2]] = np.nan
    rows[bad[1::2], 1] = np.nan
    return rows, bad.shape[0]


@pytest.mark.parametrize("n", [SEL_MAX_N - 1, SEL_MAX_N + 1])
def test_kd_point_frames_float32_vs_float64(lib, n):
    """Point layout, kd map: float32 rows (the fused selection up to SEL_MAX_N, pack_valid_rows above) against the same
    rows as float64 values (pack_valid_rows_f64).  Frame 0 is the same float32 frame for both; every later frame gives
    the same bits: pose, params, info, matches, normals, search states, accumulators, and at the end the map."""
    from test_multi_sequence_gpu import Frame, make_ctx, map_points, readback, same, single
    a, b = make_ctx(lib, max_num_alignments=4), make_ctx(lib, max_num_alignments=4)
    prev = [None, None]
    for k in range(4):
        rows, nan_rows = big_frame(k, n)
        frames = (Frame(lib, "ndarray", rows),) * 2 if k == 0 else (Frame(lib, "ndarray", rows), Frame(lib, "f64", rows))
        outs = []
        for j, ctx in enumerate((a, b)):
            st, out = single(lib, ctx, frames[j], 0.0, prev[j])
            assert st == lib.PLS_OK, (k, j)
            assert int(out["info"][5]) == nan_rows, (k, j)         # rows dropped by the selection / the scan
            if out["has"]:
                prev[j] = out["pose"].reshape(4, 4).copy()
            outs.append(out)
        same(outs[0], outs[1], k)
        if k > 0:
            nq = int(outs[0]["info"][2])
            assert nq == n - nan_rows
            (sa, ra), (sb, rb) = readback(lib, a, nq), readback(lib, b, nq)
            assert sa == sb == lib.PLS_OK, k
            same(ra, rb, (k, "correspondences"))
    assert map_points(a).tobytes() == map_points(b).tobytes()
    a.close()
    b.close()


def test_kd_pixel_queries_above_one_wave(lib):
    """Tensor layout, float32, a frame of more than SEL_MAX_N points: the queries are the non-empty pixels of the
    frame's z-buffer (projection + pack_valid_pixels), as many as the oracle's; one ICP iteration from the identity,
    checked per query against the float64 reference like every kd ICP iteration."""
    import torch
    from scipy.spatial import cKDTree
    from oracle import kd_icp_reference as ref
    from test_kd_icp_iterations_gpu import K_NORMALS, _check_iteration, _check_pose_update
    from test_multi_sequence_gpu import Frame, make_ctx, map_points, readback, single
    from pylidar_slam_b200 import synthetic as syn
    H, W = 64, 2048
    ctx = make_ctx(lib, height=H, width=W, max_num_alignments=1, num_neighbors_normals=K_NORMALS)
    st, _ = single(lib, ctx, Frame(lib, "tensor", syn.scan(0, H, W)), 0.0, None)
    assert st == lib.PLS_OK
    m = np.ascontiguousarray(map_points(ctx))
    rows = syn.scan(1, 120, 9100)        # beams and columns never exactly on a pixel's half (128 beams would be)
    assert rows.shape[0] > SEL_MAX_N
    eye = np.eye(4, dtype=np.float32)
    st, out = single(lib, ctx, Frame(lib, "tensor", rows), 0.0, eye)
    assert st == lib.PLS_OK and out["has"] and int(out["info"][0]) == 1
    vmap = orc.Projector(H, W).build_projection_map(torch.from_numpy(rows)[None])[0]
    pix = orc.map_to_points(vmap[None])[0].numpy()
    filled = np.nonzero(np.linalg.norm(pix, axis=1) > 0)[0]            # the oracle's non-empty pixels, in pixel order
    pix = pix[filled]
    nq = int(out["info"][2])
    assert nq == pix.shape[0]
    st, run = readback(lib, ctx, nq)
    assert st == lib.PLS_OK
    q = np.ascontiguousarray(run["state"][:, :3])                       # at the identity: the queries themselves
    # Query i is the winner of the i-th non-empty pixel.  It may differ from the oracle's winner only as the a3 projection
    # test allows (test_a3_projection_full_size_vs_oracle): some point of the frame lies within 2e-3 px of a rounding
    # boundary next to that pixel (atan2 / asin differ by an ulp or two between CUDA and the host), or the two winners
    # are range ties to the last bits of a float32 sqrt.
    differ = ~(q == pix).all(1)
    row, col = orc.Projector(H, W).pixels(torch.from_numpy(rows)[None])
    rc = np.stack([row[0].numpy(), col[0].numpy()], axis=1).astype(np.float64)
    near = rc[(np.abs(rc - np.floor(rc) - 0.5) < 2e-3).any(axis=1) & np.isfinite(rc).all(axis=1)]
    touched = np.zeros(H * W, bool)
    for r in (np.floor(near[:, 0]), np.ceil(near[:, 0])):
        for c in (np.floor(near[:, 1]), np.ceil(near[:, 1])):
            ok = (r >= 0) & (r < H) & (c >= 0) & (c < W)
            touched[(r[ok] * W + c[ok]).astype(np.int64)] = True
    r_q, r_pix = np.linalg.norm(q.astype(np.float64), axis=1), np.linalg.norm(pix.astype(np.float64), axis=1)
    unexplained = differ & ~touched[filled] & (np.abs(r_q - r_pix) > 2e-6 * r_pix)
    assert not unexplained.any(), (int(differ.sum()), int(unexplained.sum()))
    run.update(T=out["pose"].reshape(4, 4), params=out["params"], losses=np.array([out["info"][1]], np.float32))
    _check_iteration(ref, m, cKDTree(m.astype(np.float64)), q, eye, run, "geman_mcclure", 0.3, tag="above one wave")
    _check_pose_update(ref, eye, run, 1)
    ctx.close()
