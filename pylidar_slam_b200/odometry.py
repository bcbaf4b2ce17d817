"""Mirrors of the reference's odometry plug-in interfaces for the ICP hot path:

  OdometryAlgorithm / OdometryConfig              slam/odometry/odometry.py:13-81
  LocalMap, KdTreeLocalMap, ProjectiveLocalMap    slam/odometry/local_map.py:21-445
  RigidAlignment, GaussNewtonPointToPlaneAlignment slam/odometry/alignment.py:23-127
  ICPFrameToModel, ICPFrameToModelConfig           slam/odometry/icp_odometry.py:27-380

Same class / method / config-field names, same data_dict keys, same error behaviour; the
arithmetic runs in libplslam_b200.so (hand-written sm_90a CUDA) through the C ABI.  The
registries (`ODOMETRY`, `LOCAL_MAP`, `RIGID_ALIGNMENT`) keep the reference's discriminator
fields (`algorithm`, `type`, `mode`) and add `*_b200` members; INTEGRATION.md shows the two-line
patch that registers them inside the reference tree.
"""
import ctypes as C
import dataclasses
import time
from abc import ABC, abstractmethod
from dataclasses import dataclass, field
from enum import Enum
from typing import Any, Dict, Optional

import numpy as np
import torch

from . import _lib
from .common import Pose, SphericalProjector, assert_debug, check_tensor, euler_pose_matrix_f64

MISSING = "???"


def _cfg_to_dict(cfg) -> dict:
    if cfg is None:
        return {}
    if dataclasses.is_dataclass(cfg):
        return {f.name: getattr(cfg, f.name) for f in dataclasses.fields(cfg)}
    if isinstance(cfg, dict) or hasattr(cfg, "keys"):
        return {k: cfg[k] for k in cfg.keys()}
    raise AssertionError(f"cannot interpret {cfg!r} as a config")


class ObjectLoaderEnum:
    """slam/common/utils.py:266-302: discriminator-driven loading from a config."""

    @classmethod
    def load(cls, config, **kwargs):
        d = _cfg_to_dict(config)
        assert_debug(cls.type_name() in d, f"The config does not contains the key : '{cls.type_name()}'")
        _type = d[cls.type_name()]
        assert_debug(_type in cls.__members__,
                     f"Unknown type `{_type}`. Existing members are : {cls.__members__.keys()}")
        _class, _config = cls.__members__[_type].value
        if not isinstance(config, _config):
            names = {f.name for f in dataclasses.fields(_config)}
            config = _config(**{k: v for k, v in d.items() if k in names and v != MISSING})
        return _class(config, **kwargs)


# ----------------------------------------------------------------------------------------------------------------------
# Local maps
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class LocalMapConfig:
    pose: str = "euler"
    type: str = MISSING


@dataclass
class KdTreeLocalMapConfig(LocalMapConfig):
    local_map_size: int = 20
    num_neighbors_normals: int = 10
    type: str = "kdtree_local_map"


@dataclass
class ProjectiveLocalMapConfig(LocalMapConfig):
    local_map_size: int = 20
    type: str = "projective_local_map"
    normals_kernel_size: int = 5


class LocalMap(ABC):
    """slam/odometry/local_map.py:31-79"""

    @dataclass
    class NeighborhoodResult:
        neighbor_points: Optional[Any] = None
        neighbor_normals: Optional[Any] = None
        new_target_points: Optional[Any] = None

    def __init__(self, config: LocalMapConfig, **kwargs):
        self.config = config
        self.pose = Pose(config.pose)

    @abstractmethod
    def init(self):
        raise NotImplementedError("")

    @abstractmethod
    def update(self, new_relative_pose, new_pc_data=None, new_vertex_map=None, **kwargs) -> None:
        raise NotImplementedError("")

    @abstractmethod
    def nearest_neighbor_search(self, points, with_normals: bool = True, with_new_target_points: bool = True, **kwargs):
        raise NotImplementedError("")


def _pose16(relative_pose) -> np.ndarray:
    if isinstance(relative_pose, torch.Tensor):
        relative_pose = relative_pose.detach().cpu().numpy()
    rel = np.ascontiguousarray(np.asarray(relative_pose, dtype=np.float32).reshape(4, 4))
    return rel


def _f32c(x):
    if isinstance(x, np.ndarray):
        return np.ascontiguousarray(x, dtype=np.float32)
    return x.to(torch.float32).contiguous()


def _new(x, shape, dtype=torch.float32):
    if isinstance(x, np.ndarray):
        return np.empty(shape, dtype={torch.float32: np.float32, torch.int64: np.int64}[dtype])
    return torch.empty(shape, dtype=dtype, device=x.device)


# The reference's set_map_pointcloud(pointcloud, normals) stores the [N,3] normals where its search reads a fourth column
# (local_map.py:297-299, 399): every search with normals then raises IndexError, until the next update or init rebuilds
# the normal cache.  The flag lives on the context, which the map shares with the odometry that registers on it.
_NORMALS_INDEX_ERROR = "index 3 is out of bounds for axis 1 with size 3"


def _set_given_normals(ctx, given: bool):
    ctx.kd_given_normals = given


def _check_given_normals(ctx):
    if getattr(ctx, "kd_given_normals", False):
        raise IndexError(_NORMALS_INDEX_ERROR)


def _gated(ctx, max_distance) -> bool:
    """Whether max_distance asks for a gated registration; refuses a NaN or negative gate, and a finite one on a
    projective map, before any call."""
    d = float(max_distance)
    assert_debug(d >= 0.0, "max_distance must be >= 0 (not NaN)")
    if np.isinf(d):
        return False
    assert_debug(ctx.cfg.local_map_type == _lib.MAP_KDTREE, "a finite max_distance needs a kd-tree local map")
    return True


def _thresholded(ctx, min_eigenvalue) -> bool:
    """Whether min_eigenvalue asks for the eigenvalue-thresholded solve; refuses a NaN, negative or infinite threshold,
    and a positive one on a projective map, before any call."""
    e = float(min_eigenvalue)
    assert_debug(e >= 0.0 and np.isfinite(e), "min_eigenvalue must be finite and >= 0 (not NaN)")
    if e == 0.0:
        return False
    assert_debug(ctx.cfg.local_map_type == _lib.MAP_KDTREE, "a min_eigenvalue > 0 needs a kd-tree local map")
    return True


# Pose count A*(2*half_x+1)*(2*half_y+1) from which _pose_search takes pls_kdmap_pose_search_pyramid (branch and
# bound) instead of scoring every pose with pls_kdmap_pose_search.  Measured on an H100 SXM at 700 W, K = 8, 72 yaws
# (profiles/h100_pose_search_pyramid.json, DESIGN section 18): up to 30 M poses the exhaustive call is faster in all
# but one measured case; at 46 M poses (+-200 m at 0.5 m) the pyramid is 1.6-3.7x faster on 4 of 6 map/scan pairs and
# 4-5 % slower on 2; at 288 M and 1.15 G poses (+-1000 m on the 2 km map) it is 1.5-11.7x faster.
POSE_SEARCH_PYRAMID_MIN_POSES = 1 << 27


def _bases_f64(poses) -> np.ndarray:
    """Pose-search bases [A,4,4] (numpy or torch, host or CUDA) as a contiguous float64 host array."""
    if isinstance(poses, torch.Tensor):
        poses = poses.detach().cpu().numpy()
    check_tensor(poses, [-1, 4, 4])
    return np.ascontiguousarray(poses, dtype=np.float64)


def _pose_search(ctx, scan, poses, cell_size, half_x, half_y, num_candidates, out_scores=None):
    """The correlative pose search on ctx's kd map: scan [n,3] (numpy or torch, host or CUDA), poses [A,4,4] (float64).
    Returns (T [k,4,4] float64, scores [k] int32, index [k] int64).  Both calls return the same candidates bit for bit;
    pls_kdmap_pose_search scores every pose and is taken for out_scores, K = 0 and fewer than
    POSE_SEARCH_PYRAMID_MIN_POSES poses, pls_kdmap_pose_search_pyramid prunes and is taken otherwise, with the
    exhaustive call answering any volume below 2^31 poses that the pyramid refuses."""
    check_tensor(scan, [-1, 3])
    pts = _f32c(scan)
    bases = _bases_f64(poses)
    K = int(num_candidates)
    T, score = np.zeros((K, 4, 4), np.float64), np.zeros(K, np.int32)
    index, num = np.zeros(K, np.int64), C.c_int(0)
    args = (_lib.ptr(pts), pts.shape[0], _lib.ptr(bases), bases.shape[0], float(cell_size), int(half_x), int(half_y), K)
    outs = (_lib.ptr(T), _lib.ptr(score), _lib.ptr(index), C.byref(num))
    poses_in_volume = bases.shape[0] * (2 * int(half_x) + 1) * (2 * int(half_y) + 1)
    if out_scores is not None or K < 1 or poses_in_volume < POSE_SEARCH_PYRAMID_MIN_POSES:
        ctx.call("pls_kdmap_pose_search", *args, _lib.ptr(out_scores), *outs)
    else:
        try:
            ctx.call("pls_kdmap_pose_search_pyramid", *args, *outs)
        except AssertionError:
            # The pyramid refuses when more nodes survive a level than its work lists hold (maps where most poses
            # score alike) or when its per-(base, row) cells outgrow their limit.  Below 2^31 poses the exhaustive call
            # still answers, so the volume gets the answer it always had; beyond that the refusal stands.
            if poses_in_volume >= 1 << 31:
                raise
            ctx.call("pls_kdmap_pose_search", *args, None, *outs)
    k = num.value
    return T[:k], score[:k], index[:k]


# pls_kdmap_pose_search_scans refuses batches whose volumes together hold 2^31 poses or more
_POSE_SEARCH_SCANS_MAX_POSES = 1 << 31
_SHARED_GRID_REFUSAL = "shared occupancy box"


def _pose_search_scans(ctx, scans, bases_list, cell_size, halves, num_candidates, out_scores=None):
    """_pose_search for S scans: scans [n_s,3] (numpy or torch, host or CUDA), bases_list S arrays [A_s,4,4], halves S
    pairs (half_x, half_y).  Returns S tuples (T, scores, index), tuple s what _pose_search gives scan s; out_scores
    [sum V_s] int32 (nullable) receives every volume, scan-major.  With K >= 1 and no out_scores, a scan of at least
    POSE_SEARCH_PYRAMID_MIN_POSES poses goes to _pose_search (the pyramid, with its fallback); the others go to
    pls_kdmap_pose_search_scans in consecutive chunks of fewer than 2^31 poses.  A chunk whose shared occupancy grid is
    refused -- scans that lie far apart on a large map -- is sorted by its first base's x, halved and retried; a chunk
    of one scan goes to _pose_search."""
    S, K = len(scans), int(num_candidates)
    assert_debug(len(bases_list) == S and len(halves) == S, "one base set and one window per scan")
    pts, bases, vols = [], [], []
    for s in range(S):
        check_tensor(scans[s], [-1, 3])
        pts.append(_f32c(scans[s]))
        bases.append(_bases_f64(bases_list[s]))
        hx, hy = (int(h) for h in halves[s])
        vols.append(bases[s].shape[0] * (2 * hx + 1) * (2 * hy + 1))
    first = np.concatenate([[0], np.cumsum(vols, dtype=np.int64)])
    results = [None] * S

    def single(s):
        hx, hy = halves[s]
        view = None if out_scores is None else out_scores[first[s]:first[s + 1]]
        results[s] = _pose_search(ctx, pts[s], bases[s], cell_size, hx, hy, K, out_scores=view)

    def batched(idx):
        if len(idx) == 1:
            return single(idx[0])
        S_c, Kc = len(idx), max(K, 1)
        addresses = np.array([_lib.ptr(pts[s]) for s in idx], dtype=np.uint64)
        rows = np.array([pts[s].shape[0] for s in idx], dtype=np.int64)
        cat = np.ascontiguousarray(np.concatenate([bases[s] for s in idx]))
        num_bases = np.array([bases[s].shape[0] for s in idx], dtype=np.int32)
        hx = np.array([int(halves[s][0]) for s in idx], dtype=np.int32)
        hy = np.array([int(halves[s][1]) for s in idx], dtype=np.int32)
        vol = None if out_scores is None else np.empty(sum(vols[s] for s in idx), np.int32)
        T, score = np.zeros((S_c, Kc, 4, 4), np.float64), np.zeros((S_c, Kc), np.int32)
        index, num = np.zeros((S_c, Kc), np.int64), np.zeros(S_c, np.int32)
        try:
            ctx.call("pls_kdmap_pose_search_scans", _lib.ptr(addresses), _lib.ptr(rows), S_c, _lib.ptr(cat),
                     _lib.ptr(num_bases), float(cell_size), _lib.ptr(hx), _lib.ptr(hy), K, _lib.ptr(vol), _lib.ptr(T),
                     _lib.ptr(score), _lib.ptr(index), _lib.ptr(num))
        except AssertionError as e:
            if _SHARED_GRID_REFUSAL not in str(e):
                raise
            by_x = sorted(idx, key=lambda s: bases[s][0, 0, 3])
            batched(by_x[:S_c // 2])
            batched(by_x[S_c // 2:])
            return
        at = 0
        for c, s in enumerate(idx):
            k = int(num[c])
            results[s] = (T[c, :k], score[c, :k], index[c, :k])
            if vol is not None:
                out_scores[first[s]:first[s + 1]] = vol[at:at + vols[s]]
                at += vols[s]

    chunk, poses = [], 0
    for s in range(S):
        if out_scores is None and K >= 1 and vols[s] >= POSE_SEARCH_PYRAMID_MIN_POSES:
            single(s)
            continue
        if chunk and poses + vols[s] >= _POSE_SEARCH_SCANS_MAX_POSES:
            batched(chunk)
            chunk, poses = [], 0
        chunk.append(s)
        poses += vols[s]
    if chunk:
        batched(chunk)
    return results


def _per_scan_halves(half_extents, S):
    """One (half_x, half_y) pair for each of S scans, from one shared pair or S pairs."""
    h = np.asarray(half_extents, dtype=np.int64)
    if h.shape == (2,):
        return [(int(h[0]), int(h[1]))] * S
    assert_debug(h.shape == (S, 2), "half_extents must be one (half_x, half_y) pair or one pair per scan")
    return [(int(x), int(y)) for x, y in h]


def _score_poses(ctx, scan, poses, cell_size) -> np.ndarray:
    """The [A] int32 scores of exactly these poses: pls_kdmap_pose_search with a 1x1 window and no candidates."""
    bases = _bases_f64(poses)
    scores = np.zeros(bases.shape[0], np.int32)
    _pose_search(ctx, scan, bases, cell_size, 0, 0, 0, out_scores=scores)
    return scores


def yaw_sweep(prior_pose, yaw_range: float = np.pi, yaw_step: float = np.deg2rad(5)) -> np.ndarray:
    """The base poses of ICPFrameToModel.localize [A,4,4] float64: the prior turned by theta_a about the map's z axis
    through the prior's own position (its roll, pitch, z and xy stay).  yaw_range >= pi: the full circle,
    theta_a = 2 pi a / A with A = ceil(2 pi / yaw_step); otherwise theta_a = (a - m) yaw_step, a = 0..2m,
    m = floor(yaw_range / yaw_step)."""
    if isinstance(prior_pose, torch.Tensor):
        prior_pose = prior_pose.detach().cpu().numpy()
    prior = np.asarray(prior_pose, dtype=np.float64).reshape(4, 4)
    assert_debug(yaw_step > 0 and np.isfinite(yaw_step), "yaw_step must be finite and > 0")
    assert_debug(yaw_range >= 0, "yaw_range must be >= 0")
    if yaw_range >= np.pi:
        A = int(np.ceil(2 * np.pi / yaw_step))
        theta = 2 * np.pi * np.arange(A) / A
    else:
        m = int(np.floor(yaw_range / yaw_step))
        theta = (np.arange(2 * m + 1) - m) * yaw_step
    c, s = np.cos(theta), np.sin(theta)
    Rz = np.zeros((theta.shape[0], 3, 3))
    Rz[:, 0, 0], Rz[:, 0, 1], Rz[:, 1, 0], Rz[:, 1, 1], Rz[:, 2, 2] = c, -s, s, c, 1.0
    bases = np.tile(prior, (theta.shape[0], 1, 1))
    bases[:, :3, :3] = Rz @ prior[:3, :3]
    return bases


@dataclass
class PoseCandidate:
    """One result of ICPFrameToModel.localize: the refined pose and its score, the search's pose and score it started
    from, its rank in the search, and the refinement's iterations and status (PLS_OK, PLS_W_TINY_RESIDUAL or
    PLS_E_SINGULAR)."""
    T: np.ndarray
    score: int
    T0: np.ndarray
    coarse_score: int
    coarse_rank: int
    iterations: int
    status: int


def _pose_candidates(T0, coarse, T, iters, status, scores) -> list:
    """localize's result for one scan from its search candidates (T0 [k,4,4], coarse [k]) and their refinements (T,
    iters, status, refined scores [k]): every candidate as a PoseCandidate, ordered by status (singular last), then
    refined score (descending), then search rank."""
    singular = status == _lib.PLS_E_SINGULAR
    order = np.lexsort((np.arange(T.shape[0]), -scores.astype(np.int64), singular))
    return [PoseCandidate(T=T[r].astype(np.float64), score=int(scores[r]), T0=T0[r], coarse_score=int(coarse[r]),
                          coarse_rank=int(r), iterations=int(iters[r]), status=int(status[r])) for r in order]


_UPPER6 = [(a, b) for a in range(6) for b in range(a, 6)]


@dataclass
class RegistrationQuality:
    """How well one pose registers its scan on the kd map (ICPFrameToModel.evaluate_registrations): what a filter, a
    pose graph or an acceptance test needs of a registration.

    valid: the scan's valid rows (no NaN coordinate); inliers: those whose exact nearest map point lies within
    max_distance of the transformed row; fitness = inliers / valid; rmse = sqrt(sum d^2 / inliers), d the distance to
    that nearest point; plane_rmse = sqrt(sum r^2 / inliers), r the point-to-plane residual.  NaN where a denominator
    is zero.

    information [6,6]: J^T W J over the inliers, J = [n, p' x n] the point-to-plane Jacobian of the first ICP iteration
    and W its robust weights (the context's scheme).  The parameters are (tx, ty, tz, rx, ry, rz) of a small increment
    left-multiplied onto the pose, in the map frame.  eigenvalues [6] (ascending) and eigenvectors [6,6] (columns) are
    np.linalg.eigh(information): a small eigenvalue marks a direction the map does not constrain (a tunnel, a
    corridor, a flat field).  covariance [6,6] = (sum (w r)^2 / (inliers - 6)) information^-1, the least-squares
    formula: exact for the unweighted scheme, an approximation under robust weights.  None when inliers <= 6 or when the
    float64 Cholesky factorisation of information fails."""
    valid: int
    inliers: int
    fitness: float
    rmse: float
    plane_rmse: float
    information: np.ndarray
    covariance: Optional[np.ndarray]
    eigenvalues: np.ndarray
    eigenvectors: np.ndarray

    @staticmethod
    def from_stats(row) -> "RegistrationQuality":
        """From one row of pls_kdmap_evaluate_poses (PLS_EVAL_STATS doubles: 21 J^T W J upper, 6 J^T W r,
        sum (w r)^2, sum r^2, inliers, sum d^2, valid rows)."""
        row = np.asarray(row, np.float64)
        H = np.zeros((6, 6))
        for k, (a, b) in enumerate(_UPPER6):
            H[a, b] = H[b, a] = row[k]
        inliers, valid = int(row[29]), int(row[31])

        def ratio(num, den):
            return float(num / den) if den > 0 else float("nan")

        covariance = None
        if inliers > 6:
            try:
                L = np.linalg.cholesky(H)
                L_inv = np.linalg.inv(L)
                covariance = (row[27] / (inliers - 6)) * (L_inv.T @ L_inv)
            except np.linalg.LinAlgError:
                covariance = None
        w, v = np.linalg.eigh(H)
        return RegistrationQuality(valid=valid, inliers=inliers, fitness=ratio(inliers, valid),
                                   rmse=float(np.sqrt(ratio(row[30], inliers))),
                                   plane_rmse=float(np.sqrt(ratio(row[28], inliers))), information=H,
                                   covariance=covariance, eigenvalues=w, eigenvectors=v)


class KdTreeLocalMap(LocalMap):
    """KdTreeLocalMap (local_map.py:254-427) on the GPU: exact 1-NN over the hashed cell pyramid + lazily cached 10-NN normals.

    Pass `ctx=odometry.ctx` to work on the map an ICPFrameToModel registers against, e.g. to load a prior map with
    set_map_pointcloud and localise scans in it with register_new_frame_hypotheses."""

    def __init__(self, config: KdTreeLocalMapConfig, projector=None, ctx: Optional[_lib.Context] = None, **kwargs):
        super().__init__(config)
        self.ctx = ctx or _lib.Context(local_map_type=_lib.MAP_KDTREE, local_map_size=config.local_map_size,
                                       num_neighbors_normals=config.num_neighbors_normals)

    def init(self):
        self.ctx.call("pls_map_init")
        _set_given_normals(self.ctx, False)

    def set_map_pointcloud(self, pointcloud: np.ndarray, normals: Optional[np.ndarray] = None):
        """KdTreeLocalMap.set_map_pointcloud (local_map.py:289-299): the map becomes `pointcloud` [N,3] (float32, or
        float64 rounded to float32), held as no frame.  Later updates move it and append frames; once more than
        local_map_size frames are held, each eviction drops the oldest frame's row count from the front of the map --
        prior-map rows first, as the reference does.  One divergence: a row with a NaN or an infinite coordinate raises
        AssertionError and leaves the map unchanged (the reference stores it, and its search cannot handle it).
        `normals` [N,3] is checked and, as in the reference, makes every search with normals raise IndexError until
        the next update."""
        check_tensor(pointcloud, [-1, 3])
        if not isinstance(pointcloud, np.ndarray):  # the reference's check_tensor(.., np.ndarray): typeguard 2's TypeError
            raise TypeError(f"{type(pointcloud).__module__}.{type(pointcloud).__name__} is not an instance of numpy.ndarray")
        is64 = pointcloud.dtype == np.float64
        pc = np.ascontiguousarray(pointcloud, dtype=np.float64 if is64 else np.float32)
        self.ctx.call("pls_kdmap_set_points", _lib.ptr(pc), int(is64), pc.shape[0])
        _set_given_normals(self.ctx, False)
        if normals is not None:
            check_tensor(normals, [*pointcloud.shape])
            if not isinstance(normals, np.ndarray):
                raise TypeError(f"{type(normals).__module__}.{type(normals).__name__} is not an instance of numpy.ndarray")
            _set_given_normals(self.ctx, True)

    def search_poses(self, scan, base_poses, cell_size: float, half_extent=(0, 0), num_candidates: int = 8):
        """Correlative pose search (pls_kdmap_pose_search; no reference counterpart): scores every pose base_poses[a]
        moved by whole cells (i, j) along the map's x and y, |i| <= half_extent[0], |j| <= half_extent[1], by how many
        valid scan points land in map cells of size cell_size, and returns the best local maxima in the (a, i, j)
        volume, best first: (T [k,4,4] float64, scores [k] int32, index [k] int64 into the volume).  scan [n,3] is
        numpy or torch, host or CUDA; base_poses [A,4,4].  The map is left unchanged.  Large volumes are searched by
        branch and bound (pls_kdmap_pose_search_pyramid) with the same result, so half_extent may span the whole map."""
        hx, hy = half_extent
        return _pose_search(self.ctx, scan, base_poses, cell_size, hx, hy, num_candidates)

    def search_poses_scans(self, scans, base_poses, cell_size: float, half_extents=(0, 0), num_candidates: int = 8):
        """search_poses for S scans in one call (pls_kdmap_pose_search_scans; no reference counterpart): a localisation
        server re-localising many vehicles' scans, offline map matching a recorded drive's scans.  scans: S [n_s,3]
        arrays or tensors; base_poses: S arrays [A_s,4,4]; half_extents: one pair for every scan or one pair per scan.
        Returns S tuples (T, scores, index); tuple s is what search_poses(scans[s], base_poses[s], cell_size,
        half_extents[s], num_candidates) returns.  The map is left unchanged."""
        S = len(scans)
        assert_debug(len(base_poses) == S, "base_poses must hold one [A,4,4] array per scan")
        return _pose_search_scans(self.ctx, scans, base_poses, cell_size, _per_scan_halves(half_extents, S),
                                  num_candidates)

    def score_poses(self, scan, poses, cell_size: float) -> np.ndarray:
        """The [A] int32 scores of exactly these poses [A,4,4] (search_poses' score, without shifts)."""
        return _score_poses(self.ctx, scan, poses, cell_size)

    def frame_counts(self) -> list:
        """The point counts of the frames the map holds, oldest first (rows before them are a set cloud)."""
        counts = np.zeros(max(int(self.ctx.cfg.local_map_size), 1) + 1, dtype=np.int64)
        num = C.c_int(0)
        self.ctx.call("pls_kdmap_frames", _lib.ptr(counts), C.byref(num))
        return [int(c) for c in counts[:num.value]]

    def get_last_frame(self) -> torch.Tensor:
        """KdTreeLocalMap.get_last_frame (local_map.py:425-427): the rows of the last inserted frame, as a float32 CPU
        tensor.  IndexError while no frame is held (after set_map_pointcloud or init); a last frame of zero rows gives
        the whole map, as the reference's `[-0:]` slice does."""
        counts = self.frame_counts()
        if not counts:
            raise IndexError("list index out of range")
        return torch.from_numpy(self.points()[-counts[-1]:])

    def update(self, relative_pose, new_pc_data=None, new_vertex_map=None, **kwargs):
        _set_given_normals(self.ctx, False)
        rel = _pose16(relative_pose)
        if new_pc_data is not None:
            pts = _f32c(new_pc_data.reshape(-1, 3))
            self.ctx.call("pls_kdmap_update_points", _lib.ptr(rel), _lib.ptr(pts), pts.shape[0])
        elif new_vertex_map is not None:
            check_tensor(new_vertex_map, [1, 3, -1, -1])
            vm = _f32c(new_vertex_map)
            self.ctx.call("pls_kdmap_update_vertex_map", _lib.ptr(rel), _lib.ptr(vm), vm.shape[2], vm.shape[3])
        else:
            self.ctx.call("pls_kdmap_update_points", _lib.ptr(rel), None, 0)

    def num_points(self) -> int:
        n = C.c_int64(0)
        self.ctx.call("pls_kdmap_size", C.byref(n))
        return n.value

    def points(self) -> np.ndarray:
        out = np.empty((self.num_points(), 3), dtype=np.float32)
        self.ctx.call("pls_kdmap_points", _lib.ptr(out))
        return out

    def nearest_neighbor_search(self, target_points, with_normals: bool = True, with_new_target_points: bool = True,
                                **kwargs):
        check_tensor(target_points, [-1, 3])
        if with_normals:
            _check_given_normals(self.ctx)
        q = _f32c(target_points)
        n = q.shape[0]
        nb = _new(q, (n, 3))
        nrm = _new(q, (n, 3)) if with_normals else None
        self.ctx.call("pls_kdmap_nn_search", _lib.ptr(q), n, _lib.ptr(nb), _lib.ptr(nrm), None)
        result = self.NeighborhoodResult()
        is_torch = isinstance(q, torch.Tensor)
        result.neighbor_points = nb.unsqueeze(0) if is_torch else nb
        if with_normals:
            result.neighbor_normals = nrm.unsqueeze(0) if is_torch else nrm
        if with_new_target_points:
            result.new_target_points = q.reshape(1, n, 3) if is_torch else q
        return result


class ProjectiveLocalMap(LocalMap):
    """ProjectiveLocalMap (local_map.py:91-240) on the GPU."""

    def __init__(self, config: ProjectiveLocalMapConfig, projector: SphericalProjector = None,
                 ctx: Optional[_lib.Context] = None, **kwargs):
        super().__init__(config)
        assert_debug(projector is not None)
        self.projector = projector
        self.ctx = ctx or _lib.Context(local_map_type=_lib.MAP_PROJECTIVE, local_map_size=config.local_map_size,
                                       normals_kernel_size=config.normals_kernel_size, height=projector.height,
                                       width=projector.width, up_fov_deg=projector.up_fov,
                                       down_fov_deg=projector.down_fov)

    def init(self):
        self.ctx.call("pls_map_init")

    def update(self, relative_pose, new_vertex_map=None, new_normal_map=None, mask=None, **kwargs):
        rel = _pose16(relative_pose)
        vm = None
        if new_vertex_map is not None:
            check_tensor(new_vertex_map, [1, 3, self.projector.height, self.projector.width])
            vm = _f32c(new_vertex_map)
        self.ctx.call("pls_projmap_update", _lib.ptr(rel), _lib.ptr(vm))

    def model(self):
        """(_model_vmap, _model_nmap), each [K,3,H,W] numpy."""
        k = C.c_int(0)
        self.ctx.call("pls_projmap_num_frames", C.byref(k))
        H, W = self.projector.height, self.projector.width
        v = np.empty((k.value, 3, H, W), dtype=np.float32)
        n = np.empty((k.value, 3, H, W), dtype=np.float32)
        self.ctx.call("pls_projmap_model", _lib.ptr(v), _lib.ptr(n))
        return v, n

    def get_last_frame(self) -> torch.Tensor:
        """ProjectiveLocalMap.get_last_frame (local_map.py:238-240): projection_map_to_points of the newest vertex map,
        [H*W,3] float32 on the CPU.  TypeError on a map that holds no frame (the reference indexes None)."""
        k = C.c_int(0)
        self.ctx.call("pls_projmap_num_frames", C.byref(k))
        if k.value == 0:
            raise TypeError("'NoneType' object is not subscriptable")
        v = np.empty((3, self.projector.height, self.projector.width), dtype=np.float32)
        self.ctx.call("pls_projmap_last_frame", _lib.ptr(v))
        return torch.from_numpy(v).permute(1, 2, 0).reshape(-1, 3)

    def nearest_neighbor_search(self, target_points, with_normals: bool = True, with_new_target_points: bool = True,
                                **kwargs):
        check_tensor(target_points, [-1, 3])
        q = _f32c(target_points)
        hw = self.projector.height * self.projector.width
        nb, nrm, tgt = _new(q, (hw, 3)), _new(q, (hw, 3)), _new(q, (hw, 3))
        count = C.c_int64(0)
        self.ctx.call("pls_projmap_nn_search", _lib.ptr(q), q.shape[0], _lib.ptr(nb), _lib.ptr(nrm), _lib.ptr(tgt),
                      C.byref(count))
        nc = count.value
        res = self.NeighborhoodResult()
        wrap = (lambda a: a[:nc].unsqueeze(0)) if isinstance(q, torch.Tensor) else (lambda a: a[:nc][None])
        res.neighbor_points = wrap(nb)
        if with_normals:
            res.neighbor_normals = wrap(nrm)
        if with_new_target_points:
            res.new_target_points = wrap(tgt)
        return res


class LOCAL_MAP(ObjectLoaderEnum, Enum):
    """slam/odometry/local_map.py:437-445 (+ explicit *_b200 aliases)"""
    projective_local_map = (ProjectiveLocalMap, ProjectiveLocalMapConfig)
    kdtree_local_map = (KdTreeLocalMap, KdTreeLocalMapConfig)

    @classmethod
    def type_name(cls):
        return "type"


# ----------------------------------------------------------------------------------------------------------------------
# Rigid alignment
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class RigidAlignmentConfig:
    mode: str = MISSING
    pose: str = "euler"
    scheme: str = "huber"


@dataclass
class GaussNewtonPointToPlaneConfig(RigidAlignmentConfig):
    mode: str = "point_to_plane_gauss_newton"
    num_gn_iters: int = 1
    gauss_newton_config: Dict[str, Any] = field(default_factory=lambda: dict(max_iters=1))


def _reject_mask(mask, b, n):
    """`mask` of RigidAlignment.align ([b,n,1], alignment.py:96-121,158-182).  The reference cannot apply one: its cost
    functions multiply the [b,n,6] Jacobian IN PLACE by `mask.unsqueeze(1)` ([b,1,n,1]; optimization.py:391-392,500-501),
    which fails to broadcast -- every call with a mask ends in a RuntimeError.  Same error type here, after the
    reference's own shape check."""
    check_tensor(mask, [b, n, 1])
    raise RuntimeError(f"output with shape [{b}, {n}, 6] doesn't match the broadcast shape [{b}, {b}, {n}, 6] "
                       f"(the reference's alignments cannot apply a mask: optimization.py:391-392, 500-501)")


def _initial_params(pose, x0, b, is64, conv):
    """initial_estimate as [b,6] parameters: given as parameters, or as [b,4,4] float32 pose matrices (alignment.py:110-118)."""
    x0 = conv(x0)
    if x0.ndim == 3:
        check_tensor(x0, [b, 4, 4])
        assert_debug(not is64, "pose-matrix initial estimates are float32")
        x0 = pose.from_pose_matrix(x0)
    assert_debug((x0.size if isinstance(x0, np.ndarray) else x0.numel()) == 6 * b,
                 f"initial_estimate must be [{b},6] parameters or [{b},4,4] pose matrices")
    return conv(x0.reshape(b, 6))


def _gn_settings(gn_cfg) -> dict:
    """GaussNewton(**gauss_newton_config) defaults (optimization.py:287-294, :61-208)."""
    d = dict(_cfg_to_dict(gn_cfg))
    scheme = d.get("scheme", "default")
    assert_debug(scheme in _lib.SCHEMES, f"unknown weighting scheme {scheme}")
    return dict(scheme=scheme, sigma=float(d.get("sigma", 0.5)), max_iters=max(int(d.get("max_iters", 10)), 1),
                norm_stop=float(d.get("norm_stop_criterion", 1e-3)))


class RigidAlignment(ABC):
    def __init__(self, alignment_config: RigidAlignmentConfig, **kwargs):
        self.config = alignment_config
        self.pose = Pose(self.config.pose)

    def align(self, ref_points, tgt_points, *args, **kwargs):
        raise NotImplementedError("")


class GaussNewtonPointToPlaneAlignment(RigidAlignment):
    """GaussNewtonPointToPlaneAlignment.align (alignment.py:91-127) -> pls_align_p2plane."""

    def __init__(self, config: GaussNewtonPointToPlaneConfig, ctx: Optional[_lib.Context] = None, **kwargs):
        super().__init__(config, **kwargs)
        self.gn = _gn_settings(config.gauss_newton_config)
        self._ctx = ctx

    @property
    def ctx(self):
        from .common import default_context
        return self._ctx or default_context()

    def align(self, ref_points, tgt_points, ref_normals=None, initial_estimate=None, mask=None, **kwargs):
        """[B,N,3] points and normals (numpy or torch, host or CUDA, float32 or float64), initial_estimate [B,6] or
        [B,4,4] -> (dT [B,4,4], x [B,6], (w r)^2 [B,N]).  B > 1 aligns the batch in one call (pls_align_p2plane_batch)
        with GaussNewton.compute's joint guards and stop test (optimization.py:318-341)."""
        assert_debug(ref_normals is not None, "The argument 'ref_normals' is required for a point to plane alignemnt")
        check_tensor(tgt_points, [-1, -1, 3])
        b, n = tgt_points.shape[0], tgt_points.shape[1]
        if mask is not None:
            _reject_mask(mask, b, n)
        check_tensor(ref_points, [b, n, 3])
        check_tensor(ref_normals, [b, n, 3])
        is_np = isinstance(tgt_points, np.ndarray)
        is64 = (tgt_points.dtype == (np.float64 if is_np else torch.float64))
        dt_np, dt_t = (np.float64, torch.float64) if is64 else (np.float32, torch.float32)
        conv = (lambda a: np.ascontiguousarray(a, dtype=dt_np)) if is_np else (lambda a: a.to(dt_t).contiguous())
        ref, tgt, nrm = conv(ref_points), conv(tgt_points), conv(ref_normals)
        x0 = None
        if initial_estimate is not None:
            x0 = _initial_params(self.pose, initial_estimate, b, is64, conv)
        mk = (lambda s: np.empty(s, dtype=dt_np)) if is_np else (lambda s: torch.empty(s, dtype=dt_t, device=tgt.device))
        dT, x, loss = mk((b, 4, 4)), mk((b, 6)), mk((b, n))
        gn = (_lib.SCHEMES[self.gn["scheme"]], self.gn["sigma"], self.gn["max_iters"], self.gn["norm_stop"])
        if b == 1:
            self.ctx.call("pls_align_p2plane", _lib.ptr(ref), _lib.ptr(tgt), _lib.ptr(nrm), n, int(is64), *gn,
                          _lib.ptr(x0), _lib.ptr(dT), _lib.ptr(x), _lib.ptr(loss))
        else:
            self.ctx.call("pls_align_p2plane_batch", _lib.ptr(ref), _lib.ptr(tgt), _lib.ptr(nrm), b, n, int(is64), *gn,
                          _lib.ptr(x0), _lib.ptr(dT), _lib.ptr(x), _lib.ptr(loss), None)
        return dT, x, loss


@dataclass
class GNPointToPointConfig(RigidAlignmentConfig):
    """slam/odometry/alignment.py:131-141"""
    mode: str = "point_to_point_gn"
    num_gn_iters: int = 1
    initialize_with_svd: bool = False
    gauss_newton_config: Dict[str, Any] = field(default_factory=lambda: dict(max_iters=1))


class GaussNewtonPointToPointAlignment(RigidAlignment):
    """GaussNewtonPointToPointAlignment.align (alignment.py:144-189) -> pls_align_p2point.

    Faithful to the reference, including its Jacobian (optimization.py:485-501 is r * dr/dx, see gn_device.cuh).
    `initialize_with_svd=True` is rejected: the reference's torch weighted_procrustes builds its output with
    `.repeat(b, 4, 4)` (registration.py:58-59), a [b,16,16] tensor that its own from_pose_matrix shape check then
    refuses -- there is no reference behaviour to reproduce; `weighted_procrustes` (numpy path) is offered
    stand-alone in pylidar_slam_b200.common."""

    def __init__(self, config: GNPointToPointConfig, ctx: Optional[_lib.Context] = None, **kwargs):
        super().__init__(config, **kwargs)
        self.gn = _gn_settings(config.gauss_newton_config)
        self._ctx = ctx

    @property
    def ctx(self):
        from .common import default_context
        return self._ctx or default_context()

    def align(self, ref_points, tgt_points, initial_estimate=None, mask=None, **kwargs):
        """As GaussNewtonPointToPlaneAlignment.align without normals; B > 1 -> pls_align_p2point_batch."""
        assert_debug(not self.config.initialize_with_svd,
                     "initialize_with_svd fails inside the reference itself (registration.py:58-59 builds a [b,16,16] "
                     "tensor); use pylidar_slam_b200.common.weighted_procrustes and pass it as initial_estimate")
        check_tensor(tgt_points, [-1, -1, 3])
        b, n = tgt_points.shape[0], tgt_points.shape[1]
        check_tensor(ref_points, [b, n, 3])
        if mask is not None:
            _reject_mask(mask, b, n)
        is_np = isinstance(tgt_points, np.ndarray)
        is64 = (tgt_points.dtype == (np.float64 if is_np else torch.float64))
        dt_np, dt_t = (np.float64, torch.float64) if is64 else (np.float32, torch.float32)
        conv = (lambda a: np.ascontiguousarray(a, dtype=dt_np)) if is_np else (lambda a: a.to(dt_t).contiguous())
        ref, tgt = conv(ref_points), conv(tgt_points)
        x0 = None
        if initial_estimate is not None:
            x0 = _initial_params(self.pose, initial_estimate, b, is64, conv)
        mk = (lambda s: np.empty(s, dtype=dt_np)) if is_np else (lambda s: torch.empty(s, dtype=dt_t, device=tgt.device))
        dT, x, loss = mk((b, 4, 4)), mk((b, 6)), mk((b, n))
        gn = (_lib.SCHEMES[self.gn["scheme"]], self.gn["sigma"], self.gn["max_iters"], self.gn["norm_stop"])
        if b == 1:
            self.ctx.call("pls_align_p2point", _lib.ptr(ref), _lib.ptr(tgt), n, int(is64), *gn, _lib.ptr(x0), _lib.ptr(dT),
                          _lib.ptr(x), _lib.ptr(loss))
        else:
            self.ctx.call("pls_align_p2point_batch", _lib.ptr(ref), _lib.ptr(tgt), b, n, int(is64), *gn, _lib.ptr(x0),
                          _lib.ptr(dT), _lib.ptr(x), _lib.ptr(loss), None)
        return dT, x, loss


class RIGID_ALIGNMENT(ObjectLoaderEnum, Enum):
    """slam/odometry/alignment.py:200-208"""
    point_to_plane_gauss_newton = (GaussNewtonPointToPlaneAlignment, GaussNewtonPointToPlaneConfig)
    point_to_point_gauss_newton = (GaussNewtonPointToPointAlignment, GNPointToPointConfig)

    @classmethod
    def type_name(cls):
        return "mode"


# ----------------------------------------------------------------------------------------------------------------------
# Odometry
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class OdometryConfig:
    algorithm: str = MISSING


class OdometryAlgorithm(ABC):
    """slam/odometry/odometry.py:21-81"""

    def __init__(self, config: OdometryConfig, **kwargs):
        self.config = config
        self.elapsed: list = []

    @abstractmethod
    def init(self):
        self.elapsed = []

    def process_next_frame(self, data_dict: dict):
        beginning = time.time()
        self.do_process_next_frame(data_dict)
        self.elapsed.append(time.time() - beginning)

    @abstractmethod
    def do_process_next_frame(self, data_dict: dict):
        raise NotImplementedError("")

    def get_relative_poses(self) -> np.ndarray:
        raise NotImplementedError("")

    def get_elapsed(self) -> float:
        return sum(self.elapsed)

    @staticmethod
    def pointcloud_key() -> str:
        return "odometry_pc"

    @staticmethod
    def relative_pose_key() -> str:
        return "odometry_pose"


@dataclass
class ICPFrameToModelConfig(OdometryConfig):
    """icp_odometry.py:27-64 (visualisation fields are accepted and ignored)."""
    algorithm: str = "icp_F2M"
    device: str = "cuda:0"
    pose: str = "euler"
    max_num_alignments: int = 100
    initialization: Any = MISSING
    local_map: Any = MISSING
    alignment: Any = MISSING
    threshold_delta_pose: float = 1.e-4
    threshold_trans: float = 0.1
    threshold_rot: float = 0.3
    sigma: float = 0.1
    data_key: str = "vertex_map"
    viz_debug: bool = False
    viz_with_edl: bool = True
    viz_color_by_elevation: bool = True
    viz_grayscale: str = "viridis"
    viz_num_pcs: int = 500
    viz_z_min: float = 0.0
    viz_z_max: float = 30

    def completed(self):
        """RuntimeDefaultDict.completed (utils.py:199-262): runtime defaults kdtree + point_to_plane_GN."""
        if self.local_map is None or self.local_map == MISSING:
            self.local_map = KdTreeLocalMapConfig()
        if self.alignment is None or self.alignment == MISSING:
            self.alignment = GaussNewtonPointToPlaneConfig()
        return self


class ICPFrameToModel(OdometryAlgorithm):
    """ICPFrameToModel (icp_odometry.py:72-380): the whole frame -- input normalisation, ICP loop,
    key-frame policy, local-map update -- runs inside one `pls_process_frame` call."""

    def __init__(self, config: ICPFrameToModelConfig, projector: SphericalProjector = None, pose: Pose = None,
                 device=None, stream: Optional[int] = None, **kwargs):
        if not isinstance(config, ICPFrameToModelConfig):
            names = {f.name for f in dataclasses.fields(ICPFrameToModelConfig)}
            config = ICPFrameToModelConfig(**{k: v for k, v in _cfg_to_dict(config).items() if k in names})
        config = config.completed()
        super().__init__(config)
        assert_debug(projector is not None)
        self.projector = projector
        self.pose = pose or Pose("euler")
        dev = torch.device(device if device is not None else config.device)
        assert_debug(dev.type == "cuda", "ICPFrameToModel (CUDA) runs on a CUDA device; there is no CPU path")
        self.device = dev

        lm = _cfg_to_dict(self.config.local_map)
        al = _cfg_to_dict(self.config.alignment)
        assert_debug(lm.get("type") in LOCAL_MAP.__members__, f"Unknown type `{lm.get('type')}`")
        assert_debug(al.get("mode", "point_to_plane_gauss_newton") in RIGID_ALIGNMENT.__members__,
                     f"Unknown mode `{al.get('mode')}`")
        # the reference's ICP loop calls align(neigh, tgt, normals) (icp_odometry.py:285-288): with the point-to-point
        # alignment the normals land in `initial_estimate` and its shape check raises -- same error type here
        assert_debug(al.get("mode", "point_to_plane_gauss_newton") == "point_to_plane_gauss_newton",
                     "ICPFrameToModel needs the point-to-plane alignment (the reference's loop cannot drive point_to_point)")
        gn = _gn_settings(al.get("gauss_newton_config", dict(max_iters=1)))
        is_kd = lm["type"] == "kdtree_local_map"
        self.ctx = _lib.Context(
            height=projector.height, width=projector.width, up_fov_deg=float(projector.up_fov),
            down_fov_deg=float(projector.down_fov),
            local_map_type=_lib.MAP_KDTREE if is_kd else _lib.MAP_PROJECTIVE,
            local_map_size=int(lm.get("local_map_size", 20)),
            num_neighbors_normals=int(lm.get("num_neighbors_normals", 10)),
            normals_kernel_size=int(lm.get("normals_kernel_size", 5)),
            scheme=_lib.SCHEMES[gn["scheme"]], sigma=gn["sigma"], gn_max_iters=1,
            gn_norm_stop=gn["norm_stop"], max_num_alignments=int(self.config.max_num_alignments),
            threshold_delta_pose=float(self.config.threshold_delta_pose),
            threshold_trans=float(self.config.threshold_trans), threshold_rot=float(self.config.threshold_rot),
            device=dev.index or 0, stream=stream)
        self.gn_max_iters = self.config.max_num_alignments
        # The fused C-ABI path runs ONE Gauss-Newton step per ICP iteration (the shipped configuration,
        # alignment.py:77).  gauss_newton_config.max_iters > 1 (alignment.py:69-77,110-127: several re-linearised steps on
        # the same correspondences) takes the reference-shaped loop below, built from the fine-grained GPU plug-ins.
        self._fine_grained = gn["max_iters"] > 1
        if self._fine_grained:
            self.ctx.cfg.gn_max_iters = 1  # the context's own fused entry points stay usable (register_new_frame)
            self.local_map = LOCAL_MAP.load(self.config.local_map, projector=projector, ctx=self.ctx)
            self.rigid_alignment = RIGID_ALIGNMENT.load(self.config.alignment, ctx=self.ctx)
            self._pose_ops = Pose("euler", ctx=self.ctx)
            self._delta_since_map_update = torch.eye(4, dtype=torch.float32)
        self.relative_poses: list = []
        self.absolute_poses: list = []
        self._iter = 0
        self.last_info = np.zeros(12, dtype=np.float64)
        self._pose_out = np.zeros((4, 4), dtype=np.float32)
        self._params_out = np.zeros(6, dtype=np.float32)
        # per-frame call arguments that never change: addresses of the persistent output arrays, the has-pose cell
        self._has_pose = C.c_int(0)
        self._out_args = (_lib.ptr(self._pose_out), _lib.ptr(self._params_out), C.byref(self._has_pose),
                          _lib.ptr(self.last_info))

    def init(self):
        super().init()
        self.relative_poses = []
        self.absolute_poses = []
        self._iter = 0
        self.ctx.call("pls_odometry_init")
        if self._fine_grained:
            self.local_map.init()
            self._delta_since_map_update = torch.eye(4, dtype=torch.float32)
            self._sample_pointcloud = False

    def _interpret(self, data):
        """_read_input's three layouts (icp_odometry.py:319-358)."""
        H, W = self.projector.height, self.projector.width
        # float64 clouds keep their precision up to the projection, like the reference (icp_odometry.py:331-352)
        if isinstance(data, np.ndarray):
            check_tensor(data, [-1, 3])
            if data.dtype == np.float64:
                return _lib.INPUT_NDARRAY_F64 | _lib.PTR_HOST, np.ascontiguousarray(data), data.shape[0]
            return _lib.INPUT_NDARRAY | _lib.PTR_HOST, np.ascontiguousarray(data, dtype=np.float32), data.shape[0]
        if isinstance(data, torch.Tensor):
            if data.dim() in (3, 4):
                vm = data if data.dim() == 4 else data.unsqueeze(0)
                assert_debug(vm.shape[0] == 1, "Unexpected batched data format.")
                check_tensor(vm, [1, 3, H, W])
                return _lib.INPUT_VERTEX_MAP, vm.to(torch.float32).contiguous(), 0
            assert_debug(data.dim() == 2)
            check_tensor(data, [-1, 3])
            hint = _lib.PTR_DEVICE if data.is_cuda else _lib.PTR_HOST
            if data.dtype == torch.float64:
                return _lib.INPUT_TENSOR_F64 | hint, data.contiguous(), data.shape[0]
            if data.dtype != torch.float32 or not data.is_contiguous():
                data = data.to(torch.float32).contiguous()
            return _lib.INPUT_TENSOR | hint, data, data.shape[0]
        raise RuntimeError(f"Could not interpret the data: {data} as a pointcloud tensor")

    # -- the reference-shaped loop over the fine-grained plug-ins (icp_odometry.py:157-380), for configurations the fused
    #    path does not cover: the NN search, the normals, every Gauss-Newton step and the map update are the same CUDA
    #    kernels, the loop itself runs here (one host round trip per ICP iteration, like the reference)
    def _process_fine_grained(self, data_dict: dict):
        dev = self.device
        data = data_dict[self.config.data_key]
        if isinstance(data, np.ndarray):                                   # _read_input, icp_odometry.py:319-358
            check_tensor(data, [-1, 3])
            self._sample_pointcloud = True
            pc = torch.from_numpy(data).to(dev).unsqueeze(0)
            vmap = self.projector.build_projection_map(pc.to(torch.float32))
        elif isinstance(data, torch.Tensor):
            if data.dim() in (3, 4):
                vmap = data.to(dev) if data.dim() == 4 else data.to(dev).unsqueeze(0)
                assert_debug(vmap.shape[0] == 1, "Unexpected batched data format.")
                check_tensor(vmap, [1, 3, -1, -1])
                pc = vmap.permute(0, 2, 3, 1).reshape(1, -1, 3)
                pc = pc[:, (pc[0] != 0).any(dim=-1)][:, :1]   # the reference keeps the first non-null pixel only (:342-358)
            else:
                assert_debug(data.dim() == 2)
                pc = data.to(dev).unsqueeze(0)
                vmap = self.projector.build_projection_map(pc.to(torch.float32))
        else:
            raise RuntimeError(f"Could not interpret the data: {data} as a pointcloud tensor")
        vmap = vmap.to(torch.float32)
        vmap = torch.where(torch.isnan(vmap).any(dim=1, keepdim=True), torch.zeros_like(vmap), vmap)   # modify_nan_pmap
        pc = pc.to(torch.float32)
        pc = pc[:, ~torch.isnan(pc[0]).any(dim=-1)]                                                    # remove_nan
        if self._iter == 0:
            eye = torch.eye(4, dtype=torch.float32).unsqueeze(0)
            self.local_map.update(eye, new_vertex_map=vmap)
            self.relative_poses.append(eye.numpy())
            self.absolute_poses.append(np.eye(4, dtype=np.float64))
            self._iter += 1
            return
        init = data_dict.get("init_rpose", None)
        T = torch.eye(4, dtype=torch.float32, device=dev).unsqueeze(0) if init is None else \
            torch.from_numpy(np.asarray(init, dtype=np.float32).reshape(1, 4, 4)).to(dev)
        if self._sample_pointcloud:                                       # sample_points, icp_odometry.py:301-308
            points = pc[0]
        else:
            flat = vmap[0].permute(1, 2, 0).reshape(-1, 3)
            points = flat[flat.norm(dim=-1) > 0.0]
        params = torch.zeros(1, 6, dtype=torch.float32, device=dev)
        self.last_losses = []
        for _ in range(self.config.max_num_alignments):                   # register_new_frame, icp_odometry.py:274-297
            moved = points @ T[0, :3, :3].T + T[0, :3, 3]
            res = self.local_map.nearest_neighbor_search(moved)
            dT, delta, residuals = self.rigid_alignment.align(res.neighbor_points, res.new_target_points, res.neighbor_normals)
            self.last_losses.append(float(residuals.sum()))
            if float(torch.as_tensor(delta).norm()) < self.config.threshold_delta_pose:
                break
            params = self._pose_ops.from_pose_matrix(torch.as_tensor(dT).to(dev) @ T)
            T = self._pose_ops.build_pose_matrix(params)
        self.last_info[0] = len(self.last_losses)
        T_host = T.detach().cpu()
        new_delta = self._delta_since_map_update @ T_host[0]              # __update_map, icp_odometry.py:360-380
        dp = self._pose_ops.from_pose_matrix(new_delta.unsqueeze(0))
        dp = torch.as_tensor(dp).cpu()
        if float(dp[0, :3].norm()) > self.config.threshold_trans or float(dp[0, 3:].norm()) * 180 / np.pi > self.config.threshold_rot:
            self.local_map.update(T_host, new_vertex_map=vmap, new_pc_data=pc[0])
            self._delta_since_map_update = torch.eye(4, dtype=torch.float32)
        else:
            self.local_map.update(T_host)
            self._delta_since_map_update = new_delta
        T_np = T_host.numpy().reshape(4, 4).astype(np.float32)
        self.relative_poses.append(T_np.reshape(1, 4, 4))
        self.absolute_poses.append(self.absolute_poses[-1].dot(euler_pose_matrix_f64(torch.as_tensor(params).cpu().numpy().reshape(6))))
        if "distorted" in data_dict:
            tgt_np_pc = data_dict["distorted"]
        else:
            tgt_np_pc = pc[0].detach().cpu().numpy()
        data_dict[self.pointcloud_key()] = tgt_np_pc
        data_dict[self.relative_pose_key()] = T_np
        self._iter += 1

    def do_process_next_frame(self, data_dict: dict):
        if self._fine_grained:
            self._check_data_key(data_dict)
            return self._process_fine_grained(data_dict)
        layout, data, n, address, init = self._frame_arguments(data_dict)
        self.ctx.call("pls_process_frame", address, layout, n, _lib.ptr(init), *self._out_args)
        self._frame_outputs(data_dict, layout, data)

    def _check_data_key(self, data_dict: dict):
        assert_debug(self.config.data_key in data_dict,
                     f"Could not find the key `{self.config.data_key}` in the input dictionary.\n"
                     f"With keys : {data_dict.keys()}). Set the parameter `slam.odometry.data_key` to the desired key")

    def _frame_arguments(self, data_dict: dict):
        """The C-ABI arguments of one frame: (layout, data, n, address, init pose).  Raises before anything runs."""
        self._check_data_key(data_dict)
        layout, data, n = self._interpret(data_dict[self.config.data_key])
        init = data_dict.get("init_rpose", None)
        init = None if init is None else np.ascontiguousarray(np.asarray(init, dtype=np.float32).reshape(4, 4))
        address = _lib.ptr(data)
        if layout & _lib.PTR_HOST and n == _lib.Handoff.rows:
            # the array GridSample.filter handed out (possibly wrapped by ToTensor): its device-resident twin is used
            # instead of copying the samples host -> device again
            twin = _lib.Handoff.match(address, n, bool((layout & 0xff) >= _lib.INPUT_NDARRAY_F64), int(self.ctx.cfg.device))
            if twin:
                address, layout = twin, (layout & 0xff) | _lib.PTR_DEVICE
        return layout, data, n, address, init

    def _frame_outputs(self, data_dict: dict, layout: int, data):
        """Poses and data_dict entries of a frame whose results are in _pose_out, _params_out, _has_pose, last_info."""
        layout &= 0xff
        if int(self.last_info[6]) == _lib.PLS_W_TINY_RESIDUAL:   # GaussNewton.compute's warning (optimization.py:323-327)
            import logging
            logging.warning("The residual norm is lower than threshold 1e-7. "
                            "This would lead to invalid jacobian. We prefer Stopping ICP")
        if not self._has_pose.value:
            eye = np.eye(4, dtype=np.float32).reshape(1, 4, 4)
            self.relative_poses.append(eye)
            self.absolute_poses.append(np.eye(4, dtype=np.float64))
            self._iter += 1
            return
        T = self._pose_out.copy()
        self.relative_poses.append(T.reshape(1, 4, 4))
        self.absolute_poses.append(self.absolute_poses[-1].dot(euler_pose_matrix_f64(self._params_out)))
        if "distorted" in data_dict:
            tgt_np_pc = data_dict["distorted"]
        elif layout == _lib.INPUT_VERTEX_MAP:
            tgt_np_pc = self.last_info[8:11].astype(np.float32).reshape(1, 3)  # icp_odometry.py:342-358 quirk
        else:
            tgt_np_pc = data if isinstance(data, np.ndarray) else \
                (data.detach().cpu().numpy() if data.is_cuda or data.requires_grad else data.numpy())
            tgt_np_pc = tgt_np_pc.astype(np.float32, copy=False)  # _tgt_pc is float32 (icp_odometry.py:352)
            if self.last_info[5] > 0:
                tgt_np_pc = tgt_np_pc[~np.isnan(tgt_np_pc).any(axis=1)]
        data_dict[self.pointcloud_key()] = tgt_np_pc
        data_dict[self.relative_pose_key()] = T
        self._iter += 1

    def get_relative_poses(self) -> np.ndarray:
        if len(self.relative_poses) == 0:
            return None
        return np.concatenate(self.relative_poses, axis=0)

    # -- fine-grained entry kept for parity tests: register_new_frame (icp_odometry.py:248-299)
    def register_new_frame(self, target_points, initial_estimate=None, **kwargs):
        _check_given_normals(self.ctx)
        pts = _f32c(target_points)
        T0 = None if initial_estimate is None else _pose16(initial_estimate)
        T, params = np.zeros((1, 4, 4), np.float32), np.zeros((1, 6), np.float32)
        losses = np.zeros(self.config.max_num_alignments, np.float32)
        iters = C.c_int(0)
        self.ctx.call("pls_register_frame", _lib.ptr(pts), pts.shape[0], _lib.ptr(T0), _lib.ptr(T), _lib.ptr(params),
                      _lib.ptr(losses), C.byref(iters))
        return params, T, list(losses[:iters.value])

    def register_new_frame_hypotheses(self, target_points, initial_estimates, max_distance: float = np.inf,
                                      min_eigenvalue: float = 0.0):
        """register_new_frame for B initial estimates [B,4,4] of one scan [n,3], in one call (pls_register_hypotheses;
        no reference counterpart): relocalisation in a prior map registers a scan from many guesses -- a yaw sweep, a
        grid of positions, place-recognition candidates -- and keeps the best converged result.  Registers against the
        map this odometry's context holds and leaves it unchanged: a KdTreeLocalMap built with ctx=self.ctx (e.g.
        after set_map_pointcloud), or the odometry's own projective local map, where a sweep of yaw and offset guesses
        recovers a scan that projective association, converging only from a close pose, lost after a fast turn.
        Returns (params [B,6], T [B,4,4], losses: B lists, iterations [B]); hypothesis b's are what
        register_new_frame(target_points, initial_estimates[b]) returns, bit for bit.  A singular hypothesis does not
        stop the others: it is logged, and last_hypotheses_status[b] holds each one's status (PLS_OK,
        PLS_W_TINY_RESIDUAL or PLS_E_SINGULAR).
        max_distance gates the correspondences as in register_new_frames (kd map only: a finite gate on a projective
        map raises before any call).  Gated, the hypotheses are what register_new_frames([target_points],
        initial_estimates, zeros, max_distance) returns, and last_hypotheses_inliers[b] holds each one's inlier count in
        its last iteration (None when ungated).  min_eigenvalue > 0 solves each iteration only in the directions the map
        constrains, as in register_new_frames (kd map only), with last_hypotheses_degenerate and
        last_hypotheses_eigenvalues (None when 0).  The last_registrations_* attributes are left as they are."""
        gated, thresholded = _gated(self.ctx, max_distance), _thresholded(self.ctx, min_eigenvalue)
        if gated or thresholded:
            (params, T, losses, iters, self.last_hypotheses_status, self.last_hypotheses_inliers,
             self.last_hypotheses_degenerate, self.last_hypotheses_eigenvalues) = \
                self._register_scans([target_points], initial_estimates, np.zeros(len(initial_estimates), np.int32),
                                     max_distance, "hypotheses", min_eigenvalue)
            return params, T, losses, iters
        self.last_hypotheses_inliers = None
        self.last_hypotheses_degenerate = self.last_hypotheses_eigenvalues = None
        _check_given_normals(self.ctx)
        check_tensor(target_points, [-1, 3])
        pts = _f32c(target_points)
        if isinstance(initial_estimates, torch.Tensor):
            initial_estimates = initial_estimates.detach().cpu().numpy()
        check_tensor(initial_estimates, [-1, 4, 4])
        T0 = np.ascontiguousarray(initial_estimates, dtype=np.float32)
        B, M = T0.shape[0], int(self.config.max_num_alignments)
        T, params = np.zeros((B, 4, 4), np.float32), np.zeros((B, 6), np.float32)
        losses = np.zeros((B, M), np.float32)
        iters, status = np.zeros(B, np.int32), np.zeros(B, np.int32)
        self.ctx.call("pls_register_hypotheses", _lib.ptr(pts), pts.shape[0], _lib.ptr(T0), B, _lib.ptr(T),
                      _lib.ptr(params), _lib.ptr(losses), _lib.ptr(iters), _lib.ptr(status))
        self.last_hypotheses_status = status
        singular = np.flatnonzero(status == _lib.PLS_E_SINGULAR)
        if singular.size:
            import logging
            logging.error(f"Invalid Jacobian in Gauss Newton minimization, the hessian is not invertible "
                          f"(hypotheses {singular.tolist()})")
        return params, T, [list(losses[b, :iters[b]]) for b in range(B)], iters

    def localize(self, scan, prior_pose, radius: float, cell_size: float, yaw_range: float = np.pi,
                 yaw_step: float = np.deg2rad(5), num_candidates: int = 8, max_distance: float = np.inf,
                 min_eigenvalue: float = 0.0):
        """Finds the pose of `scan` [n,3] on the kd map this odometry's context holds (e.g. loaded with
        KdTreeLocalMap(ctx=self.ctx).set_map_pointcloud) from a coarse prior: start-up on a stored map, recovery after
        odometry is lost.  No reference counterpart.
        1. bases = yaw_sweep(prior_pose, yaw_range, yaw_step);
        2. a correlative search of those bases moved by up to ceil(radius / cell_size) cells along x and y
           (KdTreeLocalMap.search_poses) keeps num_candidates local maxima;
        3. one register_new_frame_hypotheses call refines them from their float32-rounded poses, with the
           correspondence gate max_distance (inf: none; the search and the rescoring are not gated) and the
           eigenvalue threshold min_eigenvalue of its solve (0: none);
        4. score_poses rescores the refined poses.
        The search in step 2 is exact at any radius, and a large one is searched by branch and bound, so `radius` may
        span the whole map when the position is unknown.
        Returns every candidate as a PoseCandidate, ordered by status (singular last), then refined score
        (descending), then search rank.  Needs what register_new_frame_hypotheses needs; IndexError while the map
        carries given normals."""
        _check_given_normals(self.ctx)
        assert_debug(np.isfinite(radius) and radius >= 0, "radius must be finite and >= 0")
        assert_debug(np.isfinite(cell_size) and cell_size > 0, "cell_size must be finite and > 0")
        _gated(self.ctx, max_distance)   # refused before the search
        _thresholded(self.ctx, min_eigenvalue)
        bases = yaw_sweep(prior_pose, yaw_range, yaw_step)
        half = int(np.ceil(radius / cell_size))
        T0, coarse, _ = _pose_search(self.ctx, scan, bases, cell_size, half, half, num_candidates)
        if T0.shape[0] == 0:
            return []
        _, T, _, iters = self.register_new_frame_hypotheses(scan, T0.astype(np.float32), max_distance, min_eigenvalue)
        status = self.last_hypotheses_status
        scores = _score_poses(self.ctx, scan, T.astype(np.float64), cell_size)
        return _pose_candidates(T0, coarse, T, iters, status, scores)

    def localize_scans(self, scans, prior_poses, radius, cell_size: float, yaw_range: float = np.pi,
                       yaw_step: float = np.deg2rad(5), num_candidates: int = 8, max_distance: float = np.inf,
                       min_eigenvalue: float = 0.0):
        """localize for S scans on the one kd map this odometry's context holds (no reference counterpart): a
        localisation server re-localising many vehicles' scans, offline map matching a recorded drive's scans from
        GNSS fixes.  scans: S [n_s,3] arrays or tensors; prior_poses [S,4,4]; radius a scalar or [S].
        One batched search over every scan's yaw_sweep bases (KdTreeLocalMap.search_poses_scans), one
        register_new_frames call over every candidate, one batched rescoring of the refined poses.  Returns S lists of
        PoseCandidate; list s equals localize(scans[s], prior_poses[s], radius[s], cell_size, yaw_range, yaw_step,
        num_candidates, max_distance, min_eigenvalue), field for field; max_distance and min_eigenvalue apply to the
        refinement only."""
        _check_given_normals(self.ctx)
        _gated(self.ctx, max_distance)   # refused before the search
        _thresholded(self.ctx, min_eigenvalue)
        S = len(scans)
        if isinstance(prior_poses, torch.Tensor):
            prior_poses = prior_poses.detach().cpu().numpy()
        check_tensor(prior_poses, [S, 4, 4])
        radii = np.broadcast_to(np.asarray(radius, dtype=np.float64), (S,))
        assert_debug(bool(np.all(np.isfinite(radii) & (radii >= 0))), "radius must be finite and >= 0")
        assert_debug(np.isfinite(cell_size) and cell_size > 0, "cell_size must be finite and > 0")
        bases = [yaw_sweep(prior_poses[s], yaw_range, yaw_step) for s in range(S)]
        halves = [(h, h) for h in (int(np.ceil(r / cell_size)) for r in radii)]
        found = _pose_search_scans(self.ctx, scans, bases, cell_size, halves, num_candidates)
        counts = [T0.shape[0] for T0, _, _ in found]
        if sum(counts) == 0:
            return [[] for _ in range(S)]
        T0_all = np.concatenate([T0 for T0, _, _ in found])
        _, T, _, iters = self.register_new_frames(scans, T0_all.astype(np.float32),
                                                  np.repeat(np.arange(S, dtype=np.int32), counts), max_distance,
                                                  min_eigenvalue)
        status = self.last_registrations_status
        hit = [s for s in range(S) if counts[s]]
        first = np.concatenate([[0], np.cumsum(counts)])
        scores = np.zeros(T.shape[0], np.int32)
        _pose_search_scans(self.ctx, [scans[s] for s in hit],
                           [T[first[s]:first[s + 1]].astype(np.float64) for s in hit], cell_size, [(0, 0)] * len(hit),
                           0, out_scores=scores)
        out = []
        for s in range(S):
            r = slice(first[s], first[s + 1])
            out.append(_pose_candidates(found[s][0], found[s][1], T[r], iters[r], status[r], scores[r]) if counts[s]
                       else [])
        return out

    def register_new_frames(self, scans, initial_estimates, scan_indices=None, max_distance: float = np.inf,
                            min_eigenvalue: float = 0.0):
        """register_new_frame for many scans against the one map this odometry's context holds, in one call
        (pls_register_scans; no reference counterpart): a localisation server registers many vehicles' scans on one
        city map, offline map matching registers a recorded drive's scans on a prior map.  `scans` is a list of S
        [n_i,3] arrays or tensors, `initial_estimates` [B,4,4], and registration b registers scans[scan_indices[b]]
        from initial_estimates[b] (scan_indices None: scan b, which needs B == S).  The map is a kd map, e.g. one loaded
        with KdTreeLocalMap(ctx=self.ctx).set_map_pointcloud; it is left unchanged.
        Returns (params [B,6], T [B,4,4], losses: B lists, iterations [B]); registration b's are what
        register_new_frame(scans[scan_indices[b]], initial_estimates[b]) returns, bit for bit.  A singular registration
        does not stop the others: it is logged, and last_registrations_status[b] holds each one's status (PLS_OK,
        PLS_W_TINY_RESIDUAL or PLS_E_SINGULAR).
        A finite max_distance gates the correspondences (pls_register_scans_gated): in every ICP iteration a valid row
        is an inlier when the float64 squared distance to its exact nearest map point is at most max_distance**2, and
        only inliers enter the normal equations, the loss and the count, so a stale prior map -- moved cars,
        construction, partial overlap -- cannot pull the pose towards far matches.  A registration left with too few
        inliers, or none, ends singular (PLS_E_SINGULAR) without stopping the others.  last_registrations_inliers[b]
        then holds registration b's inlier count in its last iteration (None when ungated).  max_distance = inf, the
        default, makes the ungated call, bit for bit as before; NaN or a negative gate raises before any call.
        min_eigenvalue > 0 solves every ICP iteration only in the directions the map constrains
        (pls_register_scans_degeneracy): a tunnel, a corridor or a flat field leaves some directions unconstrained, and
        there the pose keeps its initial estimate instead of sliding on noise or ending singular.  With H the
        iteration's 6x6 normal-equation matrix and N its inlier (or match) count, an eigen-direction of H is kept when
        its eigenvalue is at least min_eigenvalue * N.  The threshold mixes units: per point, translation eigenvalues
        are dimensionless (at most 1 unweighted) and rotation eigenvalues are in m^2; calibrate it from
        evaluate_registrations' eigenvalues / inliers on your own map.  last_registrations_degenerate [B] then holds
        each registration's number of degenerate directions and last_registrations_eigenvalues [B,6] the ascending
        eigenvalues of H / N, both of its last iteration (None when min_eigenvalue is 0).  0, the default, makes the
        call made without it; NaN, a negative or an infinite threshold raises before any call."""
        (params, T, losses, iters, self.last_registrations_status, self.last_registrations_inliers,
         self.last_registrations_degenerate, self.last_registrations_eigenvalues) = \
            self._register_scans(scans, initial_estimates, scan_indices, max_distance, "registrations", min_eigenvalue)
        return params, T, losses, iters

    def _register_scans(self, scans, initial_estimates, scan_indices, max_distance, what, min_eigenvalue=0.0):
        """register_new_frames' call: (params, T, losses, iterations, status, inliers or None, degenerate counts or
        None, eigenvalues or None), singular ones logged as `what`."""
        gated, thresholded = _gated(self.ctx, max_distance), _thresholded(self.ctx, min_eigenvalue)
        pts, addresses, rows, T0, index = self._scans_args(scans, initial_estimates, scan_indices)
        B, S, M = T0.shape[0], len(pts), int(self.config.max_num_alignments)
        T, params = np.zeros((B, 4, 4), np.float32), np.zeros((B, 6), np.float32)
        losses = np.zeros((B, M), np.float32)
        iters, status = np.zeros(B, np.int32), np.zeros(B, np.int32)
        inliers = np.zeros(B, np.int32) if gated else None
        degenerate = eigenvalues = None
        if thresholded:
            degenerate, eigenvalues = np.zeros(B, np.int32), np.zeros((B, 6), np.float64)
            self.ctx.call("pls_register_scans_degeneracy", _lib.ptr(addresses), _lib.ptr(rows), S, _lib.ptr(index),
                          _lib.ptr(T0), B, float(max_distance), float(min_eigenvalue), _lib.ptr(T), _lib.ptr(params),
                          _lib.ptr(losses), _lib.ptr(iters), _lib.ptr(status), _lib.ptr(inliers),
                          _lib.ptr(degenerate), _lib.ptr(eigenvalues))
        elif gated:
            self.ctx.call("pls_register_scans_gated", _lib.ptr(addresses), _lib.ptr(rows), S, _lib.ptr(index),
                          _lib.ptr(T0), B, float(max_distance), _lib.ptr(T), _lib.ptr(params), _lib.ptr(losses),
                          _lib.ptr(iters), _lib.ptr(status), _lib.ptr(inliers))
        else:
            self.ctx.call("pls_register_scans", _lib.ptr(addresses), _lib.ptr(rows), S, _lib.ptr(index), _lib.ptr(T0),
                          B, _lib.ptr(T), _lib.ptr(params), _lib.ptr(losses), _lib.ptr(iters), _lib.ptr(status))
        singular = np.flatnonzero(status == _lib.PLS_E_SINGULAR)
        if singular.size:
            import logging
            logging.error(f"Invalid Jacobian in Gauss Newton minimization, the hessian is not invertible "
                          f"({what} {singular.tolist()})")
        return params, T, [list(losses[b, :iters[b]]) for b in range(B)], iters, status, inliers, degenerate, eigenvalues

    def _scans_args(self, scans, poses, scan_indices):
        """register_new_frames' and evaluate_registrations' inputs as pls_register_scans / pls_kdmap_evaluate_poses
        take them: (float32 scans kept alive, their addresses [S], rows [S], poses [B,4,4] float32, scan_of [B] int32 or
        None).  IndexError while the map carries given normals."""
        _check_given_normals(self.ctx)
        pts = []
        for scan in scans:
            check_tensor(scan, [-1, 3])
            pts.append(_f32c(scan))
        if isinstance(poses, torch.Tensor):
            poses = poses.detach().cpu().numpy()
        check_tensor(poses, [-1, 4, 4])
        T0 = np.ascontiguousarray(poses, dtype=np.float32)
        B = T0.shape[0]
        index = None
        if scan_indices is not None:
            if isinstance(scan_indices, torch.Tensor):
                scan_indices = scan_indices.detach().cpu().numpy()
            index = np.ascontiguousarray(scan_indices, dtype=np.int32).reshape(-1)
            assert_debug(index.shape[0] == B, f"scan_indices must hold one scan index per initial estimate ({B})")
        addresses = np.array([_lib.ptr(p) for p in pts], dtype=np.uint64)
        rows = np.array([p.shape[0] for p in pts], dtype=np.int64)
        return pts, addresses, rows, T0, index

    def evaluate_registrations(self, scans, poses, max_distance: float = np.inf, scan_indices=None) -> list:
        """The quality of B poses of S scans on the kd map this odometry's context holds, in one call
        (pls_kdmap_evaluate_poses; no reference counterpart): an inlier fraction, an inlier RMSE and an information
        matrix per pose, for a filter or a pose graph fed by a localiser, for accepting or rejecting a registration,
        and for re-ranking localize's candidates (one call on their T).  Inputs as register_new_frames: `scans` S
        [n_i,3] arrays or tensors, `poses` [B,4,4], pose b applied to scans[scan_indices[b]] (None: scan b, B == S).
        A valid row is an inlier when its exact nearest map point lies within max_distance (>= 0; inf admits every
        match).  Nothing is solved and the map is left unchanged.  Returns B RegistrationQuality; with max_distance
        inf, pose b's information matrix is built from the sums the first ICP iteration of
        register_new_frame(scans[scan_indices[b]], poses[b]) forms.  IndexError while the map carries given normals."""
        pts, addresses, rows, T, index = self._scans_args(scans, poses, scan_indices)
        B = T.shape[0]
        stats = np.zeros((B, _lib.EVAL_STATS), np.float64)
        self.ctx.call("pls_kdmap_evaluate_poses", _lib.ptr(addresses), _lib.ptr(rows), len(pts), _lib.ptr(index),
                      _lib.ptr(T), B, float(max_distance), _lib.ptr(stats))
        return [RegistrationQuality.from_stats(stats[b]) for b in range(B)]


class ICPFrameToModelBatch:
    """Advances several independent ICPFrameToModel sequences by one frame each in ONE `pls_process_frames` call (no
    reference counterpart: the reference's runner processes the sequences of a dataset one after another,
    odometry_runner.py:145-175).  Every kernel of an ICP iteration is one launch for all of them, and every sequence
    computes exactly what its own process_next_frame would: its poses, data_dict entries and local map.  Each odometry
    keeps its own state, so process_next_frame and process_next_frames may be mixed on the same objects.

        odos = [ICPFrameToModel(cfg, projector=proj) for _ in range(B)]
        batch = ICPFrameToModelBatch(odos)
        for o in odos: o.init()
        batch.process_next_frames([dd0, dd1, None, dd3])   # None: no frame for that sequence this step

    Supported: kd-tree or projective local maps (one type per batch; the sequences may differ in every other setting,
    frame size and local_map_size included), gauss_newton_config.max_iters == 1, one CUDA device, at most 64
    sequences."""

    def __init__(self, odometries):
        odos = list(odometries)
        assert_debug(1 <= len(odos) <= _lib.MAX_SEQUENCES, f"between 1 and {_lib.MAX_SEQUENCES} odometries")
        for o in odos:
            assert_debug(isinstance(o, ICPFrameToModel), "ICPFrameToModelBatch batches ICPFrameToModel objects")
            assert_debug(not o._fine_grained, "batched sequences need gauss_newton_config.max_iters == 1")
            assert_debug(o.ctx.cfg.local_map_type == odos[0].ctx.cfg.local_map_type,
                         "batched sequences share one local map type: all kd-tree or all projective")
        assert_debug(len({id(o) for o in odos}) == len(odos), "an odometry is listed twice")
        assert_debug(len({int(o.ctx.cfg.device) for o in odos}) == 1, "every odometry must run on one CUDA device")
        self.odometries = odos
        B = len(odos)
        self._handles = (C.c_void_p * B)(*[o.ctx.handle.value for o in odos])
        self._poses = np.zeros((B, 16), np.float32)
        self._params = np.zeros((B, 6), np.float32)
        self._has_pose = np.zeros(B, np.int32)
        self._info = np.zeros((B, 12), np.float64)
        self._status = np.zeros(B, np.int32)

    def process_next_frames(self, data_dicts):
        """data_dicts[i] is the next frame of sequence i, or None to leave it alone.  Each data_dict receives what
        process_next_frame writes; a singular ICP raises RuntimeError after every other sequence's data_dict is filled."""
        odos = self.odometries
        B = len(odos)
        assert_debug(len(data_dicts) == B, f"one data_dict (or None) per odometry: {B} expected")
        beginning = time.time()
        args = [None if dd is None else o._frame_arguments(dd) for o, dd in zip(odos, data_dicts)]
        active = [i for i in range(B) if args[i] is not None]
        if not active:
            return
        data = (C.c_void_p * B)(*[None if a is None else a[3] for a in args])
        layouts = (C.c_int * B)(*[0 if a is None else a[0] for a in args])
        n = (C.c_int64 * B)(*[0 if a is None else a[2] for a in args])
        inits = (C.c_void_p * B)(*[None if a is None else _lib.ptr(a[4]) for a in args])
        if _lib._cuda_inputs:   # CUDA tensors: their producers on PyTorch's current stream go first
            devices = list(_lib._cuda_inputs)
            _lib._cuda_inputs.clear()
            for d in devices:
                if d == int(odos[0].ctx.cfg.device):
                    stream = torch.cuda.current_stream(d).cuda_stream
                    for i in active:
                        odos[i].ctx.call("pls_wait_stream", stream)
                else:
                    torch.cuda.current_stream(d).synchronize()
        self._status[:] = _lib.PLS_OK
        status = odos[active[0]].ctx.process_frames(self._handles, B, data, layouts, n, 0.0, inits, _lib.ptr(self._poses),
                                                    _lib.ptr(self._params), _lib.ptr(self._has_pose),
                                                    _lib.ptr(self._info), _lib.ptr(self._status))
        # every sequence whose frame completed gets its outputs, also when another one failed
        done = [i for i in active if self._status[i] == _lib.PLS_OK]
        for i in done:
            o = odos[i]
            o._pose_out[:] = self._poses[i].reshape(4, 4)
            o._params_out[:] = self._params[i]
            o._has_pose.value = int(self._has_pose[i])
            o.last_info[:] = self._info[i]
            o._frame_outputs(data_dicts[i], args[i][0], args[i][1])
        share = (time.time() - beginning) / len(active)
        for i in done:
            odos[i].elapsed.append(share)
        failed = [i for i in active if self._status[i] not in (_lib.PLS_OK, _lib.PLS_E_SINGULAR)]
        if failed or status not in (_lib.PLS_OK, _lib.PLS_E_SINGULAR):
            bad = failed[0] if failed else active[0]
            odos[bad].ctx.check(int(self._status[bad]) if failed else status)
        singular = [i for i in active if self._status[i] == _lib.PLS_E_SINGULAR]
        if singular:
            import logging
            logging.error("Invalid Jacobian in Gauss Newton minimization, the hessian is not invertible")
            raise RuntimeError(f"Invalid Jacobian in Gauss Newton minimization (sequences {singular})")


class ODOMETRY(ObjectLoaderEnum, Enum):
    """slam/odometry/__init__.py:23-32"""
    icp_F2M = (ICPFrameToModel, ICPFrameToModelConfig)

    @classmethod
    def type_name(cls):
        return "algorithm"
