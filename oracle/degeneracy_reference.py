"""TEST INFRASTRUCTURE ONLY -- a float64 restatement of the eigenvalue-thresholded solve of
pls_register_scans_degeneracy (include/plslam_b200.h), and of the scenes it is for.

  * projected_step: an iteration's 30 sums in; numpy.linalg.eigh of H, the kept directions (N > 0 and
    lambda >= min_eigenvalue * N), the step dx = -sum over the kept of v (v^T g) / lambda and H / N's eigenvalues out;
  * flat_field_scene: a map and a scan exactly on z = 0, so that x, y and yaw are exactly unconstrained;
  * tunnel_scene: a straight box tunnel along x with millimetre noise, so that only the translation along the axis is
    nearly unconstrained; TUNNEL_MIN_EIGENVALUE lies inside its eigenvalue gap.
"""
import numpy as np

from oracle import kd_icp_reference as kref

# The tunnel's eigenvalues of H / N (test_degeneracy_cpu.test_tunnel_eigenvalue_gap): the one along the axis is 3e-3 to
# 6e-3 (the mean squared x component of the k-NN normals, tilted by the noise), the next smallest, across the axis,
# about 0.2: 0.03 leaves a factor of 5 on either side.
TUNNEL_MIN_EIGENVALUE = 0.03
# The flat field's kept eigenvalues of H / N are those of z, roll and pitch (1 and the field's second moments, m^2);
# its other three are exactly 0, so any positive threshold below the kept ones separates them.
FLAT_MIN_EIGENVALUE = 1e-3


def hessian(sums):
    """H [6,6] from the 21 upper-triangle entries of the sums."""
    H = np.zeros((6, 6))
    for k, (a, b) in enumerate(kref._UPPER):
        H[a, b] = H[b, a] = sums[k]
    return H


def projected_step(sums, min_eigenvalue):
    """(step [6], kept [6] bool, eigenvalues of H / N [6] ascending; zeros when N = 0)."""
    sums = np.asarray(sums, np.float64)
    w, v = np.linalg.eigh(hessian(sums))
    g = sums[21:27]
    N = float(sums[29])
    kept = (w >= float(min_eigenvalue) * N) if N > 0 else np.zeros(6, bool)
    step = np.zeros(6)
    for k in range(6):
        if kept[k]:
            step -= v[:, k] * (v[:, k] @ g) / w[k]
    return step, kept, (w / N if N > 0 else np.zeros(6))


def _pose(x, y, z, roll, pitch, yaw):
    """The 4x4 float64 pose of build_pose's Euler convention (R = Rz Ry Rx)."""
    cx, sx, cy, sy, cz, sz = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:3, :3] = [[cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx],
                 [sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx],
                 [-sy, cy * sx, cy * cx]]
    T[:3, 3] = [x, y, z]
    return T


def flat_field_scene(seed=0, map_points=120000, scan_points=20000):
    """A 60 x 60 m field: map and scan points exactly on z = 0 (float32), so that every map normal is exactly +-z and
    the tx, ty and rz rows of J^T W J are exactly zero.  The truth is x = 2, y = -1, yaw = 0.3 on the plane; the start
    adds 5 cm in z and 3 mrad in roll and pitch -- the directions the field constrains -- and keeps the truth's x, y
    and yaw.  Returns (map [M,3], scan [N,3], truth [4,4], start [4,4]) float32."""
    rng = np.random.RandomState(seed)
    m = np.zeros((map_points, 3), np.float32)
    m[:, :2] = rng.uniform(-30, 30, (map_points, 2))
    s = np.zeros((scan_points, 3), np.float32)
    s[:, :2] = rng.uniform(-20, 20, (scan_points, 2))   # in the scan frame: the field's plane is its z = 0 too
    truth = _pose(2.0, -1.0, 0.0, 0.0, 0.0, 0.3)
    start = _pose(2.0, -1.0, 0.05, 3e-3, -3e-3, 0.3)
    return m, s, truth.astype(np.float32), start.astype(np.float32)


def tunnel_scene(seed=0, map_points=200000, scan_points=30000, noise=1e-3):
    """A straight 200 m box tunnel along x, 8 m wide (y in [-4, 4]) and 6 m high (z in [0, 6]): floor, ceiling and two
    walls, each point moved by N(0, noise) along its surface normal.  The scan sees the tunnel within 40 m of the truth
    (the identity), with its own noise.  The start is 0.5 m along the axis, 2 cm / -1.5 cm across it and 1 mrad in
    roll, pitch and yaw away.  Returns (map [M,3], scan [N,3], truth [4,4], start [4,4]) float32."""
    rng = np.random.RandomState(seed)

    def surfaces(n, x0, x1):
        per = n // 4
        x = rng.uniform(x0, x1, 4 * per)
        out = np.zeros((4 * per, 3))
        out[:, 0] = x
        a, b = rng.uniform(-4, 4, per), rng.uniform(0, 6, per)
        e = rng.normal(0, noise, 4 * per)
        out[:per, 1], out[:per, 2] = a, 0.0 + e[:per]                            # floor
        out[per:2 * per, 1], out[per:2 * per, 2] = a[::-1], 6.0 + e[per:2 * per]  # ceiling
        out[2 * per:3 * per, 1], out[2 * per:3 * per, 2] = -4.0 + e[2 * per:3 * per], b          # wall y = -4
        out[3 * per:, 1], out[3 * per:, 2] = 4.0 + e[3 * per:], b[::-1]                         # wall y = +4
        return out.astype(np.float32)

    m = surfaces(map_points, -100, 100)
    s = surfaces(scan_points, -40, 40)
    truth = np.eye(4)
    start = _pose(0.5, 0.02, -0.015, 1e-3, -1e-3, 1e-3)
    return m, s, truth.astype(np.float32), start.astype(np.float32)


def euler(T):
    """(x, y, z, roll, pitch, yaw) of a pose, as from_pose reads it (no gimbal branch: |pitch| < pi / 2)."""
    T = np.asarray(T, np.float64)
    R = T[:3, :3]
    return np.array([T[0, 3], T[1, 3], T[2, 3], np.arctan2(R[2, 1], R[2, 2]),
                     np.arctan2(-R[2, 0], np.hypot(R[0, 0], R[1, 0])), np.arctan2(R[1, 0], R[0, 0])])


def sums_at(map_f32, scan_f32, T, k=10, scheme="default", sigma=0.3):
    """The float64 accumulators of one ungated iteration at pose T (exact 1-NN and exact k-NN normals)."""
    from scipy.spatial import cKDTree
    tree = cKDTree(np.asarray(map_f32, np.float64))
    p = kref.transform(np.asarray(T, np.float64), np.asarray(scan_f32, np.float64))
    _, nb = tree.query(p, k=1, workers=-1)
    u, inv = np.unique(nb, return_inverse=True)
    nrm = kref.exact_normals(map_f32, tree, u, k)[0][inv]
    return kref.accumulate(p, np.asarray(map_f32, np.float64)[nb], nrm, scheme, sigma)
