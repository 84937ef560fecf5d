"""Reference definition of the robot-shaped collision check (fiesta_check_poses, fiesta_b200/csrc/fb_pose.h) in numpy, written from
the definition alone, for the CPU oracle test, the GPU tests and scripts/pose_bench.py.

Every fp64 operation is a separate numpy or Python float operation (rounded on its own, no contraction), in the definition's order.
The separating-axis test runs on every voxel of a window `margin` voxels wider than the candidate range on each side, so the test
also checks that the candidate range holds every touched voxel.  It works on an export_distance() array (-10000 never observed).
"""
import math

import numpy as np

R_MAX = 1.0 + 2.0 ** -20
UNDEFINED, INFINITY = -10000.0, 10000.0


def valid(pose, lo, hi):
    """Status 2 rule: p has a NaN or fails PosInMap, an R entry is non-finite or |R_jk| > 1 + 2^-20."""
    p = [float(x) for x in pose[:3]]
    if any(math.isnan(x) for x in p) or not all(lo[k] <= p[k] <= hi[k] for k in range(3)):
        return False
    return all(abs(float(x)) <= R_MAX for x in pose[3:12])               # NaN compares False


def axes(R):
    """The 15 axes: e_0..e_2, u_0..u_2, then e_k x u_j with k slowest."""
    u = [[float(R[j][i]) for i in range(3)] for j in range(3)]
    out = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]] + u
    for k in range(3):
        for j in range(3):
            a = u[j]
            out.append([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]][k])
    return out


def dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def thresholds(R, h, r):
    u = [[float(R[j][i]) for i in range(3)] for j in range(3)]
    return [r * ((abs(L[0]) + abs(L[1])) + abs(L[2])) + ((h[0] * abs(dot(u[0], L)) + h[1] * abs(dot(u[1], L))) + h[2] * abs(dot(u[2], L)))
            for L in axes(R)]


def candidate_range(pose, h, origin, res):
    """(lo, hi) inclusive voxel bounds per axis."""
    R = np.asarray(pose[3:12], np.float64).reshape(3, 3)
    lo, hi = [], []
    for k in range(3):
        e = (h[0] * abs(float(R[0, k])) + h[1] * abs(float(R[1, k]))) + h[2] * abs(float(R[2, k]))
        p = float(pose[k])
        lo.append(math.floor((p - e - origin[k]) / res) - 1)
        hi.append(math.floor((p + e - origin[k]) / res) + 1)
    return np.array(lo), np.array(hi)


def touched(pose, h, origin, res, margin=3):
    """(window lower corner (3,), touched mask over the window, candidate (lo, hi)) of a valid pose."""
    h = [float(x) for x in h]
    R = np.asarray(pose[3:12], np.float64).reshape(3, 3)
    clo, chi = candidate_range(pose, h, origin, res)
    wlo, whi = clo - margin, chi + margin
    L, T = axes(R), thresholds(R, h, 0.5 * res)
    d = []
    for k in range(3):
        v = np.arange(wlo[k], whi[k] + 1).astype(np.float64)
        d.append(((v + 0.5) * res + float(origin[k])) - float(pose[k]))
    d0, d1, d2 = d[0][:, None, None], d[1][None, :, None], d[2][None, None, :]
    hit = np.ones((len(d[0]), len(d[1]), len(d[2])), bool)
    for Lk, Tk in zip(L, T):
        proj = (Lk[0] * d0 + Lk[1] * d1) + Lk[2] * d2
        hit &= ~(np.abs(proj) > Tk)
    return wlo, hit, (clo, chi)


def outcome(wlo, hit, D, clearance, unknown_blocks):
    """(status, n_blocked, hit_idx) of a valid pose from its touched mask; D: (gx, gy, gz) export_distance() values."""
    gs = np.asarray(D.shape)
    idx = np.argwhere(hit) + wlo
    ing = np.all((idx >= 0) & (idx < gs), axis=1)
    inside = idx[ing]
    Dv = D[inside[:, 0], inside[:, 1], inside[:, 2]]
    gd = np.where(Dv < 0, INFINITY, Dv)                                   # GetDistance(Vector3i)
    blk = (gd <= clearance) | (unknown_blocks & (Dv == UNDEFINED))
    if blk.any():
        b = inside[blk]
        lin = (b[:, 0] * int(gs[1]) + b[:, 1]) * int(gs[2]) + b[:, 2]
        return 1, int(blk.sum()), int(lin.min())
    return (3 if (~ing).any() else 0), 0, -1


def check(pose, h, origin, res, lo, hi, D, clearance, unknown_blocks):
    if not valid(pose, lo, hi):
        return 2, 0, -1
    wlo, hit, _ = touched(pose, h, origin, res)
    return outcome(wlo, hit, D, clearance, unknown_blocks)


def check_all(poses, h, origin, res, lo, hi, D, settings):
    """{(clearance, unknown_blocks): (status, n_blocked, hit_idx) arrays} for every setting, one touched mask per pose."""
    rows = {s: [] for s in settings}
    for pose in poses:
        t = touched(pose, h, origin, res) if valid(pose, lo, hi) else None
        for s in settings:
            rows[s].append((2, 0, -1) if t is None else outcome(t[0], t[1], D, *s))
    return {s: (np.array([r[0] for r in v], np.int32), np.array([r[1] for r in v], np.int32), np.array([r[2] for r in v], np.int64))
            for s, v in rows.items()}


# --- pose generators shared by the tests and the benchmark
def rot_x(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def rot_z(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def random_rotations(rng, n):
    """Uniform random rotations (from unit quaternions), as (n, 3, 3) row-major matrices."""
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


def yaw_rotations(rng, n):
    return np.stack([rot_z(a) for a in rng.uniform(0, 2 * np.pi, n)])


def poses(p, R):
    return np.ascontiguousarray(np.concatenate([np.asarray(p, np.float64).reshape(-1, 3), np.asarray(R, np.float64).reshape(-1, 9)], 1))


def adversarial(rng, origin, res, gs, h):
    """Poses that probe the boundaries of the definition for half extents h: axis-aligned boxes whose faces lie exactly on voxel
    faces, 45-degree turns, R entries at and just above 1 + 2^-20, NaN and infinite entries, centres on and just outside every
    face of the map and boxes across every face."""
    o, gs = np.asarray(origin, np.float64), np.asarray(gs)
    hi = o + gs * res
    c = o + np.floor(gs / 2) * res                                       # a voxel corner near the middle
    out = []
    I = np.eye(3)
    for cen in (c, c + 0.5 * res, c + np.array([0.5, 0.0, 0.25]) * res):
        for R in (I, rot_z(math.pi / 4), rot_x(math.pi / 4) @ rot_z(math.pi / 4), rot_z(math.pi / 2), -I):
            out.append((cen, R))
    big = np.full((3, 3), R_MAX)
    for R in (I * R_MAX, -I * R_MAX, I * np.nextafter(R_MAX, 2.0), big, np.where(I > 0, np.nan, 0.0), np.where(I > 0, np.inf, 0.0),
              np.where(I > 0, -np.inf, 0.0), np.zeros((3, 3))):
        out.append((c, R))
    for bad in ((np.nan, 0, 0), (0, np.inf, 0), (0, 0, -np.inf)):
        out.append((c + np.array(bad), I))
    for k in range(3):
        for side in (o, hi):
            for off in (0.0, 0.25 * res, -0.25 * res, 1e-9):
                p = c.copy()
                p[k] = side[k] + off
                out.append((p, I))
                out.append((p, rot_z(0.3) @ rot_x(0.2)))
            p = c.copy()
            p[k] = side[k] + (h[k] if side is o else -h[k])               # a face exactly on the map's face
            out.append((p, I))
    for _ in range(10):
        out.append((o + rng.uniform(0, 1, 3) * gs * res, random_rotations(rng, 1)[0]))
    return poses([p for p, _ in out], [R for _, R in out])
