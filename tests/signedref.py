"""CPU definition of the signed field of a voxel box (include/fiesta_b200.h, fiesta_signed_*; DESIGN.md §3.13).

q is the exact integer squared Euclidean distance from each obstacle voxel of the box to the nearest non-obstacle voxel of the box,
taken from scipy.ndimage.distance_transform_edt's nearest-voxel indices (not from its floating-point distances), and S follows the
header's formula, one fp64 operation at a time.  `brute_q` is the O(n^2) definition the tests hold the model to."""
import numpy as np
from scipy import ndimage

NONE = 0x7fffffff          # FB_SIGNED_NONE: an obstacle of a box without non-obstacle voxels


def box_slices(box):
    lo, hi = box
    return tuple(slice(int(a), int(b) + 1) for a, b in zip(lo, hi))


def obstacle_mask(D_export, gs, box):
    """Obstacle voxels of the box: distance reads exactly 0 in fiesta_export_distance."""
    return np.asarray(D_export).reshape(gs)[box_slices(box)] == 0.0


def depth_sq(obst):
    """q per voxel of the boolean obstacle mask: 0 on non-obstacles, the exact squared distance to the nearest non-obstacle on
    obstacles, NONE on obstacles when the mask holds no non-obstacle."""
    obst = np.asarray(obst, bool)
    q = np.zeros(obst.shape, np.int64)
    if not obst.any():
        return q
    if obst.all():
        q[:] = NONE
        return q
    idx = ndimage.distance_transform_edt(obst, return_distances=False, return_indices=True)
    grid = np.indices(obst.shape)
    q = np.sum((idx.astype(np.int64) - grid) ** 2, axis=0)
    return np.where(obst, q, 0)


def brute_q(obst):
    """The definition itself: for every obstacle, the least squared distance to any non-obstacle of the box (O(n^2))."""
    obst = np.asarray(obst, bool)
    q = np.zeros(obst.shape, np.int64)
    free = np.argwhere(~obst)
    for v in np.argwhere(obst):
        q[tuple(v)] = NONE if len(free) == 0 else int(np.min(np.sum((free - v) ** 2, axis=1)))
    return q


def signed_values(q, D_box, res):
    """S from q and the box's GetDistance(Vector3i) values (never observed -> +10000)."""
    d = np.where(np.asarray(D_box) < 0, 10000.0, np.asarray(D_box, np.float64))
    with np.errstate(invalid="ignore"):
        depth = (1.0 - np.sqrt(q.astype(np.float64))) * res
    depth = np.where(q == NONE, -np.inf, depth)
    return np.where(q == 0, d, depth)


def field(D_export, gs, box, res):
    """(S, q) of the box on the map whose fiesta_export_distance is D_export."""
    obst = obstacle_mask(D_export, gs, box)
    q = depth_sq(obst)
    return signed_values(q, np.asarray(D_export).reshape(gs)[box_slices(box)], res), q


def stats(q):
    """fiesta_signed_stats of a q array."""
    obst = q > 0
    finite = obst & (q != NONE)
    n_obst = int(obst.sum())
    return dict(box_voxels=int(q.size), obstacles=n_obst, interior=int(np.sum(q > 1)),
                max_depth_sq=-1 if n_obst == q.size else (int(q[finite].max()) if finite.any() else 0))


def grid_values(D_export, gs, box, S):
    """The grid's GetDistance(Vector3i) values (never observed -> +10000) with the box overwritten by S: what the signed queries
    read at each voxel."""
    D = np.where(np.asarray(D_export) < 0, 10000.0, np.asarray(D_export, np.float64)).reshape(gs).copy()
    D[box_slices(box)] = S
    return D


def trilinear(V, gs, q, origin, res):
    """tests/geometry.trilinear on voxel values V (gs-shaped, negative values kept: geometry.trilinear maps an export's negatives
    to +10000 first, which would erase the depths) -> (dist, grad, in_map).  Same operations in the same order."""
    V = np.asarray(V, np.float64).reshape(gs)
    q = np.asarray(q, np.float64).reshape(-1, 3)
    o = np.asarray(origin, np.float64)
    in_map = np.all((q >= o) & (q <= o + np.asarray(gs) * res), axis=1)
    res_inv = 1.0 / res
    idx = np.floor(((q - 0.5 * res) - o) / res).astype(np.int64)
    diff = (q - ((idx + 0.5) * res + o)) * res_inv
    val = {}
    for c in [(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)]:
        v = idx + np.array(c)
        ok = np.all((v >= 0) & (v < np.asarray(gs)), axis=1)
        vc = np.where(ok[:, None], v, 0)
        val[c] = np.where(ok, V[vc[:, 0], vc[:, 1], vc[:, 2]], 10000.0)
    d0, d1, d2 = diff[:, 0], diff[:, 1], diff[:, 2]
    with np.errstate(invalid="ignore"):
        v00 = (1 - d0) * val[0, 0, 0] + d0 * val[1, 0, 0]
        v01 = (1 - d0) * val[0, 0, 1] + d0 * val[1, 0, 1]
        v10 = (1 - d0) * val[0, 1, 0] + d0 * val[1, 1, 0]
        v11 = (1 - d0) * val[0, 1, 1] + d0 * val[1, 1, 1]
        v0 = (1 - d1) * v00 + d1 * v10
        v1 = (1 - d1) * v01 + d1 * v11
        dist = (1 - d2) * v0 + d2 * v1
        g = np.empty((len(q), 3))
        g[:, 2] = (v1 - v0) * res_inv
        g[:, 1] = ((1 - d2) * (v10 - v00) + d2 * (v11 - v01)) * res_inv
        g0 = (1 - d2) * (1 - d1) * (val[1, 0, 0] - val[0, 0, 0])
        g0 = g0 + (1 - d2) * d1 * (val[1, 1, 0] - val[0, 1, 0])
        g0 = g0 + d2 * (1 - d1) * (val[1, 0, 1] - val[0, 0, 1])
        g0 = g0 + d2 * d1 * (val[1, 1, 1] - val[0, 1, 1])
        g[:, 0] = g0 * res_inv
    return np.where(in_map, dist, -1.0), g, in_map


def distance(V, gs, q, origin, res):
    """GetDistance(Vector3d) on voxel values V: -10000 outside the map, V at Pos2Vox, +10000 off the grid (the max faces)."""
    V = np.asarray(V, np.float64).reshape(gs)
    q = np.asarray(q, np.float64).reshape(-1, 3)
    o = np.asarray(origin, np.float64)
    in_map = np.all((q >= o) & (q <= o + np.asarray(gs) * res), axis=1)
    v = np.floor((q - o) / res).astype(np.int64)
    ok = np.all((v >= 0) & (v < np.asarray(gs)), axis=1)
    vc = np.where(ok[:, None], v, 0)
    return np.where(in_map, np.where(ok, V[vc[:, 0], vc[:, 1], vc[:, 2]], 10000.0), -10000.0)
