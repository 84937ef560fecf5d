"""Grid shapes at the library's limits and the helpers tests/test_gpu_geometry.py and tests/test_geometry_models.py share.

The resolution is dyadic so that ceil(size / res) is exact and every voxel centre is exactly representable."""
import numpy as np

RES = 0.25
ORIGIN = (-1.0, -0.75, 0.5)

SHAPES = [
    (1, 1, 1), (5, 1, 1), (1, 5, 1), (1, 1, 5),                         # degenerate
    (37, 1, 29), (9, 1, 4),                                              # gy == 1
    (2, 2, 2), (3, 3, 3), (2, 17, 3), (3, 2, 19),                        # below the +-2 reach, one partial tile
    (13, 11, 1), (13, 11, 2), (13, 11, 3), (13, 11, 5), (13, 11, 6), (13, 11, 7), (13, 11, 9), (13, 11, 30),   # Pz != Gz
    (13, 9, 12), (17, 3, 28),                                            # Gz == Pz, off the tile lattice
    (2046, 3, 2), (2046, 2, 5), (2, 1024, 3), (3, 2, 1024), (2046, 1024, 1), (1, 1024, 1024),             # maximal extents
]


def logit(p):
    return float(np.log(p / (1.0 - p)))


def size_of(gs):
    return tuple(g * RES for g in gs)


def shape_id(gs):
    return "x".join(str(g) for g in gs)


def special_voxels(gs):
    """Every corner, edge midpoint, face centre and the centre: {0, mid, max} on each axis."""
    ax = [sorted({0, g // 2, g - 1}) for g in gs]
    return np.array([(x, y, z) for x in ax[0] for y in ax[1] for z in ax[2]], np.int32)


def random_voxels(rng, gs, n):
    return np.stack([rng.integers(0, g, n) for g in gs], -1).astype(np.int32)


def trilinear(D_export, gs, q, origin=ORIGIN, res=RES):
    """GetDistWithGradTrilinear (ESDFMap.cpp:480-537) on an exported distance array, in the reference's operation order:
    (dist (n,), grad (n, 3), in_map (n,)).  GetDistance(Vector3i) reads never-observed voxels as +10000, and so does the
    library for the voxels of the 2x2x2 stencil outside the grid; dist is -1 where PosInMap fails (grad is then not defined)."""
    D = np.where(np.asarray(D_export) < 0, 10000.0, np.asarray(D_export)).reshape(gs)
    q = np.asarray(q, np.float64).reshape(-1, 3)
    o = np.asarray(origin, np.float64)
    in_map = np.all((q >= o) & (q <= o + np.asarray(gs) * res), axis=1)              # PosInMap, both faces inclusive
    res_inv = 1.0 / res
    idx = np.floor(((q - 0.5 * res) - o) / res).astype(np.int64)
    diff = (q - ((idx + 0.5) * res + o)) * res_inv
    val = {}
    for c in [(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)]:
        v = idx + np.array(c)
        ok = np.all((v >= 0) & (v < np.asarray(gs)), axis=1)
        vc = np.where(ok[:, None], v, 0)
        val[c] = np.where(ok, D[vc[:, 0], vc[:, 1], vc[:, 2]], 10000.0)
    d0, d1, d2 = diff[:, 0], diff[:, 1], diff[:, 2]
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
