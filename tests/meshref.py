"""CPU definition of the surface mesh of a voxel box (fiesta_mesh_*, fiesta_b200/csrc/fb_mesh.h, DESIGN.md §3.15) on the arrays
export_distance() and export_closest_obstacle() return: blocking and distances over the box, active cells and their vertices over
the extended box E = [lo - 1, hi], and one quad per sign-changing grid edge split into two triangles.  Vectorised over cells and
edges; the building blocks (crossing parameter, cell-edge order, quad order, diagonal rule) are exposed for the CPU tests."""
import numpy as np

from tests.navref import box_slices

UNDEF = -10000
INF = 10000.0

# corner k of a cell: offset ((k >> 2) & 1, (k >> 1) & 1, k & 1)
CORNERS = [((k >> 2) & 1, (k >> 1) & 1, k & 1) for k in range(8)]


def _cell_edges():
    """The 12 cell edges in the summation order: (axis, lower corner, upper corner).  x-edges, then y-edges, then z-edges; within an
    axis lexicographic in the other two offsets."""
    out = []
    for a in range(3):
        p, q = [k for k in range(3) if k != a]
        for op in (0, 1):
            for oq in (0, 1):
                o = [0, 0, 0]
                o[p], o[q] = op, oq
                k0 = CORNERS.index(tuple(o))
                o[a] = 1
                out.append((a, k0, CORNERS.index(tuple(o))))
    return out


CELL_EDGES = _cell_edges()


def _quad_offsets():
    """QUAD[a, v_blocks, i] = offset of the i-th cell of the quad around edge (v, v + e_a) from v, in the oriented order."""
    out = np.zeros((3, 2, 4, 3), np.int64)
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        q = [(0, -1, -1), (0, 0, -1), (0, 0, 0), (0, -1, 0)]              # offsets along (a, b, c)
        for vb in (0, 1):
            order = (0, 1, 2, 3) if vb else (0, 3, 2, 1)
            for i, j in enumerate(order):
                out[a, vb, i, a], out[a, vb, i, b], out[a, vb, i, c] = q[j]
    return out


QUAD = _quad_offsets()


def crossing_t(has_u, du, has_w, dw, r):
    """t on an edge from u to w (exactly one blocking): (r - d(u)) / (d(w) - d(u)) when both have a distance, else 0.5."""
    has_u, has_w = np.asarray(has_u, bool), np.asarray(has_w, bool)
    du, dw = np.asarray(du, np.float64), np.asarray(dw, np.float64)
    both = has_u & has_w
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (np.float64(r) - du) / np.where(both, dw - du, 1.0)
    return np.where(both, t, 0.5)


def vertices_of(c, blk, has, d, r, res, origin):
    """Vertex positions of active cells: c (n, 3) lower corners in grid voxels, blk / has (n, 8) bool and d (n, 8) per corner."""
    c = np.asarray(c, np.int64)
    blk, has, d = np.asarray(blk, bool), np.asarray(has, bool), np.asarray(d, np.float64)
    s = np.zeros((len(c), 3))
    n = np.zeros(len(c), np.int64)
    for a, k0, k1 in CELL_EDGES:
        ch = blk[:, k0] != blk[:, k1]
        t = crossing_t(has[:, k0], d[:, k0], has[:, k1], d[:, k1], r)
        for k in range(3):
            u = (c[:, k] + CORNERS[k0][k]).astype(np.float64)
            s[:, k] = np.where(ch, s[:, k] + (u + t if k == a else u), s[:, k])
        n += ch
    m = s / n[:, None].astype(np.float64)
    return (((m + 0.5) * np.float64(res)) + np.asarray(origin, np.float64)).astype(np.float32)


def split02(p0, p1, p2, p3):
    """The diagonal rule on float32 positions (n, 3): |p0 - p2|^2 <= |p1 - p3|^2 in fp64, x, y and z summed in that order."""
    a = np.asarray(p0, np.float32).astype(np.float64) - np.asarray(p2, np.float32).astype(np.float64)
    b = np.asarray(p1, np.float32).astype(np.float64) - np.asarray(p3, np.float32).astype(np.float64)
    return ((a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2]) <= ((b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1]) + b[:, 2] * b[:, 2])


def tris(q, s02):
    """Two triangles per quad from its vertex ids q (n, 4) in oriented order: (n, 2, 3)."""
    q = np.asarray(q)
    A = np.stack([q[:, [0, 1, 2]], q[:, [0, 2, 3]]], 1)
    B = np.stack([q[:, [1, 2, 3]], q[:, [1, 3, 0]]], 1)
    return np.where(np.asarray(s02)[:, None, None], A, B)


def from_records(D_export, closest, grid_size, box, r, unknown_blocks):
    """(blocking, has a distance, distance) over the box from the map's exports."""
    D = np.asarray(D_export).reshape(grid_size)[box_slices(box)]
    O = np.asarray(closest).reshape(tuple(grid_size) + (3,))[box_slices(box)]
    blk = np.where(D < 0, bool(unknown_blocks), D <= r)
    has = (O[..., 0] != UNDEF) & (D != INF)                    # FB_DINF records read +10000 and keep their obstacle
    return blk, has, np.where(has, D, 0.0)


def mesh(D_export, closest, grid_size, box, r, unknown_blocks, res, origin):
    """Everything fiesta_mesh_* returns: dict(vertices (V, 3) float32, triangles (T, 3) int32, stats), and cells (V, 3): the grid
    voxel of each vertex's cell (its lower corner)."""
    blk, has, d = from_records(D_export, closest, grid_size, box, r, unknown_blocks)
    return mesh_of(blk, has, d, box[0], r, res, origin)


def mesh_of(blk, has, d, lo, r, res, origin):
    """The mesh of box-shaped blocking / distance arrays whose first voxel is grid voxel lo."""
    blk = np.asarray(blk, bool)
    B = blk.shape
    # padded by one voxel on every side: padded index = E-local index, so E = [0, B] and positions B + 1 are past E
    P, H, Dp = np.pad(blk, 1), np.pad(np.asarray(has, bool), 1), np.pad(np.asarray(d, np.float64), 1)
    nE = tuple(b + 1 for b in B)

    def corner(A, o):
        return A[o[0]:o[0] + nE[0], o[1]:o[1] + nE[1], o[2]:o[2] + nE[2]]

    cb = np.stack([corner(P, o) for o in CORNERS], -1)
    active = cb.any(-1) & ~cb.all(-1)
    e = np.argwhere(active)                                    # E-index order
    vid = np.full(nE, -1, np.int64)
    vid[tuple(e.T)] = np.arange(len(e))
    sel = tuple(e.T)
    ch = np.stack([corner(H, o)[sel] for o in CORNERS], -1)
    cd = np.stack([corner(Dp, o)[sel] for o in CORNERS], -1)
    V = vertices_of(e + np.asarray(lo) - 1, cb[sel], ch, cd, r, res, origin) if len(e) else np.zeros((0, 3), np.float32)
    # sign-changing edges (v, v + e_a), v in E, in order of (E-index, axis)
    here = P[:nE[0], :nE[1], :nE[2]]
    chg = np.stack([here != P[1:, :nE[1], :nE[2]], here != P[:nE[0], 1:, :nE[2]], here != P[:nE[0], :nE[1], 1:]], -1)
    f = np.argwhere(chg)
    v, a = f[:, :3], f[:, 3]
    vb = here[tuple(v.T)].astype(np.int64)
    cells = v[:, None, :] + QUAD[a, vb]                        # (Q, 4, 3)
    q = vid[cells[..., 0], cells[..., 1], cells[..., 2]]
    assert np.all(q >= 0)
    T = tris(q, split02(V[q[:, 0]], V[q[:, 1]], V[q[:, 2]], V[q[:, 3]])).reshape(-1, 3).astype(np.int32) if len(f) else \
        np.zeros((0, 3), np.int32)
    stats = dict(box_voxels=int(np.prod(B)), blocking=int(blk.sum()), vertices=len(V), quads=len(f), triangles=2 * len(f))
    return dict(vertices=V, triangles=T, stats=stats, cells=e + np.asarray(lo) - 1)
