"""CPU definition of frontier extraction (fiesta_frontiers_*, fiesta_b200/csrc/fb_frontier.h, DESIGN.md §3.6) on the arrays
export_distance() and export_occupancy() return: the frontier predicate, scipy's 26-connected labelling, numbering by smallest
index, the size filter and the per-cluster statistics; also an independent BFS labelling and an emulation of the device's
tile-local / cross-tile union schedule."""
import collections
import itertools

import numpy as np
from scipy import ndimage

UNKNOWN = -10000.0


def l_occ(p_occ):
    return float(np.log(p_occ / (1.0 - p_occ)))


def box_slices(box):
    lo, hi = box
    return tuple(slice(int(a), int(b) + 1) for a, b in zip(lo, hi))


def frontier_mask(D_export, occ_export, grid_size, box, r, lo_occ):
    """Frontier voxels of the box: observed, occupancy <= l_occ, not blocking at clearance r (GetDistance(Vector3i) <= r blocks;
    +10000 never does), and an unknown face neighbour inside the grid."""
    D = np.asarray(D_export).reshape(grid_size)
    O = np.asarray(occ_export).reshape(grid_size)
    U = D == UNKNOWN
    P = np.pad(U, 1, constant_values=False)                   # outside the grid is not unknown
    gx, gy, gz = grid_size
    nb = np.zeros(grid_size, bool)
    for k in range(3):
        for s in (-1, 1):
            sl = [slice(1, 1 + gx), slice(1, 1 + gy), slice(1, 1 + gz)]
            sl[k] = slice(1 + s, 1 + s + grid_size[k])
            nb |= P[tuple(sl)]
    F = ~U & ~(O > lo_occ) & ~((D >= 0) & (D <= r)) & nb
    return F[box_slices(box)]


def label_scipy(F):
    """26-connected components, numbered 0..C-1 by smallest index (-1 elsewhere)."""
    lab, c = ndimage.label(F, structure=np.ones((3, 3, 3), bool))
    return renumber(lab - 1)


def renumber(lab):
    """Relabel components (any ids >= 0) by their smallest flat index."""
    flat = lab.reshape(-1)
    idx = np.nonzero(flat >= 0)[0]
    out = np.full(flat.shape, -1, np.int64)
    if len(idx):
        ids = flat[idx]
        first = np.full(ids.max() + 1, np.iinfo(np.int64).max)
        np.minimum.at(first, ids, idx)
        used = np.unique(ids)
        order = np.argsort(first[used], kind="stable")
        new = np.full(ids.max() + 1, -1, np.int64)
        new[used[order]] = np.arange(len(used))
        out[idx] = new[ids]
    return out.reshape(lab.shape)


NB26 = [d for d in itertools.product((-1, 0, 1), repeat=3) if d != (0, 0, 0)]


def label_bfs(F):
    """The same components by breadth-first search in index order (independent of scipy)."""
    B = F.shape
    lab = np.full(B, -1, np.int64)
    n = 0
    for v in zip(*np.nonzero(F)):
        if lab[v] >= 0:
            continue
        lab[v] = n
        q = collections.deque([v])
        while q:
            u = q.popleft()
            for d in NB26:
                w = (u[0] + d[0], u[1] + d[1], u[2] + d[2])
                if all(0 <= w[k] < B[k] for k in range(3)) and F[w] and lab[w] < 0:
                    lab[w] = n
                    q.append(w)
        n += 1
    return lab                                                 # index-order discovery: already numbered by smallest index


def label_schedule(F, rng):
    """The device schedule on the CPU: components inside each 8^3 tile (parent = the tile component's smallest index), then the
    unions of frontier neighbours in different tiles, applied in random order and with random argument order, by hooking the
    larger root under the smaller; then every voxel takes its root.  Returns labels numbered by root order."""
    B = F.shape
    N = F.size
    P = np.full(N, -1, np.int64)
    idx = np.arange(N).reshape(B)
    for t in itertools.product(*[range(0, b, 8) for b in B]):
        sl = tuple(slice(t[k], min(t[k] + 8, B[k])) for k in range(3))
        lab, c = ndimage.label(F[sl], structure=np.ones((3, 3, 3), bool))
        ti = idx[sl]
        for j in range(1, c + 1):
            members = ti[lab == j]
            P[members] = members.min()
    pairs = []
    for d in NB26[13:]:
        su = tuple(slice(max(0, -d[k]), B[k] - max(0, d[k])) for k in range(3))
        sv = tuple(slice(su[k].start + d[k], su[k].stop + d[k]) for k in range(3))
        u, v = idx[su], idx[sv]
        cross = np.zeros(u.shape, bool)
        for k in range(3):
            g = np.stack(np.unravel_index(u, B), 0)[k] // 8 != np.stack(np.unravel_index(v, B), 0)[k] // 8
            cross |= g
        m = F[su] & F[sv] & cross
        pairs += list(zip(u[m].tolist(), v[m].tolist()))

    def find(x):
        while P[x] != x:
            x = P[x]
        return x

    for i in rng.permutation(len(pairs)):
        a, b = pairs[i]
        if rng.random() < 0.5:
            a, b = b, a
        while True:
            a, b = find(a), find(b)
            if a == b:
                break
            if a > b:
                a, b = b, a
            old = P[b]
            P[b] = min(P[b], a)
            if old == b:
                break
            b = old
    roots = np.array([find(x) if P[x] >= 0 else -1 for x in range(N)])
    return renumber(roots.reshape(B))


def extract(D_export, occ_export, grid_size, box, r, lo_occ, min_size, res, origin):
    """Everything fiesta_frontiers_* returns: dict(labels (box-shaped int32), size, rep, bbox_lo, bbox_hi, centroid, voxels,
    stats)."""
    F = frontier_mask(D_export, occ_export, grid_size, box, r, lo_occ)
    lab = label_scipy(F)
    B = F.shape
    lo = np.asarray(box[0], np.int64)
    C = int(lab.max()) + 1 if F.any() else 0
    flat = lab.reshape(-1)
    idx = np.nonzero(flat >= 0)[0]
    ids = flat[idx]
    xyz = np.stack(np.unravel_index(idx, B), -1).astype(np.int64) + lo
    size = np.bincount(ids, minlength=C).astype(np.int64)
    keep = size >= min_size
    new = np.full(C, -1, np.int64)
    new[keep] = np.arange(int(keep.sum()))
    K = int(keep.sum())
    out_lab = (np.where(flat >= 0, new[np.maximum(flat, 0)], -1) if C else np.full(flat.shape, -1)).reshape(B).astype(np.int32)
    S = np.zeros((C, 3), np.int64)
    bl = np.full((C, 3), np.iinfo(np.int64).max)
    bh = np.full((C, 3), np.iinfo(np.int64).min)
    rep = np.zeros((C, 3), np.int64)
    for k in range(3):
        np.add.at(S[:, k], ids, xyz[:, k])
        np.minimum.at(bl[:, k], ids, xyz[:, k])
        np.maximum.at(bh[:, k], ids, xyz[:, k])
    first = np.full(C, len(ids), np.int64)
    np.minimum.at(first, ids, np.arange(len(ids)))             # first occurrence in index order
    if C:
        rep = xyz[first]
    centroid = (S.astype(np.float64) / size[:, None].astype(np.float64) + 0.5) * res + np.asarray(origin, np.float64)
    kept_ids = new[ids]
    m = kept_ids >= 0
    order = np.argsort(kept_ids[m], kind="stable")
    voxels = xyz[m][order].astype(np.int32)
    stats = dict(box_voxels=int(F.size), frontier_voxels=int(F.sum()), clusters=C, kept_clusters=K, kept_voxels=int(m.sum()))
    return dict(labels=out_lab, size=size[keep], rep=rep[keep].astype(np.int32), bbox_lo=bl[keep].astype(np.int32),
                bbox_hi=bh[keep].astype(np.int32), centroid=centroid[keep], voxels=voxels, stats=stats)
