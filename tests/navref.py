"""CPU definition of the cost-to-go field (fiesta_nav_*, fiesta_b200/csrc/fb_nav.h, DESIGN.md §3.5): the move graph of a voxel box
built from the array export_distance() returns, scipy's Dijkstra over it, a Gauss-Seidel sweep that reaches the same fixpoint in
another order, and the path rule."""
import itertools

import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

# the 26 moves in path order: (dx, dy, dz) lexicographic, dx slowest, -1 first
OFFSETS = [d for d in itertools.product((-1, 0, 1), repeat=3) if d != (0, 0, 0)]


def weights(res):
    """w[k - 1] for a move with k non-zero components: res * sqrt(k), as the library computes it."""
    return res * np.sqrt(np.array([1.0, 2.0, 3.0]))


def weight(d, res):
    return weights(res)[sum(1 for c in d if c) - 1]


def traversable(Dbox, r, unknown_blocks):
    """Not blocking in the sense of segment clearance: GetDistance(Vector3i) > r; never-observed voxels (-10000) block only with
    the unknown flag; +10000 (unreached) never blocks."""
    return np.where(Dbox < 0, not unknown_blocks, Dbox > r)


def box_slices(box):
    lo, hi = box
    return tuple(slice(int(a), int(b) + 1) for a, b in zip(lo, hi))


def move_mask(T, d):
    """Moves u -> u + d inside the box: (slices of u, slices of u + d, allowed) where allowed[u] = every voxel of the box spanned
    by u and u + d is traversable."""
    B = T.shape
    su = tuple(slice(max(0, -d[k]), B[k] - max(0, d[k])) for k in range(3))
    sv = tuple(slice(su[k].start + d[k], su[k].stop + d[k]) for k in range(3))
    A = np.ones([s.stop - s.start for s in su], bool)
    for e in itertools.product(*[range(min(0, c), max(0, c) + 1) for c in d]):
        A &= T[tuple(slice(su[k].start + e[k], su[k].stop + e[k]) for k in range(3))]
    return su, sv, A


def goal_indices(T, box, goals_vox):
    """Box-local linear indices of the goals that lie in the box on a traversable voxel (duplicates removed)."""
    lo = np.asarray(box[0])
    g = np.asarray(goals_vox, np.int64).reshape(-1, 3) - lo
    ok = np.all((g >= 0) & (g < np.asarray(T.shape)), axis=1)
    g = g[ok]
    g = g[T[tuple(g.T)]]
    return np.unique(np.ravel_multi_index(tuple(g.T), T.shape)) if len(g) else np.zeros(0, np.int64)


def field(D_export, grid_size, box, goals_vox, r, unknown_blocks, res):
    """The field of the box: Dijkstra (min_only) over the 26-connected move graph; -1 on blocked voxels, +inf where unreachable."""
    T = traversable(D_export.reshape(grid_size)[box_slices(box)], r, unknown_blocks)
    B, N = T.shape, T.size
    idx = np.arange(N).reshape(B)
    rows, cols, vals = [], [], []
    for d in OFFSETS[13:]:                                  # one direction of each symmetric pair
        su, sv, A = move_mask(T, d)
        rows.append(idx[su][A]); cols.append(idx[sv][A])
        vals.append(np.full(int(A.sum()), weight(d, res)))
    goals = goal_indices(T, box, goals_vox)
    out = np.full(N, np.inf)
    if len(goals):
        g = csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(N, N))
        out = dijkstra(g, directed=False, indices=goals, min_only=True)
    return np.where(T, out.reshape(B), -1.0)


def sweep(T, goals, res, rng):
    """The same least fixpoint by Gauss-Seidel: relax whole directions in random orders until nothing improves."""
    F = np.where(T, np.inf, -1.0)
    F.reshape(-1)[goals] = 0.0
    masks = [(d, weight(d, res)) + move_mask(T, d) for d in OFFSETS]
    while True:
        changed = False
        for i in rng.permutation(len(masks)):
            d, w, su, sv, A = masks[i]
            tgt = F[sv]
            new = np.where(A, np.minimum(tgt, F[su] + w), tgt)
            if np.any(new < tgt):
                F[sv] = new
                changed = True
        if not changed:
            return F


def _tiles_touching(v, tn, own):
    """Tiles queued for a decreased box voxel v, by the rule of fb_nav.cu: on each axis the voxel's tile, plus the tile across a
    tile face the voxel lies on; tiles outside the tile grid are skipped, and the voxel's own tile only when `own`."""
    span = [range(-1 if v[k] % 8 == 0 else 0, (1 if v[k] % 8 == 7 else 0) + 1) for k in range(3)]
    out = set()
    for o in itertools.product(*span):
        t = tuple(v[k] // 8 + o[k] for k in range(3))
        if (own or any(o)) and all(0 <= t[k] < tn[k] for k in range(3)):
            out.add(t)
    return out


def tile_worklist(T, goals, res, rng, fresh_halo):
    """The device solver's schedule emulated on the CPU: goals placed and their tiles queued as k_nav_goals does, then generations
    of k_nav_relax -- each queued 8^3 tile, in random order, stages itself and a 1-voxel halo (outside the box: blocked), relaxes
    to a local fixpoint, writes back the voxels that improved and queues the tiles across the faces of improved boundary voxels.
    The halo comes from the current field (`fresh_halo`) or from the field as it was when the generation began, the two extremes
    of what a tile can read while other tiles run.  Returns (field, generations)."""
    B = T.shape
    tn = tuple((b + 7) // 8 for b in B)
    F = np.where(T, np.inf, -1.0)
    queue = set()
    for g in np.asarray(goals, np.int64).reshape(-1):
        v = np.unravel_index(int(g), B)
        F[v] = 0.0
        queue |= _tiles_touching(v, tn, own=True)
    moves = []
    for d in OFFSETS:
        span = list(itertools.product(*[range(min(0, c), max(0, c) + 1) for c in d]))
        moves.append((d, weight(d, res), span))
    inner = (slice(1, 9),) * 3
    shifted = lambda a, e: a[tuple(slice(1 + e[k], 9 + e[k]) for k in range(3))]
    gens = 0
    while queue:
        gens += 1
        snap = None if fresh_halo else F.copy()
        nxt = set()
        for t in [tuple(x) for x in rng.permutation(sorted(queue))]:
            src = np.pad(F if fresh_halo else snap, ((1, 9),) * 3, constant_values=-1.0)
            R = src[tuple(slice(8 * t[k], 8 * t[k] + 10) for k in range(3))].copy()
            trav = R >= 0
            allowed = [(d, w, np.logical_and.reduce([shifted(trav, e) for e in span])) for d, w, span in moves]
            orig = R[inner].copy()
            while True:
                cur = R[inner]
                best = cur.copy()
                for d, w, A in allowed:
                    best = np.where(A, np.minimum(best, shifted(R, d) + w), best)
                if not np.any(best < cur):
                    break
                R[inner] = best
            lo = tuple(8 * t[k] for k in range(3))
            n = tuple(min(8, B[k] - lo[k]) for k in range(3))
            new = R[inner][:n[0], :n[1], :n[2]]
            imp = new < orig[:n[0], :n[1], :n[2]]
            F[lo[0]:lo[0] + n[0], lo[1]:lo[1] + n[1], lo[2]:lo[2] + n[2]][imp] = new[imp]
            for v in np.argwhere(imp):
                nxt |= _tiles_touching(tuple(int(v[k]) + lo[k] for k in range(3)), tn, own=False)
        queue = nxt
    return F, gens


def locate(p, origin, res, box, min_range=None, max_range=None):
    """Box-local voxels of positions p (n, 3) and whether each is usable: no NaN, voxel (Pos2Vox) inside the box, and -- when the
    map range is given (path starts) -- PosInMap."""
    p = np.asarray(p, np.float64).reshape(-1, 3)
    f = np.floor((p - np.asarray(origin)) / res)
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    ok = np.all((f >= lo) & (f <= hi), axis=1)              # NaN compares false
    if min_range is not None:
        ok &= np.all(p >= np.asarray(min_range), axis=1) & np.all(p <= np.asarray(max_range), axis=1)
    v = np.where(ok[:, None], f - lo, 0).astype(np.int64)
    return v, ok


def paths(F, box, res, starts_local, usable, max_len):
    """The path rule for many starts at once (box-local start voxels; `usable` False -> status 2).  Returns (status, len, cost,
    vox (n, max_len, 3) grid voxels, -1 past len) as fiesta_nav_paths does."""
    B = np.asarray(F.shape)
    w = weights(res)
    T = F >= 0
    AL = np.zeros((26,) + F.shape, bool)
    for k, d in enumerate(OFFSETS):
        su, _, A = move_mask(T, d)
        AL[k][su] = A
    dirs = np.array(OFFSETS)
    wk = np.array([w[int(np.count_nonzero(d)) - 1] for d in OFFSETS])
    n = len(starts_local)
    status = np.full(n, 2, np.int32)
    length = np.zeros(n, np.int32)
    cost = np.full(n, np.nan)
    vox = np.full((n, max_len, 3), -1, np.int32)
    v = np.asarray(starts_local, np.int64).reshape(-1, 3).copy()
    d0 = np.where(usable, F[tuple(np.where(usable[:, None], v, 0).T)], -1.0)
    status[usable & (d0 == np.inf)] = 1
    cost[usable & (d0 >= 0)] = d0[usable & (d0 >= 0)]
    active = np.nonzero(usable & (d0 >= 0) & (d0 < np.inf))[0]
    lo = np.asarray(box[0])
    for step in range(max_len + 1):
        if not len(active):
            break
        if step == max_len:
            status[active] = 3
            break
        va = v[active]
        vox[active, step] = va + lo
        length[active] = step + 1
        fv = F[tuple(va.T)]
        goal = fv == 0
        status[active[goal]] = 0
        active, va, fv = active[~goal], va[~goal], fv[~goal]
        choose = np.full(len(active), -1)
        for k in range(26):
            u = np.clip(va + dirs[k], 0, B - 1)
            hit = (choose < 0) & AL[k][tuple(va.T)] & (F[tuple(u.T)] + wk[k] == fv)
            choose[hit] = k
        stuck = choose < 0                                  # no predecessor: only on a field that is not the fixpoint
        status[active[stuck]] = 3
        active, va, choose = active[~stuck], va[~stuck], choose[~stuck]
        v[active] = va + dirs[choose]
    return status, length, cost, vox


def fold(F, box, res, path):
    """Fold the weights from the goal back along a path (grid voxels): fl(...fl(fl(0 + w_last) + ...) ...)."""
    acc = 0.0
    for a, b in zip(path[::-1][:-1], path[::-1][1:]):
        acc = acc + float(weight(tuple(int(c) for c in np.asarray(a) - np.asarray(b)), res))
    return acc
