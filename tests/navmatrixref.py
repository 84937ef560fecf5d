"""CPU definition of the cost matrix (fiesta_nav_matrix, fiesta_b200/csrc/fb_nav.h, DESIGN.md §3.9), built on tests/navref.py:
scipy's Dijkstra from every source at once, read at the targets, with the status and NaN rules; and an emulation of the device
schedule -- many sources' tile work lists in one list, each source retired once its targets are provably final."""
import itertools

import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

from tests import navref

PASS_CHANNELS = 32


def graph(T, res):
    """The 26-connected move graph of a box (undirected: each symmetric pair once), as navref.field builds it."""
    B, N = T.shape, T.size
    idx = np.arange(N).reshape(B)
    rows, cols, vals = [], [], []
    for d in navref.OFFSETS[13:]:
        su, sv, A = navref.move_mask(T, d)
        rows.append(idx[su][A]); cols.append(idx[sv][A])
        vals.append(np.full(int(A.sum()), navref.weight(d, res)))
    return csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(N, N))


def status(T, box, p, origin, res, min_range, max_range):
    """Status of positions p (n, 3): 0 traversable box voxel, 1 blocked box voxel, 2 NaN / outside the map / outside the box; and
    the box-local linear index (-1 unless status 0)."""
    v, ok = navref.locate(p, origin, res, box, min_range, max_range)
    st = np.full(len(v), 2, np.int32)
    idx = np.full(len(v), -1, np.int64)
    if len(v):
        trav = ok & T[tuple(v.T)]
        st[ok & ~trav] = 1
        st[trav] = 0
        idx[trav] = np.ravel_multi_index(tuple(v[trav].T), T.shape)
    return st, idx


def passes(n_sources_placed, n_targets_placed, box_voxels):
    """Passes of the device: C = min(32, sources, max(1, 2^32 // (8 * box voxels))) sources resident together."""
    if n_sources_placed == 0 or n_targets_placed == 0:
        return 0
    c = min(PASS_CHANNELS, n_sources_placed, max(1, (1 << 32) // (8 * box_voxels)))
    return -(-n_sources_placed // c)


def matrix(D_export, grid_size, box, sources, targets, r, unknown_blocks, origin, res, min_range, max_range):
    """-> (cost (n_src, n_tgt), src_status, tgt_status, stats {sources_placed, targets_placed, passes}) as fiesta_nav_matrix."""
    T = navref.traversable(D_export.reshape(grid_size)[navref.box_slices(box)], r, unknown_blocks)
    ss, si = status(T, box, sources, origin, res, min_range, max_range)
    ts, ti = status(T, box, targets, origin, res, min_range, max_range)
    cost = np.full((len(ss), len(ts)), np.nan)
    rows, cols = np.nonzero(ss == 0)[0], np.nonzero(ts == 0)[0]
    if len(rows) and len(cols):
        u, inv = np.unique(si[rows], return_inverse=True)
        G = graph(T, res)
        at = np.empty((len(u), len(cols)))
        for k in range(0, len(u), 8):                       # 8 sources' full distance arrays at a time
            at[k:k + 8] = dijkstra(G, directed=False, indices=u[k:k + 8])[:, ti[cols]]
        cost[np.ix_(rows, cols)] = at[inv]
    stats = {"sources_placed": int(len(rows)), "targets_placed": int(len(cols)), "passes": passes(len(rows), len(cols), T.size)}
    return cost, ss, ts, stats


def channel_worklist(T, sources, targets, res, rng, fresh_halo, retire=True):
    """The schedule of k_navm_relax emulated on the CPU for one pass.  sources / targets: box-local linear indices of status-0
    points.  Every channel (source) starts at +inf with 0 on its voxel and the tiles k_nav_goals would queue; each generation relaxes
    the queued (channel, tile) items in random order as navref.tile_worklist does (halo from the current field or from the field as
    the generation began), with moves from the box's move masks.  With `retire`, at the start of generation g a channel whose
    targets all read <= m_c(g - 1), the least value it wrote in generation g - 1 (placement: 0), is retired and its items are
    dropped.  Returns (fields (n_src, *B), generations, retired_early: channels retired with items still queued)."""
    B = T.shape
    tn = tuple((b + 7) // 8 for b in B)
    P = tuple(8 * t + 2 for t in tn)                           # padded: 1 voxel before, the rest after
    AL = np.zeros((27,) + P, bool)
    for k, d in enumerate(itertools.product((-1, 0, 1), repeat=3)):
        if d == (0, 0, 0):
            continue
        su, _, A = navref.move_mask(T, d)
        AL[k][tuple(slice(s.start + 1, s.stop + 1) for s in su)] = A
    W = [navref.weight(d, res) if any(d) else 0.0 for d in itertools.product((-1, 0, 1), repeat=3)]
    dirs = list(itertools.product((-1, 0, 1), repeat=3))
    n = len(sources)
    F = np.full((n,) + P, np.inf)
    targets = np.asarray(targets, np.int64)
    tv = [np.unravel_index(int(t), B) for t in targets]
    queue = set()
    for c, s in enumerate(sources):
        v = np.unravel_index(int(s), B)
        F[(c,) + tuple(x + 1 for x in v)] = 0.0
        queue |= {(c,) + t for t in navref._tiles_touching(v, tn, own=True)}
    mprev = np.zeros(n)                                        # m_c(-1): placement writes 0
    retired = np.zeros(n, bool)
    gens = early = 0
    inner = lambda t: tuple(slice(8 * t[k] + 1, 8 * t[k] + 9) for k in range(3))
    while queue:
        if retire:
            for c in range(n):
                if not retired[c] and all(F[(c,) + tuple(x + 1 for x in v)] <= mprev[c] for v in tv):
                    retired[c] = True
                    early += any(item[0] == c for item in queue)
            queue = {item for item in queue if not retired[item[0]]}
            if not queue:
                break
        gens += 1
        snap = None if fresh_halo else F.copy()
        mcur = np.full(n, np.inf)
        nxt = set()
        for item in [tuple(int(x) for x in it) for it in rng.permutation(sorted(queue))]:
            c, t = item[0], item[1:]
            src = F[c] if fresh_halo else snap[c]
            R = src[tuple(slice(8 * t[k], 8 * t[k] + 10) for k in range(3))].copy()
            A = AL[(slice(None),) + inner(t)]
            orig = R[1:9, 1:9, 1:9].copy()                  # the tile's own voxels: only this visit writes them
            while True:
                cur = R[1:9, 1:9, 1:9]
                best = cur.copy()
                for k, d in enumerate(dirs):
                    if k == 13:
                        continue
                    sh = R[tuple(slice(1 + d[j], 9 + d[j]) for j in range(3))]
                    best = np.where(A[k], np.minimum(best, sh + W[k]), best)
                if not np.any(best < cur):
                    break
                R[1:9, 1:9, 1:9] = best
            new = R[1:9, 1:9, 1:9]
            imp = new < orig
            if not imp.any():
                continue
            view = F[c][inner(t)]
            view[imp] = new[imp]
            mcur[c] = min(mcur[c], float(new[imp].min()))
            for v in np.argwhere(imp):
                g = tuple(int(v[k]) + 8 * t[k] for k in range(3))
                nxt |= {(c,) + tt for tt in navref._tiles_touching(g, tn, own=False)}
        queue = nxt
        mprev = mcur
    out = F[(slice(None),) + tuple(slice(1, 1 + b) for b in B)]
    return out, gens, early
