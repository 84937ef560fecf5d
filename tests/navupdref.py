"""CPU model of the cost-to-go field update (fiesta_nav_update, fiesta_b200/csrc/fb_nav.cu, DESIGN.md §3.11): tight supports,
the kept / withdrawn split, the start state and seed tiles of the re-relaxation, and navref.tile_worklist's tile loop generalised
to start from a given field and tile set.  The result must be navref.field on the new records, bit for bit."""
import itertools

import numpy as np

from tests import navref
from tests.navref import OFFSETS, _tiles_touching, move_mask, weight


def supports(Dold, res):
    """S[k][v]: u = v + OFFSETS[k] is a tight support of v -- the move u -> v was allowed under the old traversability (Dold >= 0),
    Dold(u) is finite and fl(Dold(u) + w) == Dold(v).  Box-shaped boolean arrays, one per move."""
    T = Dold >= 0
    S = np.zeros((26,) + Dold.shape, bool)
    for k, d in enumerate(OFFSETS):
        # move_mask(T, e) lists moves x -> x + e; here the move goes from u = v + d into v, i.e. e = -d with x = u
        e = tuple(-c for c in d)
        su, sv, A = move_mask(T, e)
        du, dv = Dold[su], Dold[sv]
        S[k][sv] = A & (du < np.inf) & (du + weight(d, res) == dv)
    return S


def allowed_into(T):
    """A[k][v]: the move from v + OFFSETS[k] into v is allowed under traversability T."""
    A = np.zeros((26,) + T.shape, bool)
    for k, d in enumerate(OFFSETS):
        su, sv, M = move_mask(T, tuple(-c for c in d))
        A[k][sv] = M
    return A


def shifted(a, d, fill):
    """out[v] = a[v + d], `fill` outside the box."""
    out = np.full_like(a, fill)
    src = tuple(slice(max(0, d[k]), a.shape[k] + min(0, d[k])) for k in range(3))
    dst = tuple(slice(max(0, -d[k]), a.shape[k] + min(0, -d[k])) for k in range(3))
    out[dst] = a[src]
    return out


def withdrawn(Dold, Tnew, res):
    """Step 2-3: kept(v) iff Tnew(v), Dold(v) finite, and Dold(v) == 0 or some tight support is kept through a move still allowed
    under Tnew.  Iterated from all-kept by withdrawals, which reach the unique solution (supports are acyclic)."""
    S = supports(Dold, res) & allowed_into(Tnew)
    cand = Tnew & (Dold > 0) & (Dold < np.inf)
    W = np.zeros(Dold.shape, bool)
    while True:
        kept = Tnew & (Dold >= 0) & (Dold < np.inf) & ~W
        has = np.zeros(Dold.shape, bool)
        for k, d in enumerate(OFFSETS):
            has |= S[k] & shifted(kept, d, False)
        nW = cand & ~has
        if np.array_equal(nW, W):
            return W
        W = nW


def start_state(Dold, Tnew, goals, W, free_neighbours=True):
    """Step 4-5: the start field and the seed tiles.  `goals`: box-local linear indices of the goals placed on Tnew."""
    B = Dold.shape
    tn = tuple((b + 7) // 8 for b in B)
    Told = Dold >= 0
    F = Dold.copy()
    F[Told & ~Tnew] = -1.0
    F[W | (Tnew & ~Told)] = np.inf
    F.reshape(-1)[np.asarray(goals, np.int64).reshape(-1)] = 0.0
    seeds = set()
    for v in np.argwhere(W):
        seeds.add(tuple(int(c) // 8 for c in v))
    for v in np.argwhere(Tnew & ~Told):                     # newly placed goals are among the newly free voxels
        v = tuple(int(c) for c in v)
        seeds |= _tiles_touching(v, tn, own=True) if free_neighbours else {tuple(c // 8 for c in v)}
    return F, seeds


def tile_relax(F, queue, res, rng, fresh_halo):
    """navref.tile_worklist's generations of k_nav_relax, from field F (modified in place) and the tile set `queue`.  Returns
    (field, generations, tile visits)."""
    B = F.shape
    tn = tuple((b + 7) // 8 for b in B)
    moves = []
    for d in OFFSETS:
        span = list(itertools.product(*[range(min(0, c), max(0, c) + 1) for c in d]))
        moves.append((d, weight(d, res), span))
    inner = (slice(1, 9),) * 3
    sh = lambda a, e: a[tuple(slice(1 + e[k], 9 + e[k]) for k in range(3))]
    gens = visits = 0
    queue = set(queue)
    while queue:
        gens += 1
        snap = None if fresh_halo else F.copy()
        nxt = set()
        for t in [tuple(x) for x in rng.permutation(sorted(queue))]:
            visits += 1
            src = np.pad(F if fresh_halo else snap, ((1, 9),) * 3, constant_values=-1.0)
            R = src[tuple(slice(8 * t[k], 8 * t[k] + 10) for k in range(3))].copy()
            trav = R >= 0
            allowed = [(d, w, np.logical_and.reduce([sh(trav, e) for e in span])) for d, w, span in moves]
            orig = R[inner].copy()
            while True:
                cur = R[inner]
                best = cur.copy()
                for d, w, A in allowed:
                    best = np.where(A, np.minimum(best, sh(R, d) + w), best)
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
    return F, gens, visits


def improvable(F, res):
    """Voxels of a field that one relaxation step would lower: the set k_nav_relax's work list must cover at generation 0."""
    T = F >= 0
    out = np.zeros(F.shape, bool)
    for d in OFFSETS:
        su, sv, A = move_mask(T, d)
        out[sv] |= A & (F[su] + weight(d, res) < F[sv])
    return out


def update(Dold, Tnew, goals, res, rng=None, fresh_halo=True, variant=None):
    """The whole update: Dold the old field, Tnew the new traversability of the box, goals box-local linear indices placed on Tnew.
    variant (negative controls): "blocked_only" withdraws nothing but the newly blocked voxels; "no_free_neighbours" seeds only
    a newly free voxel's own tile.  Returns (field, stats) with the statistics fiesta_nav_update reports."""
    rng = np.random.default_rng(0) if rng is None else rng
    Told = Dold >= 0
    W = np.zeros(Dold.shape, bool) if variant == "blocked_only" else withdrawn(Dold, Tnew, res)
    F0, seeds = start_state(Dold, Tnew, goals, W, free_neighbours=variant != "no_free_neighbours")
    tn = tuple((b + 7) // 8 for b in Dold.shape)
    bad = improvable(F0, res)
    outside = [v for v in np.argwhere(bad) if tuple(int(c) // 8 for c in v) not in seeds]
    F, gens, visits = tile_relax(F0.copy(), seeds, res, rng, fresh_halo)
    g = np.asarray(goals, np.int64).reshape(-1)
    stats = dict(became_blocked=int(np.sum(Told & ~Tnew)), became_free=int(np.sum(Tnew & ~Told)), withdrawn=int(W.sum()),
                 goals_new=int(np.sum(~Told.reshape(-1)[g])), seed_tiles=len(seeds), generations=gens, tile_visits=visits,
                 blocked=int(np.sum(F < 0)), reached=int(np.sum((F >= 0) & (F < np.inf))), improvable_outside_seeds=len(outside),
                 tiles=int(np.prod(tn)))
    return F, stats
