"""CPU definition of the topological skeleton of a voxel box (fiesta_skeleton_*, fiesta_b200/csrc/fb_skel.h, DESIGN.md §3.14) on the
arrays export_distance() and export_closest_obstacle() return: traversability, GVD anchors, subfield thinning with a vectorised
simple-point test, the graph of a voxel set with scipy's labelling, and spur pruning.  Also a thinning pass that deletes its voxels
one at a time in a given order, and the building blocks the CPU tests check on their own."""
import itertools

import numpy as np
from scipy import ndimage

from tests.frontierref import label_scipy
from tests.navref import box_slices, traversable, weights

UNDEF = -10000
INF = 10000.0
TRAV, ANCHOR, SKEL = 1, 2, 4

# neighbourhood code bits: e = (dx+1)*9 + (dy+1)*3 + (dz+1), bit 13 the voxel itself
DIRS = list(itertools.product((-1, 0, 1), repeat=3))
CENTER = 1 << 13
FULL = (1 << 27) - 1
FACE_DIRS = [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]


def _mask(pred):
    return sum(1 << e for e, d in enumerate(DIRS) if pred(d))


ZLO, ZHI = _mask(lambda d: d[2] == -1), _mask(lambda d: d[2] == 1)
YLO, YHI = _mask(lambda d: d[1] == -1), _mask(lambda d: d[1] == 1)
XLO, XHI = _mask(lambda d: d[0] == -1), _mask(lambda d: d[0] == 1)
N6 = _mask(lambda d: sum(map(abs, d)) == 1)
N18 = _mask(lambda d: sum(map(abs, d)) <= 2)


def _u(x):
    return np.uint32(x)


def _dil(a, six):
    def sh(a, m, k):
        return ((a & _u(~m & FULL)) << _u(k)) if k > 0 else ((a & _u(~m & FULL)) >> _u(-k))
    if six:
        return a | sh(a, ZHI, 1) | sh(a, ZLO, -1) | sh(a, YHI, 3) | sh(a, YLO, -3) | sh(a, XHI, 9) | sh(a, XLO, -9)
    a = a | sh(a, ZHI, 1) | sh(a, ZLO, -1)
    a = a | sh(a, YHI, 3) | sh(a, YLO, -3)
    return a | sh(a, XHI, 9) | sh(a, XLO, -9)


def _flood(seed, s, six):
    while True:
        n = _dil(seed, six) & s
        if np.array_equal(n, seed):
            return seed
        seed = n


def _lowbit(a):
    return a & (~a + _u(1))


def popcount(a):
    a = np.asarray(a, np.uint32)
    return np.array([bin(int(x)).count("1") for x in a.reshape(-1)], np.int64).reshape(a.shape) if a.size < 64 else \
        np.unpackbits(a.astype("<u4").view(np.uint8).reshape(-1, 4), axis=1).sum(1).reshape(a.shape).astype(np.int64)


def simple(codes):
    """Vectorised simple-point test on 27-bit neighbourhood codes (the centre bit is ignored): T26 = 1 and T6 = 1."""
    c = np.asarray(codes, np.uint32)
    fg = c & _u(FULL & ~CENTER)
    ok = fg != 0
    comp = _flood(_lowbit(fg), fg, False)
    ok &= comp == fg
    bg = ~c & _u(N18 & ~CENTER)
    faces = bg & _u(N6)
    ok &= faces != 0
    comp6 = _flood(_lowbit(faces), bg, True)
    ok &= (faces & ~comp6) == 0
    return ok


def codes_at(P, c):
    """Neighbourhood codes of box-local voxels c (n, 3) from the set padded by one background voxel on every side."""
    code = np.zeros(len(c), np.uint32)
    for e, d in enumerate(DIRS):
        code |= P[c[:, 0] + 1 + d[0], c[:, 1] + 1 + d[1], c[:, 2] + 1 + d[2]].astype(np.uint32) << np.uint32(e)
    return code


def deletable(code, anchor, phase):
    nb = popcount(code & np.uint32(FULL & ~CENTER))
    rule = ~anchor if phase == 1 else nb >= 2
    return rule & simple(code)


def _candidates(X, s):
    o = (s >> 2, (s >> 1) & 1, s & 1)
    c = np.argwhere(X[o[0]::2, o[1]::2, o[2]::2]) * 2 + np.array(o)
    if len(c) == 0:
        return c
    P = np.pad(X, 1)
    interior = np.ones(len(c), bool)
    for d in FACE_DIRS:
        interior &= P[c[:, 0] + 1 + d[0], c[:, 1] + 1 + d[1], c[:, 2] + 1 + d[2]]
    return c[~interior]                                        # an interior voxel is never simple (T6 = 0)


def thin_pass(X, A, phase, s):
    """Pass s of a phase, in place: every voxel of subfield s deletable on X as it stands; returns the count deleted."""
    c = _candidates(X, s)
    if len(c) == 0:
        return 0
    ok = deletable(codes_at(np.pad(X, 1), c), A[tuple(c.T)], phase)
    X[tuple(c[ok].T)] = False
    return int(ok.sum())


def thin_pass_sequential(X, A, phase, s, rng):
    """The same pass deleting one voxel at a time in a random order, each evaluated on X as it stands then."""
    c = _candidates(X, s)
    n = 0
    for i in rng.permutation(len(c)):
        v = c[i]
        P = np.pad(X, 1)
        if deletable(codes_at(P, v[None]), A[tuple(v)][None], phase)[0]:
            X[tuple(v)] = False
            n += 1
    return n


def thin(X0, A, pass_fn=None):
    """Both phases: (X after phase 1, X after phase 2, [iterations of phase 1, of phase 2]); each count includes the iteration
    that deleted nothing."""
    pass_fn = pass_fn or thin_pass
    X = np.array(X0, bool)
    out, iters = [], []
    for phase in (1, 2):
        it = 0
        while True:
            it += 1
            if sum(pass_fn(X, A, phase, s) for s in range(8)) == 0:
                break
        iters.append(it)
        out.append(X.copy())
    return out[0], out[1], iters


def anchors(T, O, defined, lo, max_cos):
    """GVD anchors of the box: T traversable (box-shaped), O closest obstacles (box-shaped, 3 ints), defined o(v)."""
    B = T.shape
    v = np.indices(B).transpose(1, 2, 3, 0).astype(np.int64) + np.asarray(lo, np.int64)
    a = O.astype(np.int64) - v
    ok_v = T & defined
    A = np.zeros(B, bool)
    for d in FACE_DIRS:
        su = tuple(slice(max(0, -d[k]), B[k] - max(0, d[k])) for k in range(3))
        sn = tuple(slice(su[k].start + d[k], su[k].stop + d[k]) for k in range(3))
        diff = np.any(O[su] != O[sn], axis=-1)
        A[su] |= ok_v[su] & ok_v[sn] & diff & anchor_pair(a[su], a[sn], max_cos)
    return A


def anchor_pair(a, b, max_cos):
    """The angle test of two obstacle offsets a = o(v) - v, b = o(u) - u (int64, last axis xyz): exact integer dot products, then
    (double)(a.b) <= max_cos * sqrt((double)(a.a) * (double)(b.b)), each fp64 operation rounded on its own."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    ab = np.sum(a * b, -1).astype(np.float64)
    aa, bb = np.sum(a * a, -1).astype(np.float64), np.sum(b * b, -1).astype(np.float64)
    return ab <= np.float64(max_cos) * np.sqrt(aa * bb)


def _nbrs(S, v):
    B = S.shape
    out = []
    for d in DIRS:
        if d == (0, 0, 0):
            continue
        u = (v[0] + d[0], v[1] + d[1], v[2] + d[2])
        if all(0 <= u[k] < B[k] for k in range(3)) and S[u]:
            out.append(u)
    return out


def graph(S, Dbox=None, lo=(0, 0, 0), res=1.0, origin=(0.0, 0.0, 0.0), walk=True):
    """The graph of voxel set S (box-shaped bool): dict of labels, per-vertex size / rep / centroid / degree / leaf, per-edge uv /
    n_vox / length / min_dist and the edge voxels (grid xyz: box-local + lo), plus deg (box-shaped).  Dbox: export_distance() over
    the box (min_dist reads GetDistance(Vector3i): unknown as +10000)."""
    S = np.asarray(S, bool)
    B = S.shape
    lo = np.asarray(lo, np.int64)
    P = np.pad(S, 1)
    c = np.argwhere(S)
    deg = np.zeros(B, np.int64)
    deg[tuple(c.T)] = popcount(codes_at(P, c) & np.uint32(FULL & ~CENTER)) if len(c) else 0
    V = S & (deg != 2)
    lab, n = ndimage.label(S, structure=np.ones((3, 3, 3), bool))
    has_v = np.zeros(n + 1, bool)
    has_v[lab[V]] = True
    flat = lab.reshape(-1)
    for k in np.nonzero(~has_v[1:])[0] + 1:                    # pure cycles: promote their smallest-index voxel
        V.reshape(-1)[np.flatnonzero(flat == k)[0]] = True
    Cc = S & ~V
    vlab, clab = label_scipy(V), label_scipy(Cc)
    nV, nE = int(vlab.max()) + 1 if V.any() else 0, int(clab.max()) + 1 if Cc.any() else 0
    vidx = np.flatnonzero(vlab.reshape(-1) >= 0)
    vids = vlab.reshape(-1)[vidx]
    vxyz = np.stack(np.unravel_index(vidx, B), -1).astype(np.int64) + lo
    size = np.bincount(vids, minlength=nV).astype(np.int64)
    first = np.full(nV, len(vids), np.int64)
    np.minimum.at(first, vids, np.arange(len(vids)))
    rep = vxyz[first] if nV else np.zeros((0, 3), np.int64)
    ssum = np.zeros((nV, 3), np.int64)
    for k in range(3):
        np.add.at(ssum[:, k], vids, vxyz[:, k])
    centroid = (ssum.astype(np.float64) / np.maximum(size, 1)[:, None].astype(np.float64) + 0.5) * res + np.asarray(origin, np.float64)
    leaf = (size == 1) & (deg.reshape(-1)[vidx[first]] == 1 if nV else np.zeros(0, bool))
    w = weights(res)
    Dg = None if Dbox is None else np.where(np.asarray(Dbox) < 0, INF, np.asarray(Dbox))
    cidx = np.flatnonzero(clab.reshape(-1) >= 0)
    cids = clab.reshape(-1)[cidx]
    order = np.argsort(cids, kind="stable")
    starts = np.searchsorted(cids[order], np.arange(nE + 1))
    PC = np.pad(Cc, 1)
    uv = np.zeros((nE, 2), np.int64)
    nvox = np.zeros(nE, np.int64)
    length, min_dist = np.zeros(nE), np.zeros(nE)
    paths = []
    degree = np.zeros(nV, np.int64)

    def key(a, cv):
        return (int(vlab[a]), int(np.ravel_multi_index(a, B)), int(np.ravel_multi_index(cv, B)))

    for e in range(nE):
        mem = [tuple(int(t) for t in np.unravel_index(i, B)) for i in cidx[order[starts[e]:starts[e + 1]]]]
        ends = [m for m in mem if int(codes_at(PC, np.array([m]))[0] & np.uint32(FULL & ~CENTER)).bit_count() <= 1]
        if len(mem) == 1:
            att = sorted((u for u in _nbrs(S, mem[0]) if V[u]), key=lambda u: np.ravel_multi_index(u, B))
            assert len(att) == 2
            cand = [(key(att[0], mem[0]), att[0], mem[0]), (key(att[1], mem[0]), att[1], mem[0])]
        else:
            assert len(ends) == 2
            cand = []
            for m in ends:
                att = [u for u in _nbrs(S, m) if V[u]]
                assert len(att) == 1
                cand.append((key(att[0], m), att[0], m))
        cand.sort()
        _, a0, c0 = cand[0]
        path = [a0, c0]
        prev, cur = a0, c0
        while True:
            nx = [u for u in _nbrs(S, cur) if u != prev]
            assert len(nx) == 1
            path.append(nx[0])
            if V[nx[0]]:
                break
            prev, cur = cur, nx[0]
        assert len(path) == len(mem) + 2
        uv[e] = (vlab[path[0]], vlab[path[-1]])
        degree[uv[e, 0]] += 1
        degree[uv[e, 1]] += 1
        nvox[e] = len(path)
        if walk:
            L = 0.0
            for p, q in zip(path, path[1:]):
                L = L + w[sum(1 for k in range(3) if p[k] != q[k]) - 1]
            length[e] = L
            if Dg is not None:
                min_dist[e] = min(Dg[p] for p in path)
            paths.append(np.array(path, np.int64) + lo)
    labels = np.full(B, -1, np.int32)
    labels[V] = vlab[V]
    labels[Cc] = -2 - clab[Cc]
    ev = np.concatenate(paths).astype(np.int32) if paths else np.zeros((0, 3), np.int32)
    return dict(labels=labels, V=V, deg=deg, vertices=dict(size=size, rep=rep.astype(np.int32), centroid=centroid,
                                                            degree=degree.astype(np.int32)),
                leaf=leaf, vertex_voxel=vidx[first] if nV else np.zeros(0, np.int64),
                edges=dict(uv=uv.astype(np.int32), n_vox=nvox, length=length, min_dist=min_dist), edge_voxels=ev)


def prune_round(S, min_branch):
    """The voxels one pruning round removes from S (box-shaped bool)."""
    G = graph(S, walk=False)
    rm = np.zeros(S.shape, bool)
    labels, leaf = G["labels"], G["leaf"]
    for e, (u, v) in enumerate(G["edges"]["uv"]):
        count = int(G["edges"]["n_vox"][e]) - 1                 # the leaf voxel counted, the other attachment not
        for a, b in ((u, v), (v, u)):
            if a != b and leaf[a] and not leaf[b] and count < min_branch:
                rm |= labels == -2 - e
                rm.reshape(-1)[G["vertex_voxel"][a]] = True
    if min_branch >= 2:
        deg = G["deg"]
        for c in np.argwhere(S & (deg == 1)):
            (u,) = _nbrs(S, tuple(c))
            if deg[u] >= 3:
                rm[tuple(c)] = True
    return rm


def prune(S, min_branch):
    """(pruned set, rounds, voxels removed); min_branch <= 1: no rounds."""
    S = np.array(S, bool)
    if min_branch <= 1:
        return S, 0, 0
    rounds = removed = 0
    while True:
        rounds += 1
        rm = prune_round(S, min_branch)
        if not rm.any():
            return S, rounds, removed
        S &= ~rm
        removed += int(rm.sum())


def from_records(D_export, closest, grid_size, box, r, unknown_blocks):
    """(X0, closest obstacles, defined) over the box from the map's exports."""
    D = np.asarray(D_export).reshape(grid_size)[box_slices(box)]
    O = np.asarray(closest).reshape(tuple(grid_size) + (3,))[box_slices(box)]
    T = traversable(D, r, unknown_blocks)
    defined = (O[..., 0] != UNDEF) & (D != INF)                # FB_DINF records read +10000 and keep their obstacle
    return T, O, defined, D


def skeleton(D_export, closest, grid_size, box, r, unknown_blocks, max_cos, min_branch, res, origin):
    """Everything fiesta_skeleton_* returns: dict(mask, labels, vertices, edges, edge_voxels, stats)."""
    T, O, defined, D = from_records(D_export, closest, grid_size, box, r, unknown_blocks)
    return skeleton_of(T, O, defined, D, box[0], max_cos, min_branch, res, origin)


def skeleton_of(T, O, defined, D, lo, max_cos, min_branch, res, origin):
    A = anchors(T, O, defined, lo, max_cos)
    _, X2, iters = thin(T, A)
    S, rounds, removed = prune(X2, min_branch)
    G = graph(S, D, lo, res, origin)
    mask = (T * TRAV | A * ANCHOR | S * SKEL).astype(np.uint8)
    stats = dict(box_voxels=int(T.size), traversable=int(T.sum()), anchors=int(A.sum()), iterations=list(iters),
                 prune_rounds=rounds, pruned_voxels=removed, skeleton_voxels=int(S.sum()), vertices=len(G["vertices"]["size"]),
                 edges=len(G["edges"]["uv"]), edge_voxels=len(G["edge_voxels"]))
    return dict(mask=mask, labels=G["labels"], vertices=G["vertices"], edges=G["edges"], edge_voxels=G["edge_voxels"], stats=stats)


def from_obstacles(obst, max_cos):
    """A crafted box: obstacles given as a bool array; X0 = the free voxels (clearance 0), closest obstacles from scipy's EDT indices
    (every o(v) defined when there is an obstacle).  Returns (X0, anchors)."""
    obst = np.asarray(obst, bool)
    T = ~obst
    if not obst.any():
        return T, np.zeros(obst.shape, bool)
    idx = ndimage.distance_transform_edt(~obst, return_distances=False, return_indices=True)
    O = np.moveaxis(idx, 0, -1).astype(np.int64)
    return T, anchors(T, O, np.ones(obst.shape, bool), (0, 0, 0), max_cos)
