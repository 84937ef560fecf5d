"""CPU definition of safe flight corridors (fiesta_inflate_boxes / fiesta_corridors, fiesta_b200/csrc/fb_corridor.h, DESIGN.md §3.8),
restated on the traversable mask of navref over the array export_distance() returns: the face-by-face inflation, the chain along a
path, and the statistics, output for output."""
import numpy as np

from tests import navref

# faces in rule order: (axis, up) for -x, +x, -y, +y, -z, +z
ORDER = ((0, False), (0, True), (1, False), (1, True), (2, False), (2, True))


class Limit:
    """The limit box [lo, hi] (inclusive grid voxels) and its traversable mask at clearance r."""

    def __init__(self, D_export, grid_size, box, r, unknown_blocks):
        self.lo, self.hi = np.asarray(box[0], np.int64), np.asarray(box[1], np.int64)
        self.T = navref.traversable(np.asarray(D_export).reshape(grid_size)[navref.box_slices(box)], r, unknown_blocks)
        self.volume = int(self.T.size)

    def free(self, lo, hi):
        """Every voxel of the box [lo, hi] (inside the limit box) is traversable."""
        return bool(self.T[tuple(slice(int(lo[k] - self.lo[k]), int(hi[k] - self.lo[k]) + 1) for k in range(3))].all())

    def inside(self, lo, hi):
        return all(self.lo[k] <= lo[k] <= hi[k] <= self.hi[k] for k in range(3))


def inflate(L, max_steps, lo, hi, order=ORDER):
    """Inflate the seed [lo, hi] -> (lo, hi, layers tested, layers grown)."""
    lo, hi = [int(x) for x in lo], [int(x) for x in hi]
    stop_lo = [max(int(L.lo[k]), lo[k] - int(max_steps[k])) for k in range(3)]
    stop_hi = [min(int(L.hi[k]), hi[k] + int(max_steps[k])) for k in range(3)]
    active = [True] * 6
    tested = grown = 0
    while any(active):
        for f, (a, up) in enumerate(order):
            if not active[f]:
                continue
            if (hi[a] >= stop_hi[a]) if up else (lo[a] <= stop_lo[a]):
                active[f] = False
                continue
            llo, lhi = list(lo), list(hi)
            llo[a] = lhi[a] = hi[a] + 1 if up else lo[a] - 1
            tested += 1
            if L.free(llo, lhi):
                if up:
                    hi[a] += 1
                else:
                    lo[a] -= 1
                grown += 1
            else:
                active[f] = False
    return lo, hi, tested, grown


def chain(L, P, max_steps):
    """The corridor of one path P (n, 3) -> (status, [(lo, hi, seed index)], blocked_at, tested, grown)."""
    P = np.asarray(P, np.int64).reshape(-1, 3)
    n = len(P)
    if n == 0:
        return 0, [], -1, 0, 0
    if np.any((P < L.lo) | (P > L.hi)):
        return 2, [], -1, 0, 0
    boxes, tested, grown = [], 0, 0
    lo, hi, j = P[0].tolist(), P[0].tolist(), 0
    while True:
        if not L.free(lo, hi):
            return 1, boxes, j, tested, grown
        lo, hi, t, g = inflate(L, max_steps, lo, hi)
        tested, grown = tested + t, grown + g
        boxes.append((lo, hi, j))
        out = np.nonzero(np.any((P[j + 1:] < lo) | (P[j + 1:] > hi), axis=1))[0]
        if not len(out):
            return 0, boxes, -1, tested, grown
        i = j + 1 + int(out[0])
        lo, hi, j = np.minimum(P[i - 1], P[i]).tolist(), np.maximum(P[i - 1], P[i]).tolist(), i


def stats(boxes, tested, grown, volume):
    return dict(boxes=boxes, layers_tested=tested, layers_grown=grown, mask_voxels=volume)


def inflate_boxes(L, seed_lo, seed_hi, max_steps):
    """fiesta_inflate_boxes -> (status (n,), lo (n, 3), hi (n, 3), stats)."""
    seed_lo, seed_hi = np.asarray(seed_lo, np.int64).reshape(-1, 3), np.asarray(seed_hi, np.int64).reshape(-1, 3)
    n = len(seed_lo)
    status = np.zeros(n, np.int32)
    lo, hi = np.full((n, 3), -1, np.int32), np.full((n, 3), -1, np.int32)
    tested = grown = 0
    for i in range(n):
        if not L.inside(seed_lo[i], seed_hi[i]):
            status[i] = 2
        elif not L.free(seed_lo[i], seed_hi[i]):
            status[i] = 1
        else:
            a, b, t, g = inflate(L, max_steps, seed_lo[i], seed_hi[i])
            lo[i], hi[i] = a, b
            tested, grown = tested + t, grown + g
    return status, lo, hi, stats(int(np.sum(status == 0)), tested, grown, L.volume if n else 0)


def corridors(L, paths, max_steps):
    """fiesta_corridors in the form ESDFMap.Corridors returns -> (status, n_boxes, blocked_at, [(lo, hi, first)], stats)."""
    n = len(paths)
    status, nb, bl = np.zeros(n, np.int32), np.zeros(n, np.int32), np.full(n, -1, np.int32)
    out, tested, grown = [], 0, 0
    for p, P in enumerate(paths):
        s, boxes, b, t, g = chain(L, P, max_steps)
        status[p], nb[p], bl[p] = s, len(boxes), b
        tested, grown = tested + t, grown + g
        out.append((np.array([x[0] for x in boxes], np.int32).reshape(-1, 3), np.array([x[1] for x in boxes], np.int32).reshape(-1, 3),
                    np.array([x[2] for x in boxes], np.int32)))
    total = sum(len(np.asarray(P).reshape(-1, 3)) for P in paths)
    return status, nb, bl, out, stats(int(nb.sum()), tested, grown, L.volume if total else 0)


def maximal(L, max_steps, seed_lo, seed_hi, lo, hi):
    """Every face of [lo, hi] sits on L, or max_steps beyond the seed's face, or its next layer holds a non-traversable voxel."""
    for a, up in ORDER:
        if up and (hi[a] >= min(L.hi[a], seed_hi[a] + max_steps[a])):
            continue
        if not up and (lo[a] <= max(L.lo[a], seed_lo[a] - max_steps[a])):
            continue
        llo, lhi = list(lo), list(hi)
        llo[a] = lhi[a] = hi[a] + 1 if up else lo[a] - 1
        if L.free(llo, lhi):
            return False
    return True
