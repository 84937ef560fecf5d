"""Reference definition of the segment clearance query (fiesta_check_segments, fiesta_b200/csrc/fb_segment.h), written from the
definition alone with exact rationals, for the CPU traversal test and the GPU tests.

A segment a-b (metres) is mapped to voxel units as Pos2Vox does, u = (p - origin) / res in fp64, and truncated to the lattice
q = floor(u * 2^20).  The voxels walked are V = {floor(p(t)) : t in [0,1]}, p(t) = qa + t (qb - qa), in t order.  floor(p(t)) is
constant between consecutive plane-crossing parameters, so sampling p at every crossing parameter and at the midpoint of every
interval between them lists V in order; a voxel first seen at a crossing parameter t, or just after it, is entered at t.
"""
import math
from fractions import Fraction

import numpy as np

Q = 1 << 20
UNDEFINED, INFINITY = -10000.0, 10000.0


def lattice(p, origin, res):
    return [math.floor((float(p[k]) - float(origin[k])) / float(res) * Q) for k in range(3)]


def in_map(p, lo, hi):
    return all(lo[k] <= p[k] <= hi[k] for k in range(3))      # NaN compares False: outside


def walk(qa, qb):
    """[(voxel, entry parameter as a Fraction)] of V in t order."""
    d = [b - a for a, b in zip(qa, qb)]
    times = {Fraction(0), Fraction(1)}
    for k in range(3):
        if d[k]:
            for m in range(min(qa[k], qb[k]) // Q, max(qa[k], qb[k]) // Q + 1):
                t = Fraction(m * Q - qa[k], d[k])
                if 0 <= t <= 1:
                    times.add(t)
    times = sorted(times)
    out = []

    def sample(s, t):
        v = tuple((qa[k] * s.denominator + s.numerator * d[k]) // (Q * s.denominator) for k in range(3))
        if not out or out[-1][0] != v:
            out.append((v, t))

    for i, t in enumerate(times):
        sample(t, t)
        if i + 1 < len(times):
            sample((t + times[i + 1]) / 2, t)
    return out


def record_distance(c, x, y, z, res):
    """distance_buffer_ of a packed record: -10000 never observed, +10000 unreached or FB_DINF, else |voxel - obstacle| * res."""
    dinf = c & 0x80000000
    c &= 0x7fffffff
    if c == 0:
        return UNDEFINED
    if c == 1 or dinf:
        return INFINITY
    ox, oy, oz = (c >> 20) - 1, (c >> 10) & 1023, c & 1023
    dx, dy, dz = float(ox - x), float(oy - y), float(oz - z)
    return math.sqrt((dx * dx + dy * dy) + dz * dz) * res


def segment_walk(ab, origin, res, lo, hi):
    """walk() of segment ab in metres, None when an endpoint is outside the map."""
    a, b = ab[:3], ab[3:]
    if not (in_map(a, lo, hi) and in_map(b, lo, hi)):
        return None
    return walk(lattice(a, origin, res), lattice(b, origin, res))


def check(ab, origin, res, lo, hi, dist, r, unknown_blocks):
    """(status, hit_idx, hit_t, min_dist) of one segment; dist: (gx, gy, gz) array of distance_buffer_ values
    (fiesta_export_distance: -10000 never observed)."""
    return apply(segment_walk(ab, origin, res, lo, hi), dist, r, unknown_blocks)


def apply(walked, dist, r, unknown_blocks):
    """The blocking rule over a segment_walk() result."""
    if walked is None:
        return 2, -1, math.nan, UNDEFINED
    gx, gy, gz = dist.shape
    mind = math.inf
    for (x, y, z), t in walked:
        D = float(dist[x, y, z]) if (0 <= x < gx and 0 <= y < gy and 0 <= z < gz) else INFINITY
        g = INFINITY if D < 0 else D                              # GetDistance(Vector3i)
        mind = min(mind, g)
        if g <= r or (unknown_blocks and D == UNDEFINED):
            return 1, (x * gy + y) * gz + z, float(t), mind
    return 0, -1, math.nan, mind


def same(got, want):
    """Bitwise equality of (status, hit_idx, hit_t, min_dist), NaN == NaN."""
    st, ix, t, md = got
    return int(st) == want[0] and int(ix) == want[1] and (float(t) == want[2] or (math.isnan(t) and math.isnan(want[2]))) \
        and float(md) == want[3]


def adversarial_voxel_units(G, rng):
    """Segments in voxel units: axis-parallel, in a face plane, through exact edges and corners in every sign combination, starting
    on a plane heading down, zero length, ending on the upper faces, and corner to corner."""
    G = np.asarray(G, float)
    c = np.floor(G / 2)
    out = []
    for k in range(3):
        for sgn in (1, -1):
            e = np.zeros(3); e[k] = sgn
            a = c + np.array([0.25, 0.5, 0.75])
            out.append((a, a + e * min(5.5, c[k] - 1)))                      # axis-parallel, off the planes
            out.append((c, c + e * 3))                                       # axis-parallel, along a lattice edge
    for sx in (1, -1):
        for sy in (1, -1):
            for sz in (1, -1):
                s = np.array([sx, sy, sz], float)
                for dirv in (np.ones(3), np.array([1.0, 2.0, 3.0]), np.array([1.0, 1.0, 0.375]), np.array([1.0, 0.375, 1.0]),
                             np.array([0.375, 1.0, 1.0])):
                    dv = s * dirv / 4
                    out.append((c - 3 * dv, c + 5 * dv))                     # through a corner (or an edge when one slope differs)
                    out.append((c, c + 6 * dv))                              # starting on a corner
                    out.append((c + 6 * dv, c))                              # ending on a corner
                out.append((c + np.array([0.5, 0.0, 0.25]), c + np.array([0.5 + 3 * sx, 0.0, 0.25 + 2 * sz])))   # in the plane y = c_y
                out.append((c + np.array([0, 0.5, 0.5]), c + np.array([-2.75, 0.5 + sy * 1.25, 0.5 + sz * 2])))  # starts on x plane heading down
    out.append((c, c))                                                       # zero length, on a corner
    out.append((c + 0.3, c + 0.3))                                           # zero length, inside a voxel
    out.append((np.zeros(3), G))                                             # corner to corner, ends on the upper faces
    out.append((G, np.zeros(3)))
    out.append((np.array([G[0], 1.5, 1.5]), np.array([G[0], 2.5, 0.25])))    # in the upper x face
    out.append((np.array([G[0] - 2.5, 1.5, G[2]]), np.array([G[0], 2.5, G[2]])))
    for _ in range(40):                                                      # random lattice-plane starts, dyadic slopes
        a = np.floor(rng.uniform(0, G)) + rng.integers(0, 4, 3) / 4 * (rng.random(3) < 0.5)
        b = np.clip(a + rng.integers(-24, 25, 3) / 4, 0, G)
        out.append((a, b))
    return [np.concatenate([np.clip(a, 0, G), np.clip(b, 0, G)]) for a, b in out]
