"""Reference definition of viewpoint coverage (fiesta_frontiers_score_viewpoints, fiesta_b200/csrc/fb_view.h) in numpy, expression
for expression, for the CPU tests, the GPU tests and scripts/viewpoint_bench.py.

A candidate p (metres) tagged with a kept cluster has status 2 when p fails PosInMap or has a NaN coordinate, 1 when its voxel
Pos2Vox(p) is outside the grid, never observed or has GetDistance(Vector3i) <= clearance, else 0.  For a status-0 candidate and a
member voxel v of its cluster, each fp64 operation rounded on its own (numpy evaluates elementwise, one rounding per operation):
  c = (v + 0.5) * res + origin,  d = c - p
  in range    (d0*d0 + d1*d1) + d2*d2 <= max_range * max_range
  in view j   s_k = (R[k,0]*d0 + R[k,1]*d1) + R[k,2]*d2,  s0 > 0 and |s1| <= tan_h * s0 and |s2| <= tan_v * s0
  visible     the segment {p, c} is clear at clearance 0 (status 0 of the segment query), decided by the `los` callable.
score[i, j] counts the members in range, in view of orientation j and visible."""
import numpy as np

UNDEFINED = -10000.0


def yaw(a):
    """World-to-sensor rows for a level sensor looking along yaw a: optical axis, horizontal axis, vertical axis."""
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, s, 0.0], [-s, c, 0.0], [0.0, 0.0, 1.0]])


def yaw_pitch(a, b):
    """The yaw matrix tilted by pitch b (positive looks up) about its horizontal axis."""
    cb, sb = np.cos(b), np.sin(b)
    P = np.array([[cb, 0.0, sb], [0.0, 1.0, 0.0], [-sb, 0.0, cb]])
    return P @ yaw(a)


def yaws(k):
    """k yaw matrices, evenly spaced from 0."""
    return np.stack([yaw(2 * np.pi * j / k) for j in range(k)])


def status(pos, dist, origin, res, lo, hi, clearance):
    """Candidate status (n,) for positions (n, 3); dist: (gx, gy, gz) export_distance() values; [lo, hi]: the PosInMap box."""
    pos = np.asarray(pos, np.float64).reshape(-1, 3)
    gs = np.asarray(dist.shape)
    out = np.full(len(pos), 2, np.int32)
    ok = ~np.any(np.isnan(pos), 1) & np.all(pos >= np.asarray(lo), 1) & np.all(pos <= np.asarray(hi), 1)
    v = np.floor((pos - np.asarray(origin, np.float64)) / res)
    v = np.where(np.isfinite(v), v, -1).astype(np.int64)
    ing = np.all((v >= 0) & (v < gs), 1)
    vc = np.where(ing[:, None], v, 0)
    D = dist[vc[:, 0], vc[:, 1], vc[:, 2]]
    stand = ing & (D != UNDEFINED) & (D > clearance)                      # unknown reads -10000; unreached +10000
    out[ok] = np.where(stand[ok], 0, 1)
    return out


def offsets(vox, p, origin, res):
    """Voxel centres c (m, 3) of member voxels vox (m, 3) and their offsets d = c - p."""
    c = (np.asarray(vox).astype(np.float64) + 0.5) * res + np.asarray(origin, np.float64)
    return c, c - np.asarray(p, np.float64)


def in_range(d, max_range):
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= max_range * max_range


def view_mask(R, d, tan_h, tan_v):
    """(m, n_orient) bool: d in the field of view of each orientation R[j] (row-major world-to-sensor)."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    s = [(R[None, :, k, 0] * d[:, 0, None] + R[None, :, k, 1] * d[:, 1, None]) + R[None, :, k, 2] * d[:, 2, None] for k in range(3)]
    return (s[0] > 0) & (np.abs(s[1]) <= tan_h * s[0]) & (np.abs(s[2]) <= tan_v * s[0])


def score(cluster, pos, R, max_range, tan_half_fov, clearance, sizes, members, dist, origin, res, lo, hi, los):
    """(status (n,), score (n, n_orient), stats dict).  sizes (K,) and members (M, 3) are the frontier result (members cluster by
    cluster); los(ab) takes (m, 6) segments {p, c} and returns their segment-query statuses at clearance 0 (the caller's flags)."""
    cluster = np.asarray(cluster, np.int64).reshape(-1)
    pos = np.asarray(pos, np.float64).reshape(-1, 3)
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    moff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    st = status(pos, dist, origin, res, lo, hi, clearance)
    sc = np.zeros((len(pos), len(R)), np.int32)
    segs, masks, owner = [], [], []
    for i in np.nonzero(st == 0)[0]:
        k = cluster[i]
        c, d = offsets(members[moff[k]:moff[k + 1]], pos[i], origin, res)
        m = view_mask(R, d, tan_half_fov[0], tan_half_fov[1]) & in_range(d, max_range)[:, None]
        w = np.any(m, 1)
        segs.append(np.concatenate([np.broadcast_to(pos[i], (int(w.sum()), 3)), c[w]], 1))
        masks.append(m[w])
        owner.append(np.full(int(w.sum()), i))
    walked = 0
    visible = 0
    if segs:
        ab = np.concatenate(segs)
        walked = len(ab)
        if walked:
            vis = np.asarray(los(ab)) == 0
            visible = int(vis.sum())
            np.add.at(sc, np.concatenate(owner)[vis], np.concatenate(masks)[vis].astype(np.int32))
    stats = dict(candidates_scored=int(np.sum(st == 0)), pairs_walked=int(walked), pairs_visible=int(visible))
    return st, sc, stats


def rings(centroids, radii, k):
    """Candidates on horizontal rings around each centroid: (len(centroids) * len(radii) * k, 3), cluster-major, and the cluster
    index of each."""
    a = 2 * np.pi * np.arange(k) / k
    off = np.concatenate([np.stack([r * np.cos(a), r * np.sin(a), np.zeros(k)], 1) for r in radii])
    pos = (np.asarray(centroids, np.float64)[:, None, :] + off[None]).reshape(-1, 3)
    return np.repeat(np.arange(len(centroids)), len(off)), pos
