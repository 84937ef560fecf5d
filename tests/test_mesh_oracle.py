"""CPU: the surface mesh's definition (tests/meshref.py, fiesta_b200/csrc/fb_mesh.h) checked on its own.  meshref agrees with a plain
per-cell, per-edge loop on random maps (unknown, unreached and local-map-reset records included, clearances on voxel distances).  Its
meshes are closed (every directed edge meets its reverse), have one quad per blocking/free face pair, and keep every vertex in its
cell.  Crafted solids: one voxel (V 8, T 12, chi 2), two solids (chi 4), a ring (chi 0), a hollow shell (chi 4, the inner surface of
negative volume), solids of positive volume, midpoint crossings at clearance 0.5 * res, an edge contact (closed, non-manifold),
adjacent boxes that agree bit for bit on their shared cells, an empty and an all-blocking box.  The header's crossing parameter,
cell-edge order, quad order and diagonal rule are checked against meshref (tests/cpp/mesh_test.cpp)."""
import collections
import os
import subprocess

import numpy as np
import pytest
from scipy import ndimage
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

from tests import meshref as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 0.125
ORIGIN = (-2.0, -3.0, -1.0)


def records(obst):
    """export_distance() / export_closest_obstacle()-like arrays of a grid whose voxels are all observed, obstacles `obst`."""
    gs = obst.shape
    if not obst.any():
        return np.full(gs, mr.INF), np.full(gs + (3,), mr.UNDEF, np.int64)
    _, idx = ndimage.distance_transform_edt(~obst, return_indices=True)
    O = np.moveaxis(idx, 0, -1).astype(np.int64)
    dv = O - np.moveaxis(np.indices(gs), 0, -1)
    D = np.sqrt(((dv[..., 0] * dv[..., 0] + dv[..., 1] * dv[..., 1]) + dv[..., 2] * dv[..., 2]).astype(np.float64)) * RES
    return D, O


def synth(gs, rng, p_obst=0.08, p_unknown=0.1, p_inf=0.03, p_dinf=0.03):
    """A random map: obstacles with their exact distances, never-observed voxels, unreached voxels and EXACT local-map reset
    records (+10000 with an obstacle kept)."""
    D, O = records(rng.random(gs) < p_obst)
    kind = rng.random(gs)
    unk, inf, dinf = kind < p_unknown, (kind >= p_unknown) & (kind < p_unknown + p_inf), kind >= 1 - p_dinf
    D = np.where(unk, float(mr.UNDEF), np.where(inf | dinf, mr.INF, D))
    O = np.where((unk | inf)[..., None], mr.UNDEF, O)
    return D, O


def solid(obst, r=0.0):
    """(blk, has, d) over the whole grid of a crafted obstacle set at clearance r."""
    D, O = records(obst)
    return mr.from_records(D, O, obst.shape, ((0, 0, 0), tuple(g - 1 for g in obst.shape)), r, False)


def loop_mesh(blk, has, d, lo, r, res, origin):
    """The definition as a plain loop over E's cells and grid edges: (vertices, triangles)."""
    B = blk.shape

    def at(A, p, default):
        i = tuple(p[k] - 1 for k in range(3))                              # E-local -> box-local
        return A[i] if all(0 <= i[k] < B[k] for k in range(3)) else default

    verts, vid = [], {}
    for x in range(B[0] + 1):
        for y in range(B[1] + 1):
            for z in range(B[2] + 1):
                bl = [at(blk, (x + i, y + j, z + k), False) for i in (0, 1) for j in (0, 1) for k in (0, 1)]
                if all(bl) or not any(bl):
                    continue
                s, n = [0.0, 0.0, 0.0], 0
                for a in range(3):
                    o1, o2 = [k for k in range(3) if k != a]
                    for p in (0, 1):
                        for q in (0, 1):
                            u = [x, y, z]
                            u[o1] += p
                            u[o2] += q
                            w = list(u)
                            w[a] += 1
                            if at(blk, u, False) == at(blk, w, False):
                                continue
                            if at(has, u, False) and at(has, w, False):
                                du, dw = float(at(d, u, 0.0)), float(at(d, w, 0.0))
                                t = (r - du) / (dw - du)
                            else:
                                t = 0.5
                            for k in range(3):
                                g = float(u[k] - 1 + lo[k])
                                s[k] = s[k] + (g + t if k == a else g)
                            n += 1
                vid[(x, y, z)] = len(verts)
                verts.append([np.float32(((s[k] / n + 0.5) * res) + origin[k]) for k in range(3)])
    tris = []
    for x in range(B[0] + 1):
        for y in range(B[1] + 1):
            for z in range(B[2] + 1):
                for a in range(3):
                    v = [x, y, z]
                    w = list(v)
                    w[a] += 1
                    bv = at(blk, v, False)
                    if bv == at(blk, w, False):
                        continue
                    b, c = (a + 1) % 3, (a + 2) % 3

                    def cell(db, dc):
                        q = list(v)
                        q[b] += db
                        q[c] += dc
                        return vid[tuple(q)]
                    ring = [cell(-1, -1), cell(0, -1), cell(0, 0), cell(-1, 0)]
                    if not bv:
                        ring = [ring[0], ring[3], ring[2], ring[1]]
                    P = [[float(t) for t in verts[i]] for i in ring]

                    def sq(p, q):
                        e = [p[k] - q[k] for k in range(3)]
                        return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]
                    if sq(P[0], P[2]) <= sq(P[1], P[3]):
                        tris += [(ring[0], ring[1], ring[2]), (ring[0], ring[2], ring[3])]
                    else:
                        tris += [(ring[1], ring[2], ring[3]), (ring[1], ring[3], ring[0])]
    return np.array(verts, np.float32).reshape(-1, 3), np.array(tris, np.int32).reshape(-1, 3)


def closed(T):
    """Every directed edge is matched by its reverse, as many times."""
    e = collections.Counter()
    for t in T:
        for i in range(3):
            e[(int(t[i]), int(t[(i + 1) % 3]))] += 1
    return all(e[(b, a)] == n for (a, b), n in e.items())


def euler(V, T):
    und = {tuple(sorted((int(t[i]), int(t[(i + 1) % 3])))) for t in T for i in range(3)}
    return len(V) - len(und) + len(T)


def volume(V, T):
    p = V.astype(np.float64)[T]
    return float(np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0)


def components(V, T):
    """Triangle sets of the mesh's vertex-connected components."""
    n = len(V)
    rows = np.concatenate([T[:, 0], T[:, 1], T[:, 2]])
    cols = np.concatenate([T[:, 1], T[:, 2], T[:, 0]])
    _, lab = connected_components(csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(n, n)), directed=False)
    return [T[lab[T[:, 0]] == c] for c in np.unique(lab[T[:, 0]])]


def face_pairs(blk):
    P = np.pad(np.asarray(blk, np.int8), 1)
    return sum(int(np.count_nonzero(np.diff(P, axis=a))) for a in range(3))


def check_invariants(w, blk, lo):
    V, T = w["vertices"], w["triangles"]
    assert closed(T)
    assert w["stats"]["quads"] == face_pairs(blk) and len(T) == 2 * w["stats"]["quads"]
    lo_m = (w["cells"] + 0.5) * RES + np.asarray(ORIGIN)
    hi_m = (w["cells"] + 1.5) * RES + np.asarray(ORIGIN)
    tol = 4 * np.finfo(np.float32).eps * np.maximum(np.abs(lo_m), np.abs(hi_m))
    assert np.all(V >= lo_m - tol) and np.all(V <= hi_m + tol)
    if len(T):
        assert set(np.unique(T)) == set(range(len(V)))                    # every vertex is used


CASES = [((9, 8, 7), ((0, 0, 0), (8, 7, 6))), ((11, 10, 9), ((2, 1, 3), (9, 8, 8))), ((8, 9, 10), ((3, 0, 0), (3, 8, 9))),
         ((7, 12, 6), ((0, 4, 1), (6, 4, 5))), ((6, 6, 6), ((2, 2, 2), (2, 2, 2)))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_meshref_equals_the_loop_on_random_maps(case):
    gs, box = CASES[case]
    rng = np.random.default_rng(case)
    D, O = synth(gs, rng, p_obst=0.15)
    for r in (0.0, 0.5 * RES, RES, np.sqrt(2.0) * RES, 2.5 * RES):
        for unk in (False, True):
            w = mr.mesh(D, O, gs, box, r, unk, RES, ORIGIN)
            blk, has, d = mr.from_records(D, O, gs, box, r, unk)
            V, T = loop_mesh(blk, has, d, box[0], r, RES, ORIGIN)
            assert np.array_equal(w["vertices"], V) and np.array_equal(w["triangles"], T), (r, unk)
            check_invariants(w, blk, box[0])
            assert w["stats"]["blocking"] == int(blk.sum()) and w["stats"]["box_voxels"] == blk.size


def test_invariants_on_larger_random_maps():
    rng = np.random.default_rng(11)
    gs = (40, 36, 33)
    D, O = synth(gs, rng, p_obst=0.02)
    box = ((0, 0, 0), (39, 35, 32))
    for r in (0.0, RES, 2.5 * RES):
        for unk in (False, True):
            w = mr.mesh(D, O, gs, box, r, unk, RES, ORIGIN)
            blk, _, _ = mr.from_records(D, O, gs, box, r, unk)
            check_invariants(w, blk, box[0])
            assert w["stats"]["vertices"] > 1000


def crafted(name):
    gs = (14, 14, 12)
    o = np.zeros(gs, bool)
    if name == "one":
        o[6, 6, 6] = True
    elif name == "two":
        o[2:5, 2:5, 2:5] = True
        o[8:12, 7:11, 5:9] = True
    elif name == "ring":
        o[3:11, 3:11, 4:7] = True
        o[5:9, 5:9, 4:7] = False
    elif name == "shell":
        o[2:11, 2:11, 2:10] = True
        o[5:8, 5:8, 5:7] = False
    elif name == "edge":
        o[5, 5, 5] = o[6, 6, 5] = True                                      # touching only along an edge
    return o


@pytest.mark.parametrize("name,chi", [("one", 2), ("two", 4), ("ring", 0), ("shell", 4)])
def test_crafted_solids(name, chi):
    o = crafted(name)
    blk, has, d = solid(o, 0.5 * RES)                                       # the obstacle cubes' faces
    w = mr.mesh_of(blk, has, d, (0, 0, 0), 0.5 * RES, RES, ORIGIN)
    V, T = w["vertices"], w["triangles"]
    assert np.array_equal(blk, o)
    check_invariants(w, blk, (0, 0, 0))
    assert euler(V, T) == chi
    if name == "one":
        assert len(V) == 8 and len(T) == 12
    # clearance 0: the same blocking set and triangles, the surface through the obstacle voxel centres
    w0 = mr.mesh_of(*solid(o), (0, 0, 0), 0.0, RES, ORIGIN)
    assert np.array_equal(w0["triangles"], T) or name != "one"
    if name == "one":                                                       # every vertex on the voxel's centre: zero-area triangles, kept
        assert len(w0["triangles"]) == 12 and np.all(w0["vertices"] == w0["vertices"][0])
        assert np.allclose(w0["vertices"][0], (6.5 * RES + np.asarray(ORIGIN)))
    vols = sorted(volume(V, c) for c in components(V, T))
    if name == "shell":
        assert len(vols) == 2 and vols[0] < 0 < vols[1]                    # the cavity's surface faces into the cavity
    else:
        assert all(v > 0 for v in vols)
    Vl, Tl = loop_mesh(blk, has, d, (0, 0, 0), 0.5 * RES, RES, ORIGIN)
    assert np.array_equal(V, Vl) and np.array_equal(T, Tl)


def test_half_voxel_clearance_gives_midpoint_crossings():
    rng = np.random.default_rng(3)
    o = rng.random((12, 11, 10)) < 0.1
    blk, has, d = solid(o, 0.5 * RES)
    assert np.array_equal(blk, o)
    w = mr.mesh_of(blk, has, d, (0, 0, 0), 0.5 * RES, RES, ORIGIN)
    mid = mr.mesh_of(blk, np.zeros_like(has), d, (0, 0, 0), 0.5 * RES, RES, ORIGIN)      # every t = 0.5
    assert np.array_equal(w["vertices"], mid["vertices"]) and np.array_equal(w["triangles"], mid["triangles"])
    one = mr.mesh_of(*solid(crafted("one"), 0.5 * RES), (0, 0, 0), 0.5 * RES, RES, ORIGIN)["vertices"]
    # one obstacle voxel at 6: each vertex is the mean of three face midpoints of its cube, 6 -+ 1/6 voxels on every axis
    u = (one.astype(np.float64) - np.asarray(ORIGIN)) / RES - 0.5
    assert len(one) == 8 and np.allclose(np.abs(u - 6.0), 1.0 / 6.0, rtol=0, atol=1e-5)


def test_edge_contact_is_closed_and_non_manifold():
    blk, has, d = solid(crafted("edge"))
    w = mr.mesh_of(blk, has, d, (0, 0, 0), 0.0, RES, ORIGIN)
    T = w["triangles"]
    assert closed(T)
    und = collections.Counter(tuple(sorted((int(t[i]), int(t[(i + 1) % 3])))) for t in T for i in range(3))
    assert max(und.values()) == 4                                           # the shared edge's cells carry four triangles
    assert w["stats"]["vertices"] == 8 + 8 - 2                              # two cells are shared by the two cubes


def test_adjacent_boxes_agree_on_shared_cells():
    rng = np.random.default_rng(8)
    gs = (24, 12, 11)
    D, O = synth(gs, rng)
    for r, unk in ((0.0, False), (RES, True), (2.5 * RES, False)):
        a = mr.mesh(D, O, gs, ((0, 0, 0), (14, 11, 10)), r, unk, RES, ORIGIN)
        b = mr.mesh(D, O, gs, ((8, 0, 0), (23, 11, 10)), r, unk, RES, ORIGIN)
        # cells whose 8 corners lie in both boxes: x in [8, 13], y in [0, 10], z in [0, 9]
        def shared(w):
            c = w["cells"]
            k = (c[:, 0] >= 8) & (c[:, 0] <= 13) & (c[:, 1] >= 0) & (c[:, 1] <= 10) & (c[:, 2] >= 0) & (c[:, 2] <= 9)
            return c[k], w["vertices"][k]
        ca, va = shared(a)
        cb, vb = shared(b)
        assert len(ca) > 50 and np.array_equal(ca, cb) and np.array_equal(va.view(np.uint32), vb.view(np.uint32))


def test_empty_and_all_blocking_boxes():
    gs = (9, 8, 7)
    box = ((1, 1, 1), (7, 6, 5))
    D, O = records(np.zeros(gs, bool))
    w = mr.mesh(D, O, gs, box, 0.0, False, RES, ORIGIN)
    assert w["stats"]["vertices"] == 0 and w["stats"]["triangles"] == 0 and w["triangles"].shape == (0, 3)
    D = np.full(gs, float(mr.UNDEF))
    O = np.full(gs + (3,), mr.UNDEF)
    w = mr.mesh(D, O, gs, box, 0.0, True, RES, ORIGIN)                      # nothing observed, unknown blocks: the whole box
    B = (7, 6, 5)
    assert w["stats"]["blocking"] == 7 * 6 * 5
    assert w["stats"]["quads"] == 2 * (B[0] * B[1] + B[1] * B[2] + B[0] * B[2])
    assert closed(w["triangles"]) and euler(w["vertices"], w["triangles"]) == 2 and volume(w["vertices"], w["triangles"]) > 0
    check_invariants(w, np.ones(B, bool), box[0])


# ---------------------------------------------------------------- the header (g++)
@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mesh") / "mesh_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "cpp", "mesh_test.cpp"), "-o", out])
    return out


def run(exe, mode, lines=None):
    txt = None if lines is None else "%d\n" % len(lines) + "\n".join(lines) + "\n"
    p = subprocess.run([exe, mode], input=txt, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    return p.stdout.splitlines()


def hx(vals):
    return " ".join(float(v).hex() for v in vals)


def test_header_orders(exe):
    out = run(exe, "order")
    assert [int(x) for x in out[0].split()] == [v for e in mr.CELL_EDGES for v in e]
    for i, (a, vb) in enumerate((a, vb) for a in range(3) for vb in (0, 1)):
        assert [int(x) for x in out[1 + i].split()] == mr.QUAD[a, vb].reshape(-1).tolist()


def test_header_crossing_parameter(exe):
    rng = np.random.default_rng(1)
    n = 4000
    du = np.sqrt(rng.integers(0, 60, n).astype(np.float64)) * RES
    dw = np.sqrt(rng.integers(0, 60, n).astype(np.float64)) * RES
    pick = rng.integers(0, 3, n)
    r = np.where(pick == 0, du, np.where(pick == 1, dw, rng.uniform(0, 1, n)))          # ties: r on an endpoint's distance
    lo, hi = np.minimum(du, dw), np.maximum(du, dw)
    ok = (lo <= r) & (r < hi)                                               # exactly one endpoint blocks
    du, dw, r = du[ok], dw[ok], r[ok]
    hu, hw = rng.random(len(r)) < 0.8, rng.random(len(r)) < 0.8
    lines = ["%d %s %d %s %s" % (a, float(b).hex(), c, float(d).hex(), float(e).hex()) for a, b, c, d, e in zip(hu, du, hw, dw, r)]
    got = np.array([float.fromhex(x) for x in run(exe, "t", lines)])
    want = mr.crossing_t(hu, du, hw, dw, r)
    assert np.array_equal(got, want) and np.all((want >= 0) & (want <= 1)) and np.any(want == 0) and np.any(want == 1)


def test_header_vertex(exe):
    rng = np.random.default_rng(2)
    gs = (16, 14, 12)
    D, O = synth(gs, rng, p_obst=0.1)
    lines, want = [], []
    for r, unk in ((0.0, False), (RES, True), (0.5 * RES, False), (2.5 * RES, True)):
        blk, has, d = mr.from_records(D, O, gs, ((0, 0, 0), (15, 13, 11)), r, unk)
        w = mr.mesh_of(blk, has, d, (0, 0, 0), r, RES, ORIGIN)
        P, H, Dp = np.pad(blk, 1), np.pad(has, 1), np.pad(d, 1)
        for c, v in zip(w["cells"], w["vertices"]):
            e = c + 1
            idx = [(e[0] + i, e[1] + j, e[2] + k) for i, j, k in mr.CORNERS]
            lines.append(" ".join([" ".join(str(int(x)) for x in c), " ".join(str(int(P[i])) for i in idx),
                                   " ".join(str(int(H[i])) for i in idx), hx([Dp[i] for i in idx]), hx([r, RES]), hx(ORIGIN)]))
            want.append(v)
    got = np.array([[float.fromhex(x) for x in ln.split()] for ln in run(exe, "vertex", lines)], np.float32)
    assert len(lines) > 1000 and np.array_equal(got, np.array(want, np.float32))


def test_header_diagonal_rule(exe):
    rng = np.random.default_rng(4)
    n = 3000
    P = rng.uniform(-3, 3, (n, 4, 3)).astype(np.float32)
    sq = rng.integers(0, 3, n) == 0                                         # squares: both diagonals equal, the tie splits p0-p2
    base = rng.uniform(-3, 3, (n, 3)).astype(np.float32)
    corners = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32) * np.float32(0.125)
    P[sq] = base[sq][:, None, :] + corners
    q = rng.integers(0, 10 ** 6, (n, 4))
    lines = [hx(P[i].reshape(-1)) + " " + " ".join(str(int(x)) for x in q[i]) for i in range(n)]
    got = np.array([[int(x) for x in ln.split()] for ln in run(exe, "split", lines)])
    s = mr.split02(P[:, 0], P[:, 1], P[:, 2], P[:, 3])
    assert np.array_equal(got[:, 0], s.astype(int)) and np.all(s[sq])
    assert np.array_equal(got[:, 1:], mr.tris(q, s).reshape(n, 6))
