"""CPU: the skeleton's definition (tests/skeletonref.py, fiesta_b200/csrc/fb_skel.h) checked on its own.  The vectorised simple-point
test agrees with scipy's labelling of the 3x3x3 neighbourhood; thinning passes give the same set when their voxels are deleted one
at a time in random orders; the number of 26-components and the Euler characteristic of the union of closed cubes are the same for
X0, after each thinning phase and after pruning; every edge path is 26-connected from a vertex voxel to a vertex voxel and its
length re-folds bit for bit.  Crafted cases: a ring around a pillar, a floating cube, a straight tunnel, a Y junction, a 2-voxel
component, a spur on a junction, an empty and an all-blocked box.  The header's simple-point test is checked on all 2^26
neighbourhoods and its anchor predicate against numpy (tests/cpp/skeleton_test.cpp)."""
import functools
import itertools
import os
import subprocess

import numpy as np
import pytest
from scipy import ndimage

from tests import skeletonref as sr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S26 = np.ones((3, 3, 3), bool)
S6 = ndimage.generate_binary_structure(3, 1)


def simple_by_label(cube):
    """T26 = 1 and T6 = 1 from ndimage.label on one 3x3x3 neighbourhood (bool, centre ignored)."""
    fg = cube.copy()
    fg[1, 1, 1] = False
    _, t26 = ndimage.label(fg, structure=S26)
    n18 = np.ones((3, 3, 3), bool)
    for c in itertools.product((0, 2), repeat=3):
        n18[c] = False
    n18[1, 1, 1] = False
    bg = ~cube & n18
    lab, _ = ndimage.label(bg, structure=S6)
    faces = {lab[1 + d[0], 1 + d[1], 1 + d[2]] for d in sr.FACE_DIRS} - {0}
    return t26 == 1 and len(faces) == 1


def test_simple_point_against_labelling():
    rng = np.random.default_rng(1)
    cubes = np.concatenate([rng.random((4000, 3, 3, 3)) < p for p in (0.2, 0.5, 0.8)])
    codes = np.array([sum(int(c.reshape(-1)[e]) << e for e in range(27)) for c in cubes], np.uint32)
    got = sr.simple(codes)
    want = np.array([simple_by_label(c) for c in cubes])
    assert np.array_equal(got, want)
    assert 0.05 < want.mean() < 0.95


def cubical_euler(X):
    """Euler characteristic of the union of the closed unit cubes of X: vertices - edges + faces - cubes of the complex."""
    P = np.pad(np.asarray(X, bool), 1)
    n = [0, 0, 0, 0]
    for shape in itertools.product((0, 1), repeat=3):       # 1 on an axis: the cell is open (one voxel wide) along it
        dim = sum(shape)
        # a cell is in the complex when a voxel touching it is; the voxels touching a cell differ on its closed axes
        acc = np.zeros(tuple(s + 1 - t for s, t in zip(X.shape, shape)), bool)
        for off in itertools.product(*[(0,) if t else (0, 1) for t in shape]):
            sl = tuple(slice(o + t, o + t + a) for o, t, a in zip(off, shape, acc.shape))
            acc |= P[sl]
        n[dim] += int(acc.sum())
    return n[0] - n[1] + n[2] - n[3]


def components(X):
    return ndimage.label(X, structure=S26)[1]


def invariants(X):
    return components(X), cubical_euler(X)


def test_euler_characteristic_model():
    assert cubical_euler(np.ones((1, 1, 1), bool)) == 1
    ring = np.ones((3, 3, 1), bool)
    ring[1, 1, 0] = False
    assert cubical_euler(ring) == 0
    shell = np.ones((3, 3, 3), bool)
    shell[1, 1, 1] = False
    assert cubical_euler(shell) == 2
    assert cubical_euler(np.zeros((2, 2, 2), bool)) == 0


def pillars(shape, k, seed):
    rng = np.random.default_rng(seed)
    o = np.zeros(shape, bool)
    o[:, :, 0] = True
    for _ in range(k):
        x, y = rng.integers(2, shape[0] - 3), rng.integers(2, shape[1] - 3)
        o[x:x + 2, y:y + 3, :] = True
    z = shape[2] // 2
    o[shape[0] // 4:shape[0] // 2, shape[1] // 4:shape[1] // 2, z:z + 2] = True       # a floating slab
    return o


def check_graph(S, G, res=0.1):
    """Edge paths: 26-connected, vertex voxel at both ends, their chain's voxels in between, length re-folded."""
    w = sr.weights(res)
    lab = G["labels"]
    ev = G["edge_voxels"].astype(np.int64)
    k = 0
    for e, n in enumerate(G["edges"]["n_vox"]):
        p = ev[k:k + n]
        k += n
        steps = np.abs(np.diff(p, axis=0))
        assert np.all(steps.max(1) == 1)
        assert lab[tuple(p[0])] >= 0 and lab[tuple(p[-1])] >= 0
        assert tuple(G["edges"]["uv"][e]) == (lab[tuple(p[0])], lab[tuple(p[-1])])
        assert np.all(lab[tuple(p[1:-1].T)] == -2 - e)
        L = functools.reduce(lambda acc, s: acc + w[int(np.count_nonzero(s)) - 1], steps, 0.0)
        assert L == G["edges"]["length"][e]
    assert k == len(ev) and np.count_nonzero(lab <= -2) == len(ev) - 2 * len(G["edges"]["n_vox"])
    assert np.array_equal(S, lab != -1)
    deg = np.zeros(len(G["vertices"]["size"]), np.int64)
    np.add.at(deg, G["edges"]["uv"].reshape(-1), 1)
    assert np.array_equal(deg, G["vertices"]["degree"])


@pytest.mark.parametrize("seed,max_cos,min_branch", [(0, 0.5, 8), (1, 0.5, 3), (2, -0.25, 8), (3, 0.0, 1)])
def test_topology_and_paths(seed, max_cos, min_branch):
    o = pillars((28, 26, 12), 6, seed)
    X0, A = sr.from_obstacles(o, max_cos)
    X1, X2, iters = sr.thin(X0, A)
    S, rounds, removed = sr.prune(X2, min_branch)
    inv = invariants(X0)
    assert inv[0] >= 1
    for X in (X1, X2, S):
        assert invariants(X) == inv
    assert np.all(A[X0 & ~X1] == 0) and np.all(X1 <= X0) and np.all(X2 <= X1) and np.all(S <= X2)
    assert iters[0] >= 2 and iters[1] >= 1
    if min_branch > 1:
        assert rounds >= 1 and removed == int(X2.sum() - S.sum())
    G = sr.graph(S, None, (0, 0, 0), 0.1, (0.0, 0.0, 0.0))
    check_graph(S, G)
    assert len(G["edges"]["n_vox"]) > 0


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_thinning_in_random_orders(seed):
    o = pillars((18, 16, 9), 4, seed + 10)
    X0, A = sr.from_obstacles(o, 0.5)
    want = sr.thin(X0, A)
    rng = np.random.default_rng(seed)
    got = sr.thin(X0, A, lambda X, A_, ph, s: sr.thin_pass_sequential(X, A_, ph, s, rng))
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]


def run(obst, max_cos=0.5, min_branch=8):
    X0, A = sr.from_obstacles(obst, max_cos)
    X1, X2, _ = sr.thin(X0, A)
    S, _, _ = sr.prune(X2, min_branch)
    for X in (X1, X2, S):
        assert invariants(X) == invariants(X0)
    G = sr.graph(S, None, (0, 0, 0), 0.1, (0.0, 0.0, 0.0))
    check_graph(S, G)
    return S, G


def test_ring_around_a_pillar():
    o = np.zeros((15, 15, 1), bool)
    o[5:10, 5:10, 0] = True
    S, G = run(o)
    assert cubical_euler(S) == 0 and components(S) == 1
    loops = [e for e, (u, v) in enumerate(G["edges"]["uv"]) if u == v]
    assert len(G["vertices"]["size"]) == 1 and len(loops) == 1                # a promoted vertex with one self-loop
    assert G["vertices"]["degree"][0] == 2 and G["vertices"]["size"][0] == 1


def test_floating_cube_keeps_its_cavity():
    o = np.zeros((14, 14, 14), bool)
    o[5:9, 5:9, 5:9] = True
    S, G = run(o)
    assert cubical_euler(S) == 2 and components(S) == 1
    _, holes = ndimage.label(~S)
    assert holes == 2                                                          # the cube stays enclosed


def test_straight_tunnel():
    o = np.ones((30, 7, 7), bool)
    o[:, 2:5, 2:5] = False
    S, G = run(o)
    assert components(S) == 1 and cubical_euler(S) == 1
    assert len(G["edges"]["n_vox"]) == 1 and G["edges"]["n_vox"][0] >= 28 and sorted(G["vertices"]["degree"]) == [1, 1]


def test_y_junction():
    o = np.ones((40, 40, 5), bool)
    o[2:21, 19:21, 2:4] = False
    for t in range(18):
        o[20 + t:22 + t, 20 + t:22 + t, 2:4] = False
        o[20 + t:22 + t, 19 - t:21 - t, 2:4] = False
    S, G = run(o)
    assert components(S) == 1 and cubical_euler(S) == 1
    assert max(G["vertices"]["degree"]) >= 3 and sum(G["vertices"]["degree"] == 1) == 3


def diagonal_with_spur(spur):
    """A diagonal line (i, i) of 20 voxels; the voxels `spur` branch off its voxel (9, 9)."""
    S = np.zeros((22, 22, 3), bool)
    for i in range(20):
        S[i, i, 1] = True
    for v in spur:
        S[v[0], v[1], 1] = True
    return S


def test_two_voxel_component_survives_pruning():
    S = diagonal_with_spur([(10, 8), (11, 7), (12, 6)])                       # a spur of 3 voxels: an edge of 4 path voxels
    S[2, 15, 1] = S[2, 16, 1] = True                                           # a 2-voxel component
    P, rounds, removed = sr.prune(S, 8)
    assert P[2, 15, 1] and P[2, 16, 1] and components(P) == 2 and invariants(P) == invariants(S)
    assert not P[10:13, 6:9, 1].any() and removed == 3 and rounds == 2
    G = sr.graph(P, None, (0, 0, 0), 0.1, (0.0, 0.0, 0.0))
    check_graph(P, G)
    assert len(G["edges"]["n_vox"]) == 1 and len(G["vertices"]["size"]) == 3    # the line's two leaves, the pair as one vertex
    assert sr.prune(S, 4)[2] == 3 and sr.prune(S, 3)[2] == 0                  # fewer than min_branch voxels, the leaf counted


def test_spur_directly_on_a_junction():
    S = diagonal_with_spur([(10, 8)])                                          # touches only the line's voxel (9, 9)
    G = sr.graph(S)
    assert G["deg"][10, 8, 1] == 1 and G["deg"][9, 9, 1] == 3
    assert not G["leaf"].all()                                                 # the spur is part of the junction's vertex
    rm = sr.prune_round(S, 2)
    assert rm[10, 8, 1] and rm.sum() == 1                                      # rule (b)
    assert not sr.prune_round(S, 1).any() and sr.prune(S, 1)[1] == 0          # min_branch <= 1: no pruning
    P, _, _ = sr.prune(S, 2)
    assert invariants(P) == invariants(S)


def test_empty_and_all_blocked_boxes():
    S, G = run(np.zeros((9, 8, 7), bool))                                      # no obstacle: no anchor, one voxel is left
    assert S.sum() == 1 and len(G["vertices"]["size"]) == 1 and len(G["edges"]["n_vox"]) == 0
    S, G = run(np.ones((9, 8, 7), bool))
    assert S.sum() == 0 and len(G["vertices"]["size"]) == 0


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("skeleton") / "skeleton_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "cpp", "skeleton_test.cpp"), "-o", out])
    return out


def test_header_simple_point_on_every_neighbourhood(exe):
    p = subprocess.run([exe, "simple"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    n, k, bad = (int(x) for x in p.stdout.split()[1::2])
    assert n == 1 << 26 and bad == 0 and 0 < k < n


def test_header_anchor_predicate(exe):
    rng = np.random.default_rng(5)
    n = 3000
    v = rng.integers(0, 2046, (n, 3))
    u = v + np.eye(3, dtype=np.int64)[rng.integers(0, 3, n)] * rng.choice((-1, 1), (n, 1))
    o = v + rng.integers(-40, 41, (n, 3))
    q = u + rng.integers(-40, 41, (n, 3))
    q[:200] = o[:200]                                                          # the same obstacle: never an anchor
    q[200:400] = u[200:400] + (o[200:400] - v[200:400])                        # parallel offsets: cos = 1
    mc = rng.uniform(-1, 1, n)
    a, b = o - v, q - u
    tie = slice(400, 1400)                                                     # max_cos at the pair's own cosine
    ab = np.sum(a[tie] * b[tie], 1).astype(np.float64)
    mc[tie] = ab / np.sqrt(np.sum(a[tie] ** 2, 1).astype(np.float64) * np.sum(b[tie] ** 2, 1).astype(np.float64))
    mc[tie] = np.clip(mc[tie], -1.0, np.nextafter(1.0, 0.0))
    exact = np.array([[1, 1, 0], [1, 0, 1], [0, 1, 1]])                        # cos = 0.5 exactly
    a[1400:1403], b[1400:1403], mc[1400:1403] = exact, exact[[1, 2, 0]], 0.5
    q[1400:1403] = u[1400:1403] + b[1400:1403]
    o[1400:1403] = v[1400:1403] + a[1400:1403]
    a, b = o - v, q - u
    txt = [str(n)] + [" ".join(str(int(x)) for x in (*v[i], *o[i], *u[i], *q[i])) + " " + float(mc[i]).hex() for i in range(n)]
    p = subprocess.run([exe, "anchor"], input="\n".join(txt) + "\n", capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    got = np.array([c == "1" for c in p.stdout.strip()])
    want = np.any(o != q, 1) & sr.anchor_pair(a, b, mc)
    assert np.array_equal(got, want)
    assert want[1400:1403].all() and not want[:200].any()
    assert 0.1 < want.mean() < 0.9 and want[tie].sum() > 100
