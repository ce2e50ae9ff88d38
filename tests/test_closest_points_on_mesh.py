"""find_closest_points_on_mesh (closest points on the posed mesh over a refitted bounding-volume tree) on the device, against the linear
scan that defines it and a float64 restatement.

The result for query p is the face with the smallest (d2_f, f) among the candidates, the faces with finite vertices and finite
d2_f <= max_dist^2; so it must not depend on the tree: the emulated traversal equals the emulated linear scan bit for bit, and on the
GPU two trees over one mesh give the same bits. Against float64 (``_closest64``, Ericson 5.1.5 in numpy), with u = 2^-24 and S the largest
coordinate magnitude of the instance's vertices and the query, K pinned at about four times the worst value measured over the fixtures
below on the emulator and on an H100:
  distance   | |q - p| - D64 | <= K_D u S                         D64 the float64 distance from p to the mesh
  face       face == the float64 closest face                    wherever the float64 gap to the second-best face exceeds 2 K_D u S
  point      | q - sum_k b_k x[face_k] | <= K_B u S,  b_k >= -K_B u,  | sum_k b_k - 1 | <= K_B u
The self-checks show that these reject a projection without the edge regions, the nearest vertex instead of the nearest surface point,
and (through the tree-independence check) a leaf that skips its last face and a prune on >=.
"""
import copy

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_vertex_normals import _tube

EPS32 = 2.0 ** -24
LEAF_FACES, TREE_STACK = 4, 32  # kLeafFaces, kTreeStack (ik_types.h)

# worst measured ratios over these fixtures and three seeds, on the emulator / on an H100 80GB HBM3 at a 700 W power limit: distance 1.28
# / 1.28 (humanoid72_far), point and barycentrics 2.27 / 2.38 (humanoid72_far); each K is about four times the larger
K_D = 5.0
K_B = 10.0


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _edge_mesh():
    """A single triangle; an isolated vertex; a zero-area face on exactly collinear points; a face that repeats an index; a small fan.
    Positions on a 1/64 grid."""
    rng = np.random.default_rng(23)
    x = np.zeros((16, 3))
    x[0:3] = [(0, 0, 0), (1, 0, 0), (0, 1, 0)]
    x[3] = (5, 5, 5)  # isolated
    x[4:7] = [(1, 1, 1), (2, 2, 2), (4, 4, 4)]  # collinear
    x[7] = (3, 0, 0.25)
    ang = 2 * np.pi * np.arange(8) / 8
    x[8:16] = np.stack([3 + np.cos(ang), np.sin(ang), rng.normal(scale=0.2, size=8)], -1)
    x = np.round(x * 64) / 64
    faces = [(0, 1, 2), (4, 5, 6), (8, 8, 9)] + [(7, 8 + k, 8 + (k + 1) % 8) for k in range(8)]
    ch = mc.create_test_character(3)
    V = x.shape[0]
    index = np.zeros((V, mc.MAX_SKIN_JOINTS), np.int32)
    weight = np.zeros((V, mc.MAX_SKIN_JOINTS), np.float32)
    weight[:, 0] = 1.0
    ch.skinning = mc.Skinning(x.astype(np.float32), index, weight, mc.synthetic_skinning(ch, 1, 0).inverse_bind_pose, np.array(faces, np.int32))
    ch.name = "edges"
    return ch


def _tiny_mesh():
    """Fewer faces than a leaf holds: two triangles sharing an edge, and the single-face mesh on its own."""
    ch = _edge_mesh()
    sk = ch.skinning
    ch.skinning = mc.Skinning(sk.rest_vertices, sk.skin_index, sk.skin_weight, sk.inverse_bind_pose, np.array([(0, 1, 2), (1, 7, 2)], np.int32))
    ch.name = "tiny"
    return ch


FIXTURES = {
    "chain3": lambda: _tube(lambda: mc.create_test_character(3), 6, 8, 1, "chain3"),
    "humanoid72": lambda: _tube(lambda: mc.humanoid72()[0], 12, 12, 2, "humanoid72"),
    "bodyhands300": lambda: _tube(lambda: mc.bodyhands300()[0], 8, 8, 3, "bodyhands300"),
    "humanoid72_far": lambda: _tube(lambda: mc.humanoid72()[0], 12, 12, 4, "humanoid72_far", far=True),
    "edges": _edge_mesh,
    "tiny": _tiny_mesh,
}
_cache = {}


def _fixture(name):
    if name not in _cache:
        _cache[name] = FIXTURES[name]()
    return _cache[name]


def _posed(ch, B, seed):
    """[B, V, 3] float32: the rest mesh (instance 0) and, for the tubes, skinned at seeded random poses; the edge meshes are scaled by
    powers of two and shifted by quarters."""
    x = np.asarray(ch.skinning.rest_vertices, np.float32)
    if ch.name in ("edges", "tiny"):
        b = np.arange(B)
        return ((2.0 ** (b % 3))[:, None, None] * x[None] + 0.25 * np.stack([b, -2 * b, 3 * b], -1)[:, None, :]).astype(np.float32)
    theta = np.random.default_rng(seed).uniform(-0.4, 0.4, (B, ch.num_params))
    theta[0] = 0.0
    t, q, s = mc.forward_kinematics(ch, theta)
    return mc.skin_points(ch, np.concatenate([t, q, s[..., None]], -1)).astype(np.float32)


def _face_normals(faces, x):
    f = np.asarray(faces, np.int64)
    n = np.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]])
    return n / np.maximum(np.linalg.norm(n, axis=-1, keepdims=True), 1e-30)


def _queries(ch, x, n, seed, scan_only=False):
    """[n, 3] float32 queries for one instance x [V, 3]: surface samples offset along the face normal (scan-like), uniform in the inflated
    bounding box, and unless scan_only: vertices exactly, midpoints of face edges, points 1e3 units out, and non-finite points."""
    rng = np.random.default_rng(seed)
    f = np.asarray(ch.skinning.faces, np.int64)
    x64 = x.astype(np.float64)
    good = np.isfinite(x64[f]).all((1, 2))
    fi = rng.choice(np.flatnonzero(good), n)
    w = rng.dirichlet(np.ones(3), n)
    surf = (w[:, :, None] * x64[f[fi]]).sum(1) + rng.normal(scale=0.3, size=(n, 1)) * _face_normals(f, x64)[fi]
    if scan_only:
        return surf.astype(np.float32)
    lo, hi = x64.min(0), x64.max(0)
    pad = 0.2 * (hi - lo) + 1.0
    box = rng.uniform(lo - pad, hi + pad, (n, 3))
    k = max(n // 8, 2)
    vert = x64[f[rng.integers(0, len(f), k), rng.integers(0, 3, k)]]
    e = rng.integers(0, len(f), k)
    mid = 0.5 * (x64[f[e, 0]] + x64[f[e, 1]])
    d = rng.normal(size=(4, 3))
    far = 0.5 * (lo + hi) + 1e3 * d / np.linalg.norm(d, axis=1, keepdims=True)
    bad = np.array([(np.nan, 0, 0), (np.inf, 0, 0), (0, -np.inf, 1), (np.nan, np.nan, np.nan)])
    q = np.concatenate([surf[: n // 2], box[: n // 4], vert, mid, far, bad])
    return q.astype(np.float32)


# ---- float64 references --------------------------------------------------------------------------------------------------------------
def _project64(p, a, b, c, edges=True):
    """Closest point and barycentrics of triangles (a, b, c) to p, in float64 (Ericson 5.1.5): vertex A, vertex B, edge AB, vertex C,
    edge AC, edge BC, interior, the first region that holds. Broadcasts over leading axes. ``edges`` = False drops the edge regions (a
    wrong variant for the self-checks)."""
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    dt = lambda u, v: (u * v).sum(-1)
    d1, d2, d3, d4, d5, d6 = dt(ab, ap), dt(ac, ap), dt(ab, bp), dt(ac, bp), dt(ab, cp), dt(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    with np.errstate(divide="ignore", invalid="ignore"):
        v_ab = d1 / (d1 - d3)
        w_ac = d2 / (d2 - d6)
        w_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        den = 1.0 / (va + vb + vc)
    v_in, w_in = vb * den, vc * den
    one, zero = np.ones_like(d1), np.zeros_like(d1)
    bary = np.stack([1.0 - v_in - w_in, v_in, w_in], -1)
    sel = lambda m, val: np.where(m[..., None], np.stack(val, -1), bary)
    if edges:
        bary = sel((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), (zero, 1.0 - w_bc, w_bc))
        bary = sel((vb <= 0) & (d2 >= 0) & (d6 <= 0), (1.0 - w_ac, zero, w_ac))
    bary = sel((d6 >= 0) & (d5 <= d6), (zero, zero, one))
    if edges:
        bary = sel((vc <= 0) & (d1 >= 0) & (d3 <= 0), (1.0 - v_ab, v_ab, zero))
    bary = sel((d3 >= 0) & (d4 <= d3), (zero, one, zero))
    bary = sel((d1 <= 0) & (d2 <= 0), (one, zero, zero))
    q = bary[..., 0:1] * a + bary[..., 1:2] * b + bary[..., 2:3] * c
    return q, bary


def _closest64(faces, x, p, edges=True, chunk=16, use=None):
    """For one instance x [V, 3] and queries p [n, 3]: (D64 [n] the float64 distance to the mesh over faces with finite vertices (inf when
    none), face [n] (-1), gap [n] to the second-best face, q [n, 3]). ``use``: a mask of the faces to search (all by default)."""
    f = np.asarray(faces, np.int64)
    x = np.asarray(x, np.float64)
    a, b, c = x[f[:, 0]], x[f[:, 1]], x[f[:, 2]]
    ok = np.isfinite(x[f]).all((1, 2)) & (True if use is None else use)
    n = p.shape[0]
    D, face, gap, Q = np.full(n, np.inf), np.full(n, -1), np.full(n, np.inf), np.zeros((n, 3))
    for s in range(0, n, chunk):
        pp = np.asarray(p[s:s + chunk], np.float64)[:, None, :]
        with np.errstate(invalid="ignore", over="ignore"):
            q, _ = _project64(pp, a[None], b[None], c[None], edges)
            d = np.linalg.norm(q - pp, axis=-1)
        d = np.where(ok[None] & np.isfinite(d), d, np.inf)
        order = np.argsort(d, axis=1, kind="stable")[:, :2]
        r = np.arange(d.shape[0])
        best, second = d[r, order[:, 0]], d[r, order[:, 1]] if d.shape[1] > 1 else np.full(d.shape[0], np.inf)
        fin = np.isfinite(best)
        D[s:s + chunk] = best
        face[s:s + chunk] = np.where(fin, order[:, 0], -1)
        with np.errstate(invalid="ignore"):
            gap[s:s + chunk] = second - best
        Q[s:s + chunk] = np.where(fin[:, None], q[r, order[:, 0]], 0.0)
    return D, face, gap, Q


def _degenerate(faces, x):
    """Faces of zero area at positions x [V, 3]: whether such a face is a candidate depends on the rounding of its region tests (its
    interior branch gives NaN), so it is searched apart."""
    f = np.asarray(faces, np.int64)
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        return (np.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]]) == 0).all(-1)


def _ratios(faces, x, p, q, face, bary, ref=None):
    """(distance ratio, face mismatches beyond the gap, point / barycentric ratio) of one instance's results against float64. Where a
    zero-area face is as close as the others in float64, only |q - p| in [D64 over all faces, D64 over the others] is required."""
    deg = _degenerate(faces, x)
    D, f64, gap, _ = _closest64(faces, x, p, use=~deg) if ref is None else ref
    Dall = _closest64(faces, x, p)[0] if deg.any() else D
    x64 = np.asarray(x, np.float64)
    fin = np.isfinite(x64).all(1)
    S = np.maximum(np.abs(x64[fin]).max() if fin.any() else 0.0, np.nan_to_num(np.abs(p.astype(np.float64)), posinf=0.0).max(1))
    S = np.maximum(S, 1e-30)
    valid = face >= 0
    assert np.array_equal(valid, np.isfinite(D)), "valid differs from the float64 candidates"
    assert (q[~valid] == 0).all() and (bary[~valid] == 0).all()
    v = valid
    d = np.linalg.norm(q[v].astype(np.float64) - p[v].astype(np.float64), axis=-1)
    err = np.abs(d - D[v])
    amb = Dall[v] < D[v]
    err[amb] = np.maximum(np.maximum(Dall[v][amb] - d[amb], d[amb] - D[v][amb]), 0.0)
    rd = float((err / (EPS32 * S[v])).max(initial=0.0))
    sure = v & (gap > 2 * K_D * EPS32 * S) & ~(Dall < D)
    wrong = int((face[sure] != f64[sure]).sum())
    fv = np.asarray(faces, np.int64)[face[v]]
    b = bary[v].astype(np.float64)
    recon = (b[:, :, None] * x64[fv]).sum(1)
    rb = max(float((np.abs(recon - q[v]).max(-1) / (EPS32 * S[v])).max(initial=0.0)),
             float((np.maximum(-b.min(-1), 0) / EPS32).max(initial=0.0)), float((np.abs(b.sum(-1) - 1) / EPS32).max(initial=0.0)))
    return rd, wrong, rb


def _check(faces, x, p, q, face, bary, where):
    """x [B, V, 3], p [B, N, 3] and the results of every instance against the bounds."""
    worst = [0.0, 0.0]
    for b in range(x.shape[0]):
        rd, wrong, rb = _ratios(faces, x[b], p[b], q[b], face[b], bary[b])
        assert rd <= K_D and wrong == 0 and rb <= K_B, (where, b, rd, wrong, rb)
        worst = [max(worst[0], rd), max(worst[1], rb)]
    return worst


# ---- CPU ----------------------------------------------------------------------------------------------------------------------------
def _segment64(p, a, b):
    t = np.clip(((p - a) * (b - a)).sum(-1) / ((b - a) ** 2).sum(-1), 0.0, 1.0)
    return np.linalg.norm(a + t[..., None] * (b - a) - p, axis=-1)


def test_numpy_reference_agrees_with_an_independent_minimisation():
    """On random triangles and points in every Voronoi region: the float64 restatement against (1) the distance as the minimum of the
    plane projection (when it falls inside) and the three segment distances, and (2) dense barycentric sampling."""
    rng = np.random.default_rng(5)
    T, n = 200, 40
    tri = rng.normal(size=(T, 3, 3))
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    # points around each triangle: barycentric coordinates in [-1, 2] and an offset along the normal reach all seven regions
    w = rng.uniform(-1.0, 2.0, (T, n, 2))
    nrm = np.cross(b - a, c - a)
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    p = a[:, None] + w[..., :1] * (b - a)[:, None] + w[..., 1:] * (c - a)[:, None] + rng.normal(size=(T, n, 1)) * nrm[:, None]
    q, bary = _project64(p, a[:, None], b[:, None], c[:, None])
    d = np.linalg.norm(q - p, axis=-1)
    # regions, from the barycentrics: a vertex (one 1), an edge (one 0), the interior (all > 0)
    zeros = (bary == 0).sum(-1)
    region = np.where(zeros == 2, np.argmax(bary, -1), np.where(zeros == 1, 3 + np.argmin(bary, -1), 6))
    assert set(np.unique(region)) == set(range(7))
    assert np.allclose(bary.sum(-1), 1.0, atol=1e-12) and (bary >= -1e-12).all()
    # (1) the same distance by another route
    A, B, Cc = (v[:, None].repeat(n, 1) for v in (a, b, c))
    h = ((p - A) * nrm[:, None]).sum(-1)
    foot = p - h[..., None] * nrm[:, None]
    M = np.stack([B - A, Cc - A], -1)
    lam = np.linalg.solve(np.einsum("...ki,...kj->...ij", M, M), np.einsum("...ki,...k->...i", M, foot - A)[..., None])[..., 0]
    inside = (lam >= 0).all(-1) & (lam.sum(-1) <= 1)
    alt = np.minimum.reduce([_segment64(p, A, B), _segment64(p, A, Cc), _segment64(p, B, Cc), np.where(inside, np.abs(h), np.inf)])
    assert np.abs(d - alt).max() <= 1e-12 * max(1.0, alt.max())
    # (2) dense sampling, then the sampled minimum refined by the grid's resolution
    k = 120
    i, j = np.meshgrid(np.arange(k + 1), np.arange(k + 1), indexing="ij")
    keep = i + j <= k
    u, v = i[keep] / k, j[keep] / k
    for t in range(0, T, 20):
        pts = a[t] + u[:, None] * (b[t] - a[t]) + v[:, None] * (c[t] - a[t])
        dist = np.linalg.norm(p[t][:, None, :] - pts[None], axis=-1).min(1)
        edge = max(np.linalg.norm(b[t] - a[t]), np.linalg.norm(c[t] - a[t]), np.linalg.norm(c[t] - b[t]))
        assert (d[t] <= dist + 1e-12).all() and (dist <= d[t] + edge / k).all()


@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _emu_tree(L, faces, ref):
    faces, ref = _c(faces, np.int32), _c(ref, np.float32)
    F, V = faces.shape[0], ref.shape[0]
    sizes = np.zeros(2, np.int32)
    ns, nc, lf, ls = np.full(2 * F, -7, np.int32), np.full(2 * F, -7, np.int32), np.full(F, -7, np.int32), np.full(TREE_STACK + 1, -7, np.int32)
    rc = L.emu_mesh_tree(V, F, faces.ctypes.data, V, ref.ctypes.data, sizes.ctypes.data, ns.ctypes.data, nc.ctypes.data, lf.ctypes.data, ls.ctypes.data)
    assert rc == 0, L.emu_last_error()
    n, depth = int(sizes[0]), int(sizes[1])
    return n, depth, ns[:n], nc[:n], lf, ls[:depth + 1]


def _emu_run(L, faces, ref, x, p, max_dist=np.inf, mode=0, visits=False):
    faces, ref, x, p = _c(faces, np.int32), _c(ref, np.float32), _c(x, np.float32), _c(p, np.float32)
    B, V, _ = x.shape
    N = p.shape[1]
    q, face, bary = np.full((B, N, 3), np.nan, np.float32), np.full((B, N), -7, np.int32), np.full((B, N, 3), np.nan, np.float32)
    vis = np.zeros((B, N), np.int32)
    rc = L.emu_closest_points(V, faces.shape[0], faces.ctypes.data, ref.ctypes.data, B, N, x.ctypes.data, p.ctypes.data, float(max_dist), mode,
                              q.ctypes.data, face.ctypes.data, bary.ctypes.data, vis.ctypes.data if visits else None)
    assert rc == 0, L.emu_last_error()
    return (q, face, bary, vis) if visits else (q, face, bary)


def _instances(ch, B, seed, N):
    x = _posed(ch, B, seed)
    p = np.stack([_queries(ch, x[b], N, seed + 100 + b) for b in range(B)])
    return x, p


N_CPU = {"chain3": 96, "humanoid72": 64, "bodyhands300": 48, "humanoid72_far": 64, "edges": 96, "tiny": 64}


def test_mesh_tree_invariants(emu):
    for name in FIXTURES:
        ch = _fixture(name)
        faces, rest = ch.skinning.faces, ch.skinning.rest_vertices
        F = faces.shape[0]
        n, depth, ns, nc, lf, ls = _emu_tree(emu, faces, rest)
        assert np.array_equal(np.sort(lf), np.arange(F)), name
        leaf = nc > 0
        assert (nc[leaf] <= LEAF_FACES).all() and (nc >= 0).all()
        cover = np.zeros(F, np.int64)
        for s, k in zip(ns[leaf], nc[leaf]):
            cover[s:s + k] += 1
        assert (cover == 1).all(), name  # every face in exactly one leaf
        assert 1 <= depth <= TREE_STACK and ls[0] == 0 and ls[-1] == n and (np.diff(ls) > 0).all()
        level = np.repeat(np.arange(depth), np.diff(ls))
        inner = np.flatnonzero(~leaf)
        assert (level[ns[inner]] == level[inner] + 1).all() and (level[ns[inner] + 1] == level[inner] + 1).all()
        children = np.concatenate([ns[inner], ns[inner] + 1, [0]])
        assert np.array_equal(np.sort(children), np.arange(n))  # every node but the root has one parent
        # the boxes at the reference pose: exact over the leaf faces' vertices, and every parent holds its children
        boxes = np.zeros((n, 6), np.float32)
        assert emu.emu_mesh_tree_boxes(rest.shape[0], F, _c(faces, np.int32).ctypes.data, _c(rest, np.float32).ctypes.data,
                                       _c(rest, np.float32).ctypes.data, boxes.ctypes.data) == 0
        for i in inner:
            for c in (ns[i], ns[i] + 1):
                assert (boxes[i, :3] <= boxes[c, :3]).all() and (boxes[i, 3:] >= boxes[c, 3:]).all(), (name, i)
        for i in np.flatnonzero(leaf)[:50]:
            v = rest[faces[lf[ns[i]:ns[i] + nc[i]]].reshape(-1)]
            assert np.array_equal(boxes[i, :3], v.min(0)) and np.array_equal(boxes[i, 3:], v.max(0))
        again = _emu_tree(emu, faces, rest)
        assert all(np.array_equal(u, w) for u, w in zip(again[2:], (ns, nc, lf, ls))) and again[:2] == (n, depth)
    # sizes of the tube meshes at kLeafFaces = 4 (DESIGN §4): 10 223 and 18 599 nodes
    for name, F in (("humanoid72", 20448), ("bodyhands300", 37200)):
        ch = _fixture(name)
        assert ch.skinning.faces.shape[0] == F
        n = _emu_tree(emu, ch.skinning.faces, ch.skinning.rest_vertices)[0]
        assert n == 2 * -(-F // LEAF_FACES) - 1, (name, n)  # ceil(F / 4) leaves: every split keeps whole leaves


def test_mesh_tree_is_rejected_with_a_message(emu):
    faces = np.array([(0, 1, 2)], np.int32)
    x = np.zeros((3, 3), np.float32)
    buf = [np.zeros(64, np.int32) for _ in range(5)]

    def call(V, F, f, Vt, ref):
        return emu.emu_mesh_tree(V, F, None if f is None else f.ctypes.data, Vt, None if ref is None else ref.ctypes.data, *[b.ctypes.data for b in buf])

    nan = x.copy(); nan[1, 2] = np.nan
    inf = x.copy(); inf[0, 0] = np.inf
    for args, msg in (((3, 0, None, 3, x), "no faces"), ((3, 1, faces, 4, np.zeros((4, 3), np.float32)), "differs"), ((3, 1, faces, 3, None), "null"),
                      ((3, 1, faces, 3, nan), "not finite"), ((3, 1, faces, 3, inf), "not finite")):
        assert call(*args) == 1 and msg in emu.emu_last_error().decode(), (msg, emu.emu_last_error())
    assert call(3, 1, faces, 3, x) == 0  # all vertices equal: a degenerate but valid reference


def _reference_poses(ch, x, seed):
    """Reference positions for trees over ch's faces: the rest mesh, a posed instance, all vertices equal, and the rest mesh shuffled."""
    rest = ch.skinning.rest_vertices
    perm = np.random.default_rng(seed).permutation(rest.shape[0])
    return {"rest": rest, "posed": x[-1], "equal": np.zeros_like(rest) + rest[0], "shuffled": rest[perm]}


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_traversal_equals_the_linear_scan(emu, name):
    ch = _fixture(name)
    faces = ch.skinning.faces
    x, p = _instances(ch, 2, 7, N_CPU[name])
    scan = _emu_run(emu, faces, ch.skinning.rest_vertices, x, p, mode=1)
    for tree, ref in _reference_poses(ch, x, 8).items():
        got = _emu_run(emu, faces, ref, x, p)
        for u, w in zip(got, scan):
            assert np.array_equal(u, w, equal_nan=True), (name, tree)
    # a bound: the same selection restricted to max_dist, and bit for bit the scan's
    d = np.linalg.norm(scan[0] - p, axis=-1)
    md = float(np.median(d[scan[1] >= 0]))
    lim = _emu_run(emu, faces, ch.skinning.rest_vertices, x, p, max_dist=md)
    assert all(np.array_equal(u, w, equal_nan=True) for u, w in zip(lim, _emu_run(emu, faces, x[0], x, p, max_dist=md, mode=1)))
    keep = (scan[1] >= 0) & (d <= md * (1 - 1e-6))
    assert np.array_equal(lim[1][keep], scan[1][keep]) and (lim[1][d > md * (1 + 1e-6)] == -1).all()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulator_meets_the_float64_bounds(emu, name):
    ch = _fixture(name)
    x, p = _instances(ch, 2, 17, N_CPU[name])
    q, face, bary = _emu_run(emu, ch.skinning.faces, ch.skinning.rest_vertices, x, p)
    _check(ch.skinning.faces, x, p, q, face, bary, name)
    assert (face[:, -4:] == -1).all()  # the non-finite queries


def test_edge_cases_on_the_edge_mesh(emu):
    ch = _fixture("edges")
    faces, rest = ch.skinning.faces, ch.skinning.rest_vertices
    x = rest[None]
    # a vertex shared by faces 2 .. 10 (vertex 8): distance 0 in several faces, the lowest index wins
    p = np.array([[rest[8], rest[7], rest[3], (0.0, 0.0, -0.5)]], np.float32)
    q, face, bary = _emu_run(emu, faces, rest, x, p)
    shares8 = np.flatnonzero((faces == 8).any(1))
    assert face[0, 0] == shares8.min() and np.array_equal(q[0, 0], rest[8])
    assert face[0, 1] == 3 and np.array_equal(q[0, 1], rest[7])  # the hub, in faces 3 .. 10
    # exactly at max_dist: (0, 0, -0.5) is 0.5 from vertex 0 of face 0, d2 = 0.25 exactly
    for md, want in ((0.5, 0), (np.nextafter(np.float32(0.5), np.float32(0)), -1), (np.inf, 0), (0.0, -1)):
        f = _emu_run(emu, faces, rest, x, p[:, 3:], max_dist=md)[1]
        assert f[0, 0] == want, (md, f)
    # the collinear face (4, 5, 6) has zero area: beside its middle, its edge regions give the point on the segment
    mid = np.array([[[2.0, 2.0, 2.0 + 1e-3]]], np.float32)
    q, face, _ = _emu_run(emu, faces, rest, x, mid)
    assert face[0, 0] == 1 and np.abs(q[0, 0] - (2 + 1e-3 / 3)).max() <= 1e-6
    # a face with a non-finite vertex is never chosen
    xn = x.copy()
    xn[0, 1] = (np.inf, 0, 0)
    f = _emu_run(emu, faces, rest, xn, np.array([[(0.1, 0.1, 0.0)]], np.float32))[1]
    assert f[0, 0] != 0


def test_checks_reject_wrong_closest_points(emu):
    """Each check against a mistake it is there to catch."""
    ch = _fixture("humanoid72")
    faces = ch.skinning.faces
    x, p = _instances(ch, 1, 27, 64)
    x, p = x[0], p[0, :-4]
    ref = _closest64(faces, x, p)
    # a projection without the edge regions
    _, f_ne, _, q_ne = _closest64(faces, x, p, edges=False)
    fin = f_ne >= 0
    d_ne = np.linalg.norm(q_ne - p, axis=-1)
    S = np.abs(x).max()
    assert (np.abs(d_ne[fin] - ref[0][fin]) / (EPS32 * S)).max() > 100 * K_D
    # the nearest vertex instead of the nearest surface point
    dv = np.linalg.norm(p[:, None, :].astype(np.float64) - x[None].astype(np.float64), axis=-1)
    nv = dv.argmin(1)
    assert (np.abs(dv[np.arange(len(p)), nv] - ref[0]) / (EPS32 * S)).max() > 100 * K_D
    # the right answer passes
    q, face, bary = _emu_run(emu, faces, ch.skinning.rest_vertices, x[None], p[None])
    rd, wrong, rb = _ratios(faces, x, p, q[0], face[0], bary[0], ref)
    assert rd <= K_D and wrong == 0 and rb <= K_B
    # a leaf that skips its last face, and a prune on >=: the traversal no longer equals the scan (on ties at shared vertices, for the
    # prune)
    for name in ("chain3", "humanoid72"):
        c = _fixture(name)
        xs, ps = _instances(c, 1, 37, 96)
        scan = _emu_run(emu, c.skinning.faces, c.skinning.rest_vertices, xs, ps, mode=1)
        for mode in (2, 3):
            found = any(not np.array_equal(_emu_run(emu, c.skinning.faces, r, xs, ps, mode=mode)[1], scan[1])
                        for r in _reference_poses(c, xs, 9).values())
            assert found, (name, mode)


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = _fixture("chain3")
    with pytest.raises(ValueError, match="CUDA"):
        tsk.find_closest_points_on_mesh(ch, torch.zeros(4, 3), torch.zeros(ch.skinning.num_vertices, 3))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_run(dc, x, p, max_dist=float("inf"), stream=None):
    B, N = p.shape[0], p.shape[1]
    q = torch.full((B, N, 3), float("nan"), device=x.device)
    face = torch.full((B, N), -7, dtype=torch.int32, device=x.device)
    bary = torch.full((B, N, 3), float("nan"), device=x.device)
    s = torch.cuda.current_stream().cuda_stream if stream is None else stream
    dc.closest_points_on_mesh_device(B, N, x.data_ptr(), p.data_ptr(), max_dist, q.data_ptr(), face.data_ptr(), bary.data_ptr(), s)
    return q, face, bary


def _np(t):
    return tuple(u.cpu().numpy() for u in t)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_meets_the_float64_bounds_whatever_the_tree(name):
    ch = _fixture(name)
    dc = ms.DeviceCharacter(ch, 0)
    assert dc.mesh_tree_error is None
    x, p = _instances(ch, 3, 41, N_CPU[name] * 2)
    xd, pd = _dev(x), _dev(p)
    out = _device_run(dc, xd, pd)
    q, face, bary = _np(out)
    _check(ch.skinning.faces, x, p, q, face, bary, name)
    assert (face[:, -4:] == -1).all()
    # trees from other reference poses give the same bits
    for tree, ref in _reference_poses(ch, x, 42).items():
        dc.set_mesh_tree(ref)
        again = _device_run(dc, xd, pd)
        assert all(torch.equal(u, w) for u, w in zip(again, out)), (name, tree)
    # a bound
    md = float(np.median(np.linalg.norm(q - p, axis=-1)[face >= 0]))
    ql, fl, bl = _np(_device_run(dc, xd, pd, md))
    d = np.linalg.norm(q - p, axis=-1)
    keep = (face >= 0) & (d <= md * (1 - 1e-6))
    assert np.array_equal(fl[keep], face[keep]) and (fl[d > md * (1 + 1e-6)] == -1).all()
    assert (ql[fl < 0] == 0).all() and (bl[fl < 0] == 0).all()


@pytest.mark.gpu
def test_results_do_not_depend_on_the_batch():
    ch = _fixture("humanoid72")
    dc = ms.DeviceCharacter(ch, 0)
    B, N = 4099, 64
    xs, ps = _instances(ch, 8, 51, N)
    idx = np.arange(B) % 8
    xd = _dev(xs)[torch.from_numpy(idx).cuda()]
    pd = _dev(ps)[torch.from_numpy(idx).cuda()] + 0.01 * torch.arange(B, device="cuda", dtype=torch.float32)[:, None, None]
    full = _device_run(dc, xd, pd)
    for b in (0, 3, 2050, B - 1):
        for size in (1, 7):
            lo = min(b, B - size)
            sl = slice(lo, lo + size)
            part = _device_run(dc, xd[sl].contiguous(), pd[sl].contiguous())
            assert all(torch.equal(u[b - lo], w[b]) for u, w in zip(part, full)), (b, size)
    sub = [0, 2050, B - 1]
    _check(ch.skinning.faces, xd[sub].cpu().numpy(), pd[sub].cpu().numpy(), *(u[sub].cpu().numpy() for u in full), "B=4099")


@pytest.mark.gpu
def test_refit_in_several_slices_meets_the_bounds():
    """bodyhands300's tree takes 446 KB of boxes per instance, so 1300 instances need three slices of the 256 MiB scratch."""
    ch = _fixture("bodyhands300")
    dc = ms.DeviceCharacter(ch, 0)
    B, N, V = 1300, 32, ch.skinning.num_vertices
    nodes = 2 * -(-ch.skinning.faces.shape[0] // LEAF_FACES) - 1
    assert B * nodes * 24 > 2 * (256 << 20)
    xs, ps = _instances(ch, 4, 61, N)
    idx = torch.from_numpy(np.arange(B) % 4).cuda()
    gen = torch.Generator(device="cuda").manual_seed(62)
    xd = _dev(xs)[idx] + 0.05 * torch.randn(B, V, 3, device="cuda", generator=gen)
    pd = _dev(ps)[idx]
    full = _device_run(dc, xd, pd)
    sub = [0, 600, 601, 1203, B - 1]
    _check(ch.skinning.faces, xd[sub].cpu().numpy(), pd[sub].cpu().numpy(), *(u[sub].cpu().numpy() for u in full), "slices")
    alone = _device_run(dc, xd[sub].contiguous(), pd[sub].contiguous())
    assert all(torch.equal(u, w[sub]) for u, w in zip(alone, full))


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_drops_and_clones_the_tree():
    ch = _fixture("edges")
    sk = ch.skinning
    V, F = sk.num_vertices, sk.faces.shape[0]
    bare = mc.Character(ch.parents, ch.offsets, ch.prerot, ch.num_params, ch.pt_outer, ch.pt_inner, ch.pt_vals, ch.pt_offsets, [], "bare")
    dc = ms.DeviceCharacter(bare, 0)
    x, p = _instances(ch, 2, 91, 16)
    xd, pd = _dev(x), _dev(p)
    q, bary = torch.empty(2, p.shape[1], 3, device="cuda"), torch.empty(2, p.shape[1], 3, device="cuda")
    face = torch.empty(2, p.shape[1], dtype=torch.int32, device="cuda")
    ptrs = [xd.data_ptr(), pd.data_ptr(), q.data_ptr(), face.data_ptr(), bary.data_ptr()]
    N = p.shape[1]

    def call(B=2, n=N, md=float("inf"), ptr=ptrs, h=None):
        return dc._L.mb2_character_closest_points_on_mesh_device(dc._h if h is None else h, B, n, ms.C.c_void_p(ptr[0]), ms.C.c_void_p(ptr[1]), md,
                                                                  ms.C.c_void_p(ptr[2]), ms.C.c_void_p(ptr[3]), ms.C.c_void_p(ptr[4]), None)

    def err():
        return dc._L.mb2_last_error().decode()

    assert call() == 1 and "no mesh faces" in err()
    assert dc._L.mb2_character_set_mesh_tree(dc._h, V, sk.rest_vertices.ctypes.data_as(ms._fp)) == 1 and "no faces" in err()
    dc.set_skinning(sk)
    assert dc.mesh_tree_error is None
    ref = _np(_device_run(dc, xd, pd))
    for kw, msg in (({"B": -1}, "negative"), ({"n": -1}, "negative"), ({"md": float("nan")}, "max_dist"), ({"md": -1.0}, "max_dist")):
        assert call(**kw) == 1 and msg in err(), (kw, err())
    for k in range(5):
        bad = list(ptrs); bad[k] = 0
        assert call(ptr=bad) == 1 and "null" in err(), k
    host = np.zeros((2, N, 3), np.float32)
    bad = list(ptrs); bad[2] = host.ctypes.data
    assert call(ptr=bad) == 1 and "device memory" in err()
    assert call(B=0, ptr=[0] * 5) == 0 and call(n=0, ptr=[0] * 5) == 0  # nothing to do
    # a rejected tree keeps the earlier one
    nan = np.ascontiguousarray(sk.rest_vertices.copy()); nan[2, 1] = np.nan
    assert dc._L.mb2_character_set_mesh_tree(dc._h, V, nan.ctypes.data_as(ms._fp)) == 1 and "not finite" in err()
    assert dc._L.mb2_character_set_mesh_tree(dc._h, V + 1, sk.rest_vertices.ctypes.data_as(ms._fp)) == 1 and "differs" in err()
    assert dc._L.mb2_character_set_mesh_tree(dc._h, V, None) == 1 and "null" in err()
    assert all(np.array_equal(u, w) for u, w in zip(_np(_device_run(dc, xd, pd)), ref))
    # the clone computes the same bits with the tree it copied
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        face.fill_(-7)
        assert call(h=clone) == 0
        torch.cuda.synchronize()
        assert np.array_equal(face.cpu().numpy(), ref[1]) and np.array_equal(q.cpu().numpy(), ref[0]) and np.array_equal(bary.cpu().numpy(), ref[2])
    finally:
        dc._L.mb2_character_destroy(clone)
    # replacing the faces drops the tree; removing the tree too
    dc._check(dc._L.mb2_character_set_mesh_faces(dc._h, V, F, sk.faces.ctypes.data_as(ms._ip)))
    assert call() == 1 and "no mesh tree" in err()
    dc.set_mesh_tree(sk.rest_vertices)
    assert call() == 0
    dc.set_mesh_tree(None)
    assert call() == 1 and "no mesh tree" in err()


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_streams_and_errors():
    from momentum_b200 import torch_skeleton as tsk

    ch = _fixture("humanoid72")
    faces, V = ch.skinning.faces, ch.skinning.num_vertices
    dev = torch.device("cuda", 0)
    x, p = _instances(ch, 3, 71, 40)
    xd, pd = _dev(x), _dev(p)
    ref = _device_run(ms.DeviceCharacter(ch, 0), xd, pd)
    valid, q, face, bary = tsk.find_closest_points_on_mesh(ch, pd, xd)
    assert valid.dtype == torch.bool and q.dtype == torch.float32 and face.dtype == torch.int32 and bary.dtype == torch.float32
    assert q.shape == (3, p.shape[1], 3) and face.shape == (3, p.shape[1]) and valid.shape == face.shape
    assert torch.equal(q, ref[0]) and torch.equal(face, ref[1]) and torch.equal(bary, ref[2]) and torch.equal(valid, ref[1] >= 0)
    # float64 in: float64 out, the same values; outputs carry no gradient
    x64 = xd.double().requires_grad_(True)
    p64 = pd.double().requires_grad_(True)
    v2, q2, f2, b2 = tsk.find_closest_points_on_mesh(ch, p64, x64)
    assert q2.dtype == torch.float64 and b2.dtype == torch.float64 and f2.dtype == torch.int32
    assert not q2.requires_grad and not b2.requires_grad and torch.equal(q2.float(), q) and torch.equal(f2, face)
    # broadcasting: unbatched points against batched vertices, and the reverse; unbatched both
    one = tsk.find_closest_points_on_mesh(ch, pd[1], xd)
    assert one[2].shape == (3, p.shape[1]) and torch.equal(one[2][1], face[1])
    rev = tsk.find_closest_points_on_mesh(ch, pd, xd[1])
    assert torch.equal(rev[2][1], face[1])
    single = tsk.find_closest_points_on_mesh(ch, pd[2], xd[2])
    assert single[2].shape == (p.shape[1],) and torch.equal(single[2], face[2]) and torch.equal(single[0], valid[2])
    # a side stream
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        side = tsk.find_closest_points_on_mesh(ch, pd, xd)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(side[2], face) and torch.equal(side[1], q)
    # a DeviceCharacter
    dc = ms.DeviceCharacter(ch, 0)
    assert torch.equal(tsk.find_closest_points_on_mesh(dc, pd, xd)[2], face)
    # max_dist
    md = float(torch.linalg.norm(q - pd, dim=-1)[valid].median())
    lim = tsk.find_closest_points_on_mesh(ch, pd, xd, max_dist=md)
    assert torch.equal(lim[2], _device_run(dc, xd, pd, md)[1])
    # errors
    for args, msg in (((pd, torch.zeros(V + 1, 3, device=dev)), "vertices_target must be"), ((pd[..., :2], xd), "points_source must be"),
                      ((pd[:2], xd), "batches"), ((pd.cpu(), xd), "CUDA")):
        with pytest.raises(ValueError, match=msg):
            tsk.find_closest_points_on_mesh(ch, *args)
    with pytest.raises(ValueError, match="max_dist"):
        tsk.find_closest_points_on_mesh(ch, pd, xd, max_dist=-1.0)
    plain = copy.copy(ch)
    plain.skinning = mc.synthetic_skinning(ch, 3, 0)
    with pytest.raises(ValueError, match="no mesh faces"):
        tsk.find_closest_points_on_mesh(plain, pd, torch.zeros(plain.skinning.num_vertices, 3, device=dev))
    # a mesh without faces has no tree; a rejected tree keeps the earlier one
    empty = copy.copy(_fixture("chain3"))
    sk = empty.skinning
    empty.skinning = mc.Skinning(sk.rest_vertices, sk.skin_index, sk.skin_weight, sk.inverse_bind_pose, np.zeros((0, 3), np.int32))
    with pytest.raises(ValueError, match="no closest-point tree"):
        tsk.find_closest_points_on_mesh(empty, torch.zeros(2, 3, device=dev), torch.zeros(sk.num_vertices, 3, device=dev))
    nan = ch.skinning.rest_vertices.copy(); nan[0, 0] = np.nan
    with pytest.raises(ms.MomentumB200Error, match="not finite"):
        dc.set_mesh_tree(nan)
    assert torch.equal(tsk.find_closest_points_on_mesh(dc, pd, xd)[2], face)
    # replacing character.skinning gives a new handle: the new faces are searched
    ch2 = copy.copy(_fixture("chain3"))
    sk2 = ch2.skinning
    xc, pc = _instances(ch2, 1, 73, 32)
    before = tsk.find_closest_points_on_mesh(ch2, _dev(pc), _dev(xc))
    half = sk2.faces[::2].copy()
    ch2.skinning = mc.Skinning(sk2.rest_vertices, sk2.skin_index, sk2.skin_weight, sk2.inverse_bind_pose, half)
    after = tsk.find_closest_points_on_mesh(ch2, _dev(pc), _dev(xc))
    _check(half, xc, pc, *(u.cpu().numpy() for u in after[1:]), "new skinning")
    assert not torch.equal(before[2], after[2])


@pytest.mark.gpu
def test_fitting_composition_matches_finite_differences_of_the_distance():
    """skin_points at a pose -> closest points of scan-like points (under no_grad) -> sum |p - sum_k b_k x[face_k]|^2 -> backward to the
    model parameters through skin_points and forward kinematics, against float64 central differences of the true squared point-to-mesh
    distance. Queries whose closest face is unique by a margin."""
    from momentum_b200 import torch_skeleton as tsk

    ch = _fixture("chain3")
    faces = ch.skinning.faces
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(12)
    theta = rng.uniform(-0.3, 0.3, (1, ch.num_params))

    def mesh64(th):
        t, q, s = mc.forward_kinematics(ch, th)
        return mc.skin_points(ch, np.concatenate([t, q, s[..., None]], -1))[0]

    x0 = mesh64(theta)
    p = _queries(ch, x0.astype(np.float32), 600, 13, scan_only=True).astype(np.float64)
    D, f64, gap, _ = _closest64(faces, x0, p)
    p = p[gap > 0.02][:40]
    assert len(p) >= 20

    def loss64(th):
        return float((_closest64(faces, mesh64(th), p)[0] ** 2).sum())

    th = torch.from_numpy(theta).to(dev).requires_grad_(True)
    x = tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, th))
    pd = torch.from_numpy(p).to(dev).requires_grad_(True)
    with torch.no_grad():
        valid, _, face, bary = tsk.find_closest_points_on_mesh(ch, pd, x)
    assert valid.all()
    tri = torch.from_numpy(faces.astype(np.int64)).to(dev)[face.long()]  # [N, 3]
    qd = (bary.unsqueeze(-1) * x[0][tri]).sum(-2)
    loss = ((pd - qd) ** 2).sum()
    loss.backward()
    assert abs(loss.item() - loss64(theta)) <= 1e-4 * max(1.0, loss64(theta))
    g = th.grad.cpu().numpy()
    h = 1e-5
    for i in range(ch.num_params):
        d = np.zeros_like(theta); d[0, i] = h
        fd = (loss64(theta + d) - loss64(theta - d)) / (2 * h)
        assert abs(fd - g[0, i]) <= 2e-3 * max(abs(fd), 1.0), (i, fd, g[0, i])
    # with respect to p: 2 (p - q)
    assert np.abs(pd.grad.cpu().numpy() - 2 * (p - _closest64(faces, x0, p)[3])).max() <= 1e-3
