"""find_closest_points (the closest target point of each query point, with the normal-compatible variant) on the device, over a tree built
per call, against the linear scan that defines it and a float64 reference.

The result for query p is the target j with the smallest (d2_j, j) among the candidates: finite t_j with finite d2_j <= max_dist^2 and,
in the normal variant, dot(n_p, n_j) >= max_normal_dot, where d2 and the dot are explicit fmaf chains. So it must not depend on the
tree: the emulated traversal equals the emulated linear scan bit for bit, and the device equals the emulated scan bit for bit. Against
float64 (a numpy brute force), with u = 2^-24 and S the largest coordinate magnitude of the instance's targets and the query, the chosen
target's float64 distance is within K u S of the float64 minimum; K is pinned at about four times the worst value measured over the
fixtures below on the emulator and on an H100.
The self-checks show that the checks reject a prune on >=, a leaf that skips its last point, and a strict > normal test.
"""
import ctypes

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_vertex_normals import _tube

EPS32 = 2.0 ** -24
LEAF_POINTS, SORT_TILE, NON_FINITE_CODE = 8, 1024, 1 << 30  # kLeafPoints, kSortTile, kMortonNonFinite (ik_types.h)

# worst measured ratio (float64 distance of the chosen target minus the float64 minimum, in u S) over these fixtures, near-tie midpoint
# queries included, on the emulator / on an H100 80GB HBM3 at a 700 W power limit: 0.0083 / 0.0083 (both on "random"); K is about four
# times the larger
K_D = 0.035


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _unit(v):
    return (v / np.maximum(np.linalg.norm(v, axis=-1, keepdims=True), 1e-30)).astype(np.float32)


def _random(seed, M):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(M, 3)).astype(np.float32), _unit(rng.normal(size=(M, 3)))


def _tube_targets(name):
    make, rings, segments = {"humanoid72": (lambda: mc.humanoid72()[0], 12, 12), "bodyhands300": (lambda: mc.bodyhands300()[0], 8, 8)}[name]
    ch = _tube(make, rings, segments, 2, name)
    x = ch.skinning.rest_vertices.astype(np.float32)
    return x, mc.vertex_normals(ch.skinning.faces, x).astype(np.float32)


def _scan(far=False):
    ch = _tube(lambda: mc.humanoid72()[0], 12, 12, 2, "humanoid72", far=far)
    return mc.synthetic_scan(ch, 20000, seed=5)


def _lattice():
    """An integer lattice: many queries at exactly equal distances from several targets, so the index decides."""
    g = np.stack(np.meshgrid(*[np.arange(-6, 7)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    rng = np.random.default_rng(3)
    g = g[rng.permutation(len(g))]
    n = np.zeros_like(g); n[:, 2] = 1.0
    n[::3] = (0, 0, -1)
    return g, n


def _duplicates():
    """Exact duplicates spread over the cloud, several per point, indices shuffled."""
    rng = np.random.default_rng(4)
    base = rng.normal(size=(300, 3)).astype(np.float32)
    x = np.concatenate([base, base, base[:100], base[::7]])
    perm = rng.permutation(len(x))
    n = _unit(rng.normal(size=(len(x), 3)))
    return x[perm], n


def _underflow_cluster():
    """A 4 x 4 x 4 lattice of spacing 1e-24 (all pairwise d2 underflow to exactly 0), indexed in decreasing Morton order: every target is
    a candidate at d2 = 0, so the lowest index (the last in sorted order, in the leaf the traversal enters last) must win. Points with
    equal coordinates have equal codes and a stable sort keeps the lower index first, so among exact duplicates the lower index is always
    visited first; d2 ties at 0 between distinct points are what let a prune on >= go wrong."""
    g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), -1).reshape(-1, 3)
    code = np.zeros(len(g), np.int64)
    for bit in range(2):
        for k in range(3):
            code |= ((g[:, k] >> bit) & 1) << (3 * bit + 2 - k)
    x = (g[np.argsort(-code, kind="stable")] * 1e-24).astype(np.float32)
    n = np.zeros_like(x); n[:, 2] = 1.0
    return x, n


def _flat(seed=6):
    x, n = _random(seed, 500)
    x[:, 1] = 2.5
    return x, n


CLOUDS = {
    "random": lambda: _random(1, 5000),
    "humanoid72": lambda: _tube_targets("humanoid72"),
    "bodyhands300": lambda: _tube_targets("bodyhands300"),
    "scan": lambda: _scan(),
    "random_far": lambda: tuple([_random(1, 5000)[0] + np.float32(100.0), _random(1, 5000)[1]]),
    "scan_far": lambda: _scan(far=True),
    "lattice": _lattice,
    "duplicates": _duplicates,
    "underflow": _underflow_cluster,
    "flat": _flat,
}
_cache = {}


def _cloud(name):
    if name not in _cache:
        _cache[name] = CLOUDS[name]()
    return _cache[name]


def _queries(x, n, seed):
    """[n, 3] queries near cloud x: targets exactly, targets jittered, uniform in the inflated box, a few far points and non-finite ones;
    with normals (unit, random sign flips)."""
    rng = np.random.default_rng(seed)
    fin = x[np.isfinite(x).all(1)].astype(np.float64)
    lo, hi = fin.min(0), fin.max(0)
    ext = np.maximum(hi - lo, 1e-30)
    k = n // 4
    on = fin[rng.integers(0, len(fin), k)]
    jit = fin[rng.integers(0, len(fin), k)] + rng.normal(scale=0.01, size=(k, 3)) * ext
    box = rng.uniform(lo - 0.2 * ext, hi + 0.2 * ext, (n - 2 * k - 6, 3))
    far = 0.5 * (lo + hi) + 1e3 * _unit(rng.normal(size=(3, 3)))
    bad = np.array([(np.nan, 0, 0), (np.inf, 0, 0), (0, -np.inf, 1)])
    q = np.concatenate([on, jit, box, far, bad]).astype(np.float32)
    return q, _unit(rng.normal(size=(len(q), 3)))


def _midpoints(x, n, seed):
    """[n, 3] near-tie queries: the midpoints of n random targets and their nearest neighbours, where rounding decides"""
    from scipy.spatial import cKDTree

    rng = np.random.default_rng(seed)
    x64 = x.astype(np.float64)
    i = rng.integers(0, len(x), n)
    _, j = cKDTree(x64).query(x64[i], k=2)
    return (0.5 * (x64[i] + x64[j[:, 1]])).astype(np.float32)


_i32, _f32, _p = ctypes.c_int32, ctypes.c_float, ctypes.c_void_p
# the entries of tests/emu/emu_closest_cloud.cu, declared here next to the only tests that call them
_SIGNATURES = {
    "emu_cloud_tree": [_i32] + [_p] * 5,
    "emu_closest_cloud": [_i32] * 4 + [_p] * 4 + [_f32, _f32, _i32] + [_p] * 3,
}


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    for name, argtypes in _SIGNATURES.items():
        getattr(L, name).argtypes = argtypes
    return L


def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def _emu_tree(L, x):
    M = len(x)
    P = 1
    while P * LEAF_POINTS < M:
        P *= 2
    codes = np.zeros(max(M, 1), np.uint32)
    perm = np.zeros(max(M, 1), np.int32)
    boxes = np.zeros((2 * P - 1, 6), np.float32)
    sizes = np.zeros(2, np.int32)
    xx = _c(x.reshape(-1, 3), np.float32)
    assert L.emu_cloud_tree(M, xx.ctypes.data, codes.ctypes.data, perm.ctypes.data, boxes.ctypes.data, sizes.ctypes.data) == 0
    assert sizes[0] == P
    return codes[:M], perm[:M], boxes, int(sizes[1])


def _emu_run(L, p, x, pn=None, xn=None, max_dist=np.inf, max_normal_dot=0.0, mode=0):
    """p [B, N, 3], x [B or 1, M, 3] (batched when B > 1 and x has B rows); returns (points, normals or None, index)."""
    p = _c(p, np.float32)
    x = _c(x, np.float32)
    B, N = p.shape[:2]
    M = x.shape[1]
    batched = x.shape[0] == B and B > 1
    normals = pn is not None
    pn = _c(pn, np.float32) if normals else None
    xn = _c(xn, np.float32) if normals else None
    q = np.zeros((B, N, 3), np.float32)
    qn = np.zeros((B, N, 3), np.float32) if normals else None
    idx = np.zeros((B, N), np.int32)
    ptr = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    rc = L.emu_closest_cloud(B, N, M, int(batched), ptr(p), ptr(pn), ptr(x), ptr(xn), float(max_dist), float(max_normal_dot), mode, ptr(q), ptr(qn),
                             ptr(idx))
    assert rc == 0, L.emu_last_error()
    return q, qn, idx


def _same(a, b):
    """bitwise equality of two result tuples"""
    return all((u is None and v is None) or (u.shape == v.shape and np.array_equal(u.view(np.uint32) if u.dtype == np.float32 else u,
                                                                                      v.view(np.uint32) if v.dtype == np.float32 else v))
               for u, v in zip(a, b))


def _ratio(x, p, idx):
    """Worst (|t_chosen - p| - min_j |t_j - p|) / (u S) in float64 over the valid queries, and whether every finite query found one."""
    x64 = x.astype(np.float64)
    worst = 0.0
    fin_t = np.isfinite(x64).all(1)
    for i in range(len(p)):
        if not np.isfinite(p[i]).all():
            assert idx[i] == -1
            continue
        d = np.sqrt(((x64[fin_t] - p[i].astype(np.float64)) ** 2).sum(1))
        assert idx[i] >= 0
        dc = np.sqrt(((x64[idx[i]] - p[i].astype(np.float64)) ** 2).sum())
        S = max(np.abs(x64[fin_t]).max(), np.abs(p[i]).max())
        worst = max(worst, (dc - d.min()) / (EPS32 * S))
    return worst


# ---- CPU: the emulated build ------------------------------------------------------------------------------------------------------
BUILDS = {
    "random_5000": lambda: _random(1, 5000)[0],
    "one": lambda: np.array([[1.0, 2.0, 3.0]], np.float32),
    "all_equal": lambda: np.full((100, 3), 0.75, np.float32),
    "flat_axis": lambda: _flat()[0],
    "M_13": lambda: _random(2, 13)[0],
    "M_0": lambda: np.zeros((0, 3), np.float32),
    "non_finite": lambda: np.concatenate([_random(3, 2100)[0], np.array([(np.nan, 0, 0), (0, np.inf, 0), (1, 1, -np.inf)] * 5, np.float32)])[
        np.random.default_rng(0).permutation(2115)],
    "lattice": lambda: _lattice()[0],
}


@pytest.mark.parametrize("name", list(BUILDS))
def test_emulated_build_sorts_by_morton_code_and_boxes_the_leaves(emu, name):
    x = BUILDS[name]()
    M = len(x)
    codes, perm, boxes, leaves = _emu_tree(emu, x)
    assert leaves == (M + LEAF_POINTS - 1) // LEAF_POINTS
    np.testing.assert_array_equal(perm, np.argsort(codes, kind="stable"))
    assert np.array_equal(np.sort(perm), np.arange(M))
    finite = np.isfinite(x).all(1)
    assert np.all(codes[~finite] == NON_FINITE_CODE) and np.all(codes[finite] < NON_FINITE_CODE)
    assert np.all(finite[perm][: finite.sum()])  # non-finite points come last
    if name == "flat_axis":  # a zero extent gives 0 on that axis: the y bits (1, 4, 7, ...) of every code are clear
        ymask = sum(1 << (3 * b + 1) for b in range(10))
        assert np.all(codes & ymask == 0)
    if name == "all_equal":
        assert np.all(codes == 0)
    P = boxes.shape[0] // 2 + 1
    xs = x[perm]
    for l in range(P):
        b = boxes[P - 1 + l]
        pts = xs[l * LEAF_POINTS: (l + 1) * LEAF_POINTS]
        if len(pts) == 0:
            assert np.all(b[:3] == np.inf) and np.all(b[3:] == -np.inf), "padding leaves are empty"
            continue
        with np.errstate(invalid="ignore"):
            lo, hi = np.nanmin(np.where(np.isnan(pts), np.inf, pts), 0), np.nanmax(np.where(np.isnan(pts), -np.inf, pts), 0)
        np.testing.assert_array_equal(b, np.concatenate([lo, hi]).astype(np.float32))
    for n in range(P - 1):
        c0, c1 = boxes[2 * n + 1], boxes[2 * n + 2]
        np.testing.assert_array_equal(boxes[n], np.concatenate([np.minimum(c0[:3], c1[:3]), np.maximum(c0[3:], c1[3:])]))


# ---- CPU: tree independence ---------------------------------------------------------------------------------------------------------
N_CPU = 400


@pytest.mark.parametrize("name", list(CLOUDS))
def test_emulated_traversal_equals_the_linear_scan(emu, name):
    x, xn = _cloud(name)
    p, pn = _queries(x, N_CPU, 11)
    for args in ({}, {"pn": pn[None], "xn": xn[None], "max_normal_dot": 0.0}, {"pn": pn[None], "xn": xn[None], "max_normal_dot": -0.3},
                 {"max_dist": 0.05 * float(np.abs(x).max())}):
        tr = _emu_run(emu, p[None], x[None], mode=0, **args)
        sc = _emu_run(emu, p[None], x[None], mode=1, **args)
        assert _same(tr, sc), (name, args.keys())


def test_emulated_traversal_equals_the_scan_in_2d_and_batched(emu):
    rng = np.random.default_rng(9)
    x2 = np.concatenate([rng.normal(size=(3, 700, 2)), np.zeros((3, 700, 1))], -1).astype(np.float32)  # 2-D, padded with z = 0
    p2 = np.concatenate([rng.normal(size=(3, 90, 2)), np.zeros((3, 90, 1))], -1).astype(np.float32)
    assert _same(_emu_run(emu, p2, x2), _emu_run(emu, p2, x2, mode=1))
    assert _same(_emu_run(emu, p2, x2[:1]), _emu_run(emu, p2, x2[:1], mode=1))  # one shared target


@pytest.mark.parametrize("name", ["random", "scan", "random_far", "scan_far", "humanoid72"])
def test_emulator_meets_the_float64_bound(emu, name):
    x, _ = _cloud(name)
    p = np.concatenate([_queries(x, N_CPU, 12)[0], _midpoints(x, N_CPU, 5)])
    _, _, idx = _emu_run(emu, p[None], x[None])
    assert _ratio(x, p, idx[0]) <= K_D


# ---- CPU: edges ---------------------------------------------------------------------------------------------------------------------
def test_edges(emu):
    x = np.array([(0, 0, 0), (3, 0, 0), (0, 4, 0), (0, 0, 0)], np.float32)
    p = np.array([[(0, 0, 0), (1.5, 0, 0)]], np.float32)
    # max_dist = 0 matches coincident points, the lower of two duplicates
    _, _, idx = _emu_run(emu, p[:, :1], x[None], max_dist=0.0)
    assert idx[0, 0] == 0
    # a target at exactly max_dist (d2 == max_dist^2 in float) is valid; the next float up is not
    o = np.zeros((1, 1, 3), np.float32)
    for r in (np.float32(5.0), np.float32(0.75), np.float32(1e-3)):
        at = np.array([[(r, 0, 0)]], np.float32)
        up = np.array([[(np.nextafter(r, np.float32(np.inf)), 0, 0)]], np.float32)
        assert np.float32(r * r) < np.float32(up[0, 0, 0] * up[0, 0, 0])
        assert _emu_run(emu, o, at, max_dist=r)[2][0, 0] == 0
        assert _emu_run(emu, o, up, max_dist=r)[2][0, 0] == -1
    # the normal test: a dot exactly equal to max_normal_dot is accepted; all incompatible gives -1 and zeros
    n_up = np.array([[(0, 0, 1)] * 4], np.float32)
    qn = np.array([[(0, 1, 0), (0, 0, 1)]], np.float32)
    pts, nrm, idx = _emu_run(emu, p, x[None], pn=qn, xn=n_up, max_normal_dot=0.0)
    assert idx[0, 0] == 0  # dot 0 == 0
    pts, nrm, idx = _emu_run(emu, p, x[None], pn=-qn, xn=n_up, max_normal_dot=0.5)
    assert np.all(idx == -1) and np.all(pts == 0) and np.all(nrm == 0)
    # non-finite queries are invalid; non-finite targets and target normals are never chosen; a NaN query normal matches nothing
    xb = np.array([(np.nan, 0, 0), (0, np.inf, 0), (1, 1, 1)], np.float32)
    pb = np.array([[(np.nan, 0, 0), (0, 0, 0), (np.inf, 1, 1)]], np.float32)
    _, _, idx = _emu_run(emu, pb, xb[None])
    assert list(idx[0]) == [-1, 2, -1]
    nb = np.array([[(np.nan, 0, 1), (0, 0, 1), (0, 0, 1)]], np.float32)
    _, _, idx = _emu_run(emu, np.array([[(1, 1, 0.9)]], np.float32), xb[None], pn=np.array([[(0, 0, 1)]], np.float32), xn=nb, max_normal_dot=-1.0)
    assert idx[0, 0] == 2
    xs = np.array([(1, 1, 1), (1, 1, 1.5)], np.float32)
    _, _, idx = _emu_run(emu, np.array([[(1, 1, 1)]], np.float32), xs[None], pn=np.array([[(0, 0, 1)]], np.float32),
                         xn=np.array([[(np.nan, 0, 1), (0, 0, 1)]], np.float32), max_normal_dot=-1.0)
    assert idx[0, 0] == 1  # a NaN target normal fails the test even at max_normal_dot = -1
    _, _, idx = _emu_run(emu, np.array([[(1, 1, 1)]], np.float32), xs[None], pn=np.array([[(np.nan, 0, 1)]], np.float32),
                         xn=np.array([[(0, 0, 1), (0, 0, 1)]], np.float32), max_normal_dot=-1.0)
    assert idx[0, 0] == -1
    # M = 0: every query -1 and zeros
    pts, _, idx = _emu_run(emu, p, np.zeros((1, 0, 3), np.float32))
    assert np.all(idx == -1) and np.all(pts == 0)


def test_checks_reject_wrong_variants(emu):
    # a prune on >=: the underflow cluster, queries on its points
    x, xn = _cloud("underflow")
    p = x[:64][None]
    assert _same(_emu_run(emu, p, x[None]), _emu_run(emu, p, x[None], mode=1))
    assert not _same(_emu_run(emu, p, x[None], mode=2), _emu_run(emu, p, x[None], mode=1))
    assert np.all(_emu_run(emu, p, x[None], mode=1)[2] == 0)
    # a leaf that drops its last point
    x, _ = _cloud("random")
    q, _ = _queries(x, N_CPU, 11)
    assert not _same(_emu_run(emu, q[None], x[None], mode=3), _emu_run(emu, q[None], x[None], mode=1))
    # a strict > normal test: the lattice's normals are +-z, queries with normal x meet dot == 0 == max_normal_dot
    x, xn = _cloud("lattice")
    q = (x[:50] + np.float32(0.25))[None]
    qn = np.tile(np.array([(1, 0, 0)], np.float32), (1, 50, 1))
    good = _emu_run(emu, q, x[None], pn=qn, xn=xn[None], max_normal_dot=0.0, mode=1)
    assert np.all(good[2] >= 0)
    assert not _same(_emu_run(emu, q, x[None], pn=qn, xn=xn[None], max_normal_dot=0.0, mode=4), good)


def test_synthetic_scan_is_seeded_and_on_the_posed_surface():
    ch = _tube(lambda: mc.humanoid72()[0], 12, 12, 2, "humanoid72")
    a, na = mc.synthetic_scan(ch, 500, seed=3)
    b, nb = mc.synthetic_scan(ch, 500, seed=3)
    assert a.dtype == np.float32 and a.shape == (500, 3) and np.array_equal(a, b) and np.array_equal(na, nb)
    np.testing.assert_allclose(np.linalg.norm(na, axis=1), 1.0, atol=1e-5)
    c, _ = mc.synthetic_scan(ch, 500, seed=3, noise=0.0)
    x = ch.skinning.rest_vertices
    assert np.sqrt(((c[:, None] - x[None]) ** 2).sum(-1)).min(1).max() < 0.5 * np.abs(x).max()


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    monkeypatch.setattr(ms, "closest_points_device", lambda *a, **k: pytest.fail("library called"))
    with pytest.raises(ValueError, match="CUDA tensors"):
        tsk.find_closest_points(torch.zeros(4, 3), torch.zeros(5, 3))
    with pytest.raises(TypeError, match="missing"):
        tsk.find_closest_points(torch.zeros(4, 3))


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _device_run(p, x, pn=None, xn=None, max_dist=np.inf, max_normal_dot=0.0, batched=None):
    """The C-ABI on host arrays p [B, N, 3], x [B or 1, M, 3]; returns numpy (points, normals or None, index)."""
    B, N = p.shape[:2]
    M = x.shape[1]
    batched = x.shape[0] == B and B > 1 if batched is None else batched
    pd, xd = _dev(_c(p, np.float32)), _dev(_c(x, np.float32))
    pnd = _dev(_c(pn, np.float32)) if pn is not None else None
    xnd = _dev(_c(xn, np.float32)) if xn is not None else None
    q = torch.empty(B, N, 3, device="cuda:0")
    qn = torch.empty(B, N, 3, device="cuda:0") if pn is not None else None
    idx = torch.empty(B, N, dtype=torch.int32, device="cuda:0")
    ptr = lambda t: 0 if t is None or t.numel() == 0 else t.data_ptr()  # noqa: E731
    ms.closest_points_device(0, B, N, M, batched, ptr(pd), ptr(pnd), ptr(xd), ptr(xnd), max_dist, max_normal_dot, ptr(q), ptr(qn), ptr(idx),
                             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return q.cpu().numpy(), None if qn is None else qn.cpu().numpy(), idx.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CLOUDS))
def test_device_equals_the_emulated_scan(emu, name):
    x, xn = _cloud(name)
    p, pn = _queries(x, 2000, 21)
    for args in ({}, {"pn": pn[None], "xn": xn[None], "max_normal_dot": 0.0}, {"max_dist": 0.05 * float(np.abs(x).max())}):
        assert _same(_device_run(p[None], x[None], **args), _emu_run(emu, p[None], x[None], mode=1, **args)), (name, args.keys())
    if name != "underflow":  # there every d2 underflows to 0 in float, so the index decides: the bound is for normal-range distances
        pm = _midpoints(x, 300, 5)
        _, _, idx = _device_run(pm[None], x[None])
        assert _ratio(x, pm, idx[0]) <= K_D


@pytest.mark.gpu
def test_device_batched_and_shared_targets_in_2d_and_3d(emu):
    from momentum_b200 import torch_skeleton as tsk

    rng = np.random.default_rng(31)
    B, N, M = 5, 300, 3000
    x = rng.normal(size=(B, M, 3)).astype(np.float32)
    xn = _unit(rng.normal(size=(B, M, 3)))
    p = rng.normal(size=(B, N, 3)).astype(np.float32)
    pn = _unit(rng.normal(size=(B, N, 3)))
    for xx, xxn in ((x, xn), (x[:1], xn[:1])):
        assert _same(_device_run(p, xx), _emu_run(emu, p, xx, mode=1))
        assert _same(_device_run(p, xx, pn, xxn, max_normal_dot=0.2), _emu_run(emu, p, xx, pn, xxn, max_normal_dot=0.2, mode=1))
    # 2-D through the torch wrapper: the same bits as the emulated scan with z = 0
    x2, p2 = x[..., :2].copy(), p[..., :2].copy()
    pts, idx, valid = tsk.find_closest_points(_dev(p2), _dev(x2))
    pad = lambda a: np.concatenate([a, np.zeros(a.shape[:-1] + (1,), np.float32)], -1)  # noqa: E731
    q, _, ie = _emu_run(emu, pad(p2), pad(x2), mode=1)
    assert np.array_equal(idx.cpu().numpy(), ie) and np.array_equal(pts.cpu().numpy(), q[..., :2]) and bool(valid.all())
    pts, idx, valid = tsk.find_closest_points(_dev(p2), _dev(x2[0]))
    q, _, ie = _emu_run(emu, pad(p2), pad(x2[:1]), mode=1)
    assert np.array_equal(idx.cpu().numpy(), ie) and np.array_equal(pts.cpu().numpy(), q[..., :2])


@pytest.mark.gpu
def test_results_do_not_depend_on_the_batch():
    rng = np.random.default_rng(41)
    B, N, M = 4099, 16, 200
    x = rng.normal(size=(B, M, 3)).astype(np.float32)
    xn = _unit(rng.normal(size=(B, M, 3)))
    p = rng.normal(size=(B, N, 3)).astype(np.float32)
    pn = _unit(rng.normal(size=(B, N, 3)))
    full = _device_run(p, x, pn, xn, max_normal_dot=0.0)
    shared = _device_run(p, x[:1], pn, xn[:1], max_normal_dot=0.0)
    for b in (0, 1, 2048, 4098):
        alone = _device_run(p[b:b + 1], x[b:b + 1], pn[b:b + 1], xn[b:b + 1], max_normal_dot=0.0, batched=True)
        assert _same(alone, tuple(a[b:b + 1] for a in full))
        alone = _device_run(p[b:b + 1], x[:1], pn[b:b + 1], xn[:1], max_normal_dot=0.0)
        assert _same(alone, tuple(a[b:b + 1] for a in shared))


def _scratch_bytes(M, normals):
    tiles = (M + SORT_TILE - 1) // SORT_TILE
    P = 1
    while P * LEAF_POINTS < M:
        P *= 2
    return 4 * (tiles * 6 + 6 + 4 * M + tiles * 256 + 256 + (6 if normals else 3) * M + (2 * P - 1) * 6)


@pytest.mark.gpu
def test_build_in_several_slices_gives_the_same_bits(emu):
    M, N = 100_000, 32
    slice_ = (256 << 20) // _scratch_bytes(M, True)
    B = 2 * slice_ + 3  # three slices
    rng = np.random.default_rng(51)
    x = rng.normal(size=(B, M, 3)).astype(np.float32)
    xn = _unit(rng.normal(size=(B, M, 3)))
    p = rng.normal(size=(B, N, 3)).astype(np.float32)
    pn = _unit(rng.normal(size=(B, N, 3)))
    full = _device_run(p, x, pn, xn)
    for b in (0, slice_ - 1, slice_, 2 * slice_ - 1, 2 * slice_, B - 1):
        alone = _device_run(p[b:b + 1], x[b:b + 1], pn[b:b + 1], xn[b:b + 1], batched=True)
        assert _same(alone, tuple(a[b:b + 1] for a in full)), b
    for b in (slice_, B - 1):
        assert _same(tuple(a[b:b + 1] for a in full), _emu_run(emu, p[b:b + 1], x[b:b + 1], pn[b:b + 1], xn[b:b + 1], mode=1))


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_and_accepts_zero_sizes():
    dev = "cuda:0"
    p = torch.zeros(2, 4, 3, device=dev)
    x = torch.ones(2, 5, 3, device=dev)
    q = torch.empty(2, 4, 3, device=dev)
    qn = torch.empty(2, 4, 3, device=dev)
    idx = torch.empty(2, 4, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    P = lambda t: t.data_ptr()  # noqa: E731

    def call(*, device=0, B=2, N=4, M=5, batched=1, src=P(p), srcn=0, tgt=P(x), tgtn=0, md=float("inf"), mnd=0.0, out=P(q), outn=0, oi=P(idx)):
        return ms.closest_points_device(device, B, N, M, batched, src, srcn, tgt, tgtn, md, mnd, out, outn, oi, s)

    for kw, msg in (({"B": -1}, "must not be negative"), ({"N": -1}, "must not be negative"), ({"M": -1}, "must not be negative"),
                    ({"device": -1}, "device must not be negative"), ({"md": float("nan")}, "max_dist"), ({"md": -1.0}, "max_dist"),
                    ({"mnd": float("nan")}, "max_normal_dot"), ({"srcn": P(p)}, "both null or both set"),
                    ({"srcn": P(p), "tgtn": P(x)}, "out_normals"), ({"outn": P(qn)}, "out_normals"), ({"src": 0}, "null argument"),
                    ({"oi": 0}, "null argument"), ({"tgt": 0}, "null argument")):
        with pytest.raises(ms.MomentumB200Error, match=msg):
            call(**kw)
    host = np.zeros((2, 4, 3), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        call(src=host.ctypes.data)
    # zero sizes: B = 0 and N = 0 are no-ops (nulls allowed); M = 0 gives every query -1 and zeros
    call(B=0, src=0, tgt=0, out=0, oi=0)
    call(N=0, src=0, out=0, oi=0)
    q.fill_(7.0); qn.fill_(7.0); idx.fill_(7)
    call(M=0, tgt=0)
    call(M=0, tgt=0, srcn=P(p), outn=P(qn))
    torch.cuda.synchronize()
    assert bool((idx == -1).all()) and bool((q == 0).all()) and bool((qn == 0).all())


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_and_errors():
    from momentum_b200 import torch_skeleton as tsk

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(61)
    x = torch.from_numpy(rng.normal(size=(3, 50, 3))).to(dev)  # float64
    p = torch.from_numpy(rng.normal(size=(3, 20, 3))).to(dev).requires_grad_(True)
    n = torch.nn.functional.normalize(torch.from_numpy(rng.normal(size=(3, 50, 3))).to(dev), dim=-1)
    pn = torch.nn.functional.normalize(torch.from_numpy(rng.normal(size=(3, 20, 3))).to(dev), dim=-1)
    pts, idx, valid = tsk.find_closest_points(p, x)
    assert pts.shape == (3, 20, 3) and pts.dtype == torch.float64 and idx.dtype == torch.int32 and valid.dtype == torch.bool
    assert not pts.requires_grad and bool(valid.all())
    assert torch.equal(pts, torch.gather(x.float(), 1, idx.long().unsqueeze(-1).expand(-1, -1, 3)).double())  # computed in float32
    # broadcasting: an unbatched source against batched targets, and a batched source against one target
    a = tsk.find_closest_points(p[1], x)
    assert a[0].shape == (3, 20, 3) and torch.equal(a[1][1], idx[1])
    b = tsk.find_closest_points(p, x[1])
    assert b[0].shape == (3, 20, 3) and torch.equal(b[1][1], idx[1])
    c = tsk.find_closest_points(p[1], x[1])
    assert c[0].shape == (20, 3) and torch.equal(c[1], idx[1])
    # the normal variant, positional and by keyword; float32 in, float32 out
    r = tsk.find_closest_points(p.float(), pn.float(), x.float(), n.float(), max_normal_dot=0.1)
    assert len(r) == 4 and r[1].shape == (3, 20, 3) and r[0].dtype == torch.float32
    ok = r[3]
    dots = (pn.float() * r[1]).sum(-1)
    assert bool((dots[ok] >= 0.1 - 1e-6).all())
    r2 = tsk.find_closest_points(points_source=p.float(), normals_source=pn.float(), points_target=x.float(), normals_target=n.float(),
                                 max_normal_dot=0.1)
    assert all(torch.equal(u, v) for u, v in zip(r, r2))
    # max_dist
    _, idx_d, valid_d = tsk.find_closest_points(p, x, max_dist=0.2)
    d = (tsk.find_closest_points(p, x)[0] - p).norm(dim=-1)
    assert bool((d[valid_d] <= 0.2 + 1e-6).all()) and bool((d[~valid_d] >= 0.2 - 1e-6).all()) and bool(valid_d.any())
    assert bool((idx_d[~valid_d] == -1).all())
    # empty sizes
    e = tsk.find_closest_points(p[:, :0], x)
    assert e[0].shape == (3, 0, 3)
    e = tsk.find_closest_points(p, x[:, :0])
    assert bool((e[1] == -1).all()) and not bool(e[2].any())
    for args, kw, err, msg in (((p, x[:2]), {}, ValueError, "batches"), ((p[..., :2], x), {}, ValueError, "points_target"),
                               ((p, x), {"max_dist": -1.0}, ValueError, "max_dist"), ((p, pn, x, n), {"max_normal_dot": float("nan")}, ValueError, "NaN"),
                               ((p[..., :2], pn[..., :2], x[..., :2], n[..., :2]), {}, ValueError, "3-D"), ((p, pn, x, n[:, :3]), {}, ValueError, "shape"),
                               ((p, x.cpu()), {}, ValueError, "CUDA"), ((p, x), {"bogus": 1}, TypeError, "bogus"),
                               ((p[..., :1], x[..., :1]), {}, ValueError, "D = 2 or 3")):
        with pytest.raises(err, match=msg):
            tsk.find_closest_points(*args, **kw)


@pytest.mark.gpu
def test_fitting_composition_matches_finite_differences():
    """solve_ik -> model_parameters_to_skeleton_state -> skin_points -> compute_vertex_normals -> find_closest_points with normals against
    a synthetic_scan (under no_grad) -> point-to-plane loss through the gather: the gradient with respect to the solved model parameters
    against float64 central differences of the numpy restatement with the correspondences held fixed."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    ch.skinning = mc.synthetic_tube_mesh(ch, 4, 6, 5)
    rng = np.random.default_rng(4)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    scan, scan_n = mc.synthetic_scan(ch, 3000, theta=theta_star[0], seed=6)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)
    tg = torch.from_numpy(targets).to(dev).double()
    theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                        position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
    theta = theta.detach().double().requires_grad_(True)
    sd, snd = _dev(scan).double(), _dev(scan_n).double()
    x = tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, theta))
    nx = tsk.compute_vertex_normals(ch, x)
    with torch.no_grad():
        _, _, index, valid = tsk.find_closest_points(x, nx, sd, snd, max_normal_dot=0.0)
    assert float(valid.float().mean()) > 0.3
    g = index.clamp(min=0).long().unsqueeze(-1).expand(*index.shape, 3)
    t = torch.gather(sd.expand(B, -1, -1), -2, g)
    tn = torch.gather(snd.expand(B, -1, -1), -2, g)
    loss = ((((x - t) * tn).sum(-1) ** 2) * valid).sum()
    loss.backward()
    ind, val = index.clamp(min=0).cpu().numpy(), valid.cpu().numpy()

    def loss64(th):
        tt, q, s = mc.forward_kinematics(ch, th)
        pts = mc.skin_points(ch, np.concatenate([tt, q, s[..., None]], -1))
        r = ((pts - scan.astype(np.float64)[ind]) * scan_n.astype(np.float64)[ind]).sum(-1)
        return float(((r ** 2) * val).sum())

    th = theta.detach().cpu().numpy()
    assert abs(loss.item() - loss64(th)) <= 1e-3 * max(1.0, loss64(th))
    gth = theta.grad.cpu().numpy()
    h = 1e-5
    for (b, i) in [(0, 0), (0, 4), (1, 7), (1, n - 1)]:
        d = np.zeros_like(th); d[b, i] = h
        fd = (loss64(th + d) - loss64(th - d)) / (2 * h)
        assert abs(fd - gth[b, i]) <= 2e-3 * max(abs(fd), 1.0), (b, i, fd, gth[b, i])
