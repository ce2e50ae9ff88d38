"""compute_vertex_normals (area-weighted vertex normals) on the device and its backward, against float64 restatements.

References: the forward is compared with ``character.vertex_normals`` (float64 numpy); the gradient with torch float64 autograd of
pymomentum's composition (``_normals_torch``: index_select, cross, index_add_, normalize). With eps = 2^-24, e1 / e2 the edges from a
face's corner 0, A_v = sum over the corners that are v of |e1_f| |e2_f|, and n_v the float64 sum, the bounds are, K pinned at about four
times the worst value measured over the fixtures below on the emulator and on an H100:
  forward   |out - out64| <= K_F eps A_v / |n_v|                                                   elementwise; exactly 0 where n_v = 0
  gradient  |g_u - g64_u| <= K_G eps sum over the corners k of faces f that are u of |x_{k+1} - x_{k+2}| (c_i0 + c_i1 + c_i2)
            with c_w = |gbar_w| A_w / |n_w|^2, or |gbar_w| / 1e-12 on the clamp branch                elementwise
The self-checks show that the bounds reject averaged unit face normals, a dropped incident face, a backward without the (I - n n^T)
projection and swapped next / previous corners.
"""
import copy

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib

EPS32 = 2.0 ** -24

# worst measured ratios over these fixtures and several seeds, on the emulator / on an H100 80GB HBM3 at a 700 W power limit: forward
# 2.02 (bodyhands300) / 1.90 (humanoid72_far), gradient 1.10 (bodyhands300) / 1.15 (bodyhands300); each K is about four times the larger
K_F = 8.0
K_G = 5.0


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _tube(make, rings, segments, seed, name, far=False):
    ch = make()
    if far:  # the root, and with it the mesh, 100 units out
        ch.offsets = ch.offsets.copy()
        ch.offsets[0] += np.float32(100.0)
    ch.skinning = mc.synthetic_tube_mesh(ch, rings, segments, seed)
    ch.name = name
    return ch


def _edge_faces_and_rest():
    """A single triangle; an isolated vertex; a zero-area face on exactly representable collinear points, whose vertices have no other
    face; a 64-face fan around a hub; a face that repeats a ring vertex; a zero-area face hanging off the ring. Positions lie on a 1/64
    grid, so the collinear faces stay exactly collinear under the per-instance scaling by powers of two and shifts by quarters."""
    rng = np.random.default_rng(17)
    x = np.zeros((74, 3))
    x[0:3] = [(0, 0, 0), (1, 0, 0), (0, 1, 0)]
    x[3] = (5, 5, 5)
    x[4:7] = [(1, 1, 1), (2, 2, 2), (4, 4, 4)]
    x[7] = (10, 0, 0.3)
    ang = 2 * np.pi * np.arange(64) / 64
    r = rng.uniform(1.0, 2.0, 64)
    x[8:72] = np.stack([10 + r * np.cos(ang), r * np.sin(ang), rng.normal(scale=0.1, size=64)], -1)
    x[72] = x[9] + 1.0
    x[73] = x[9] + 2.0
    x = np.round(x * 64) / 64
    x[72], x[73] = x[9] + 1.0, x[9] + 2.0
    faces = [(0, 1, 2), (4, 5, 6)] + [(7, 8 + k, 8 + (k + 1) % 64) for k in range(64)] + [(8, 8, 9), (9, 72, 73)]
    return np.array(faces, np.int32), x.astype(np.float32)


def _edge_mesh():
    ch = mc.create_test_character(3)
    faces, x = _edge_faces_and_rest()
    V = x.shape[0]
    index = np.zeros((V, mc.MAX_SKIN_JOINTS), np.int32)
    weight = np.zeros((V, mc.MAX_SKIN_JOINTS), np.float32)
    weight[:, 0] = 1.0
    ch.skinning = mc.Skinning(x, index, weight, mc.synthetic_skinning(ch, 1, 0).inverse_bind_pose, faces)
    ch.name = "edges"
    return ch


FIXTURES = {
    "chain3": lambda: _tube(lambda: mc.create_test_character(3), 6, 8, 1, "chain3"),
    "humanoid72": lambda: _tube(lambda: mc.humanoid72()[0], 12, 12, 2, "humanoid72"),
    "bodyhands300": lambda: _tube(lambda: mc.bodyhands300()[0], 8, 8, 3, "bodyhands300"),
    "humanoid72_far": lambda: _tube(lambda: mc.humanoid72()[0], 12, 12, 4, "humanoid72_far", far=True),
    "edges": _edge_mesh,
}
_cache = {}


def _fixture(name):
    if name not in _cache:
        _cache[name] = FIXTURES[name]()
    return _cache[name]


def _positions(ch, B, seed):
    """[B, V, 3] float32: the rest mesh moved per vertex (tubes), or scaled by powers of two and shifted by quarters (the edge mesh)."""
    x = np.asarray(ch.skinning.rest_vertices, np.float32)
    if ch.name == "edges":
        b = np.arange(B)
        return ((2.0 ** (b % 3))[:, None, None] * x[None] + 0.25 * np.stack([b, -2 * b, 3 * b], -1)[:, None, :]).astype(np.float32)
    return (x[None] + np.random.default_rng(seed).normal(scale=0.1, size=(B,) + x.shape)).astype(np.float32)


def _upstream(ch, B, seed):
    return np.random.default_rng(seed).normal(size=(B, ch.skinning.num_vertices, 3)).astype(np.float32)


# ---- float64 references and bounds -------------------------------------------------------------------------------------------------
def _normals_torch(faces, x):
    """pymomentum's compute_vertex_normals (tensor_skinning.cpp:354-383) in torch: x [B, V, 3]."""
    f = torch.from_numpy(np.asarray(faces, np.int64))
    x0, x1, x2 = (x.index_select(-2, f[:, k]) for k in range(3))
    n_f = torch.cross(x1 - x0, x2 - x0, dim=-1)
    n = torch.zeros_like(x)
    for k in range(3):
        n = n.index_add(-2, f[:, k], n_f)
    return torch.nn.functional.normalize(n, dim=-1)


def _grad64(faces, x, G):
    x64 = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    (_normals_torch(faces, x64) * torch.from_numpy(np.asarray(G, np.float64))).sum().backward()
    return x64.grad.numpy()


def _grad_formula(faces, x, G, project=True, swap=False):
    """The backward as the kernels compute it, in float64: h_v, G_f = the sum of h over f's corners, (x_{k+1} - x_{k+2}) x G_f per corner.
    ``project`` = False drops (I - n n^T), ``swap`` = True exchanges next and previous corners: the wrong variants of the self-checks."""
    f = np.asarray(faces, np.int64)
    x, G = np.asarray(x, np.float64), np.asarray(G, np.float64)
    n_f = np.cross(x[:, f[:, 1]] - x[:, f[:, 0]], x[:, f[:, 2]] - x[:, f[:, 0]])
    n = np.zeros_like(x)
    np.add.at(n, (slice(None), f.reshape(-1)), np.repeat(n_f, 3, axis=1))
    ln = np.linalg.norm(n, axis=-1, keepdims=True)
    u = n / np.maximum(ln, 1e-300)
    h = np.where(ln < 1e-12, G / 1e-12, ((G - u * (u * G).sum(-1, keepdims=True)) if project else G) / np.maximum(ln, 1e-300))
    Gf = h[:, f[:, 0]] + h[:, f[:, 1]] + h[:, f[:, 2]]
    g = np.zeros_like(x)
    for k in range(3):
        nxt, prv = f[:, (k + 1) % 3], f[:, (k + 2) % 3]
        if swap:
            nxt, prv = prv, nxt
        np.add.at(g, (slice(None), f[:, k]), np.cross(x[:, nxt] - x[:, prv], Gf))
    return g


def _scales(faces, x, G=None):
    """(forward scale [B, V], |n_v| [B, V], gradient scale [B, V]) of the bounds, eps included."""
    f = np.asarray(faces, np.int64)
    x = np.asarray(x, np.float64)
    e1, e2 = x[:, f[:, 1]] - x[:, f[:, 0]], x[:, f[:, 2]] - x[:, f[:, 0]]
    n = np.zeros_like(x)
    np.add.at(n, (slice(None), f.reshape(-1)), np.repeat(np.cross(e1, e2), 3, axis=1))
    A = np.zeros(x.shape[:2])
    np.add.at(A, (slice(None), f.reshape(-1)), np.repeat(np.linalg.norm(e1, axis=-1) * np.linalg.norm(e2, axis=-1), 3, axis=1))
    nn = np.linalg.norm(n, axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        fwd = np.where(nn > 0, EPS32 * A / nn, np.inf)
        if G is None:
            return fwd, nn, None
        gn = np.linalg.norm(np.asarray(G, np.float64), axis=-1)
        c = np.where(nn < 1e-12, gn / 1e-12, gn * A / nn ** 2)
    Cf = c[:, f[:, 0]] + c[:, f[:, 1]] + c[:, f[:, 2]]
    gs = np.zeros(x.shape[:2])
    for k in range(3):
        el = np.linalg.norm(x[:, f[:, (k + 1) % 3]] - x[:, f[:, (k + 2) % 3]], axis=-1)
        np.add.at(gs, (slice(None), f[:, k]), el * Cf)
    return fwd, nn, EPS32 * gs


def _ratio(err, scale):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, err / scale[..., None], 0.0)
    return float(np.nan_to_num(r, nan=np.inf).max())


def _forward_ratio(faces, x, out):
    fwd, nn, _ = _scales(faces, x)
    out = np.asarray(out, np.float64)
    if not (out[nn == 0] == 0).all():  # isolated vertices and vertices whose faces have zero area: exactly 0
        return np.inf
    return _ratio(np.abs(out - mc.vertex_normals(faces, x)), fwd)


def _grad_ratio(faces, x, G, g, g64=None):
    _, _, gs = _scales(faces, x, G)
    g64 = _grad64(faces, x, G) if g64 is None else g64
    return _ratio(np.abs(np.asarray(g, np.float64) - g64), gs)


def _check(faces, x, G, out, g, where):
    rf = _forward_ratio(faces, x, out) if out is not None else 0.0
    rg = _grad_ratio(faces, x, G, g) if g is not None else 0.0
    assert rf <= K_F and rg <= K_G, (where, rf, rg)
    return rf, rg


# ---- CPU ----------------------------------------------------------------------------------------------------------------------------
def test_numpy_reference_and_gradient_formula_agree_with_torch_autograd():
    for name in ("chain3", "edges", "humanoid72"):
        ch = _fixture(name)
        faces = ch.skinning.faces
        x = _positions(ch, 2, 1)
        G = _upstream(ch, 2, 2)
        ref = _normals_torch(faces, torch.from_numpy(x.astype(np.float64))).numpy()
        assert np.abs(mc.vertex_normals(faces, x) - ref).max() <= 1e-12, name
        assert np.array_equal(mc.vertex_normals(faces, x[1]), mc.vertex_normals(faces, x)[1])
        g64 = _grad64(faces, x, G)
        assert np.abs(_grad_formula(faces, x, G) - g64).max() <= 1e-9 * max(1.0, np.abs(g64).max()), name
    # an isolated vertex gives exactly 0, and non-finite positions propagate
    ch = _fixture("edges")
    x = _positions(ch, 1, 0)
    assert (mc.vertex_normals(ch.skinning.faces, x)[0, 3] == 0).all()
    x[0, 1, 0] = np.nan
    assert np.isnan(mc.vertex_normals(ch.skinning.faces, x)[0, 0:3]).all()


def test_tube_mesh_generator():
    for name, (V, lo, hi) in (("humanoid72", (10368, 9000, 11000)), ("bodyhands300", (19200, 18000, 22000))):
        ch = _fixture(name)
        sk = ch.skinning
        assert sk.num_vertices == V and lo <= V <= hi
        assert sk.faces.dtype == np.int32 and sk.faces.shape[1] == 3
        again = mc.synthetic_tube_mesh(mc.humanoid72()[0] if name == "humanoid72" else mc.bodyhands300()[0], 12 if name == "humanoid72" else 8,
                                       12 if name == "humanoid72" else 8, 2 if name == "humanoid72" else 3)
        for field in ("rest_vertices", "skin_index", "skin_weight", "inverse_bind_pose", "faces"):
            assert np.array_equal(getattr(again, field), getattr(sk, field)), field
        # closed and consistently oriented: every directed edge once, and its reverse too
        f = sk.faces
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
        code = e[:, 0] * V + e[:, 1]
        assert np.unique(code).size == code.size
        assert np.isin(e[:, 1] * V + e[:, 0], code).all()
        assert np.array_equal(np.unique(f), np.arange(V))  # every vertex is referenced
        # face areas differ, and the normals point out of their tubes (12 x 12 or 8 x 8 vertices per joint)
        area = np.linalg.norm(np.cross(*(sk.rest_vertices[f[:, k]] - sk.rest_vertices[f[:, 0]] for k in (1, 2))), axis=-1)
        assert area.std() > 0.05 * area.mean()
        per = V // ch.num_joints
        x = sk.rest_vertices.astype(np.float64).reshape(ch.num_joints, per, 3)
        n = mc.vertex_normals(f, sk.rest_vertices).reshape(ch.num_joints, per, 3)
        assert ((n * (x - x.mean(1, keepdims=True))).sum(-1) > 0).mean() > 0.99
        # the skin weights follow synthetic_skinning's rule: 1 to 8 influences, normalised
        assert np.allclose(sk.skin_weight.sum(1), 1.0, atol=1e-6) and (sk.skin_weight[:, 0] > 0).all()


@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _emu_run(L, faces, x, G):
    faces, x, G = np.ascontiguousarray(faces, np.int32), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(G, np.float32)
    B, V, _ = x.shape
    out, g = np.full_like(x, np.nan), np.full_like(x, np.nan)
    assert L.emu_vertex_normals(V, faces.shape[0], faces.ctypes.data, B, x.ctypes.data, out.ctypes.data) == 0
    assert L.emu_vertex_normals_backward(V, faces.shape[0], faces.ctypes.data, B, x.ctypes.data, G.ctypes.data, g.ctypes.data) == 0
    return out, g


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_forward_and_backward_meet_the_bounds(emu, name):
    ch = _fixture(name)
    x, G = _positions(ch, 3, 11), _upstream(ch, 3, 12)
    out, g = _emu_run(emu, ch.skinning.faces, x, G)
    _check(ch.skinning.faces, x, G, out, g, name)
    if name == "edges":
        assert (out[:, 3] == 0).all() and (g[:, 3] == 0).all()  # the isolated vertex
        assert (out[:, 4:7] == 0).all() and (out[:, 72:74] == 0).all()  # vertices whose only faces have zero area


def test_mesh_face_table_on_a_hand_written_mesh(emu):
    faces = np.array([(0, 1, 2), (2, 1, 3), (1, 1, 0)], np.int32)  # vertex 4 is isolated, face 2 lists vertex 1 twice
    start, corner = np.full(6, -1, np.int32), np.full(9, -1, np.int32)
    assert emu.emu_mesh_faces_tables(5, 3, faces.ctypes.data, start.ctypes.data, corner.ctypes.data) == 0
    assert start.tolist() == [0, 2, 6, 8, 9, 9]
    # 3 f + k, faces ascending, corners ascending within a face
    assert corner.tolist() == [0, 8, 1, 4, 6, 7, 2, 3, 5]


def test_mesh_faces_are_rejected_with_a_message(emu):
    ok = np.array([(0, 1, 2)], np.int32)
    start, corner = np.zeros(8, np.int32), np.zeros(8, np.int32)
    cases = ((0, 1, ok, "at least one vertex"), (3, -1, ok, "must not be negative"), (3, 1, None, "null"),
             (3, 2**31 // 3 + 1, None, "too many faces"), (3, 1, np.array([(0, 1, 3)], np.int32), "outside"),
             (3, 1, np.array([(0, -1, 2)], np.int32), "outside"))
    for V, F, f, msg in cases:
        rc = emu.emu_mesh_faces_tables(V, F, None if f is None else f.ctypes.data, start.ctypes.data, corner.ctypes.data)
        assert rc == 1 and msg in emu.emu_last_error().decode(), (V, F, msg, emu.emu_last_error())
    # degenerate faces, repeated indices and no faces at all are accepted
    for V, F, f in ((3, 1, np.array([(1, 1, 1)], np.int32)), (3, 0, None)):
        assert emu.emu_mesh_faces_tables(V, F, None if f is None else f.ctypes.data, start.ctypes.data, corner.ctypes.data) == 0


def test_bounds_reject_wrong_normals():
    """Each bound against a mistake it is there to catch."""
    ch = _fixture("humanoid72")
    faces = ch.skinning.faces
    x, G = _positions(ch, 2, 31), _upstream(ch, 2, 32)
    f = faces.astype(np.int64)
    x64 = x.astype(np.float64)
    n_f = np.cross(x64[:, f[:, 1]] - x64[:, f[:, 0]], x64[:, f[:, 2]] - x64[:, f[:, 0]])
    unit = n_f / np.linalg.norm(n_f, axis=-1, keepdims=True)
    avg = np.zeros_like(x64)
    np.add.at(avg, (slice(None), f.reshape(-1)), np.repeat(unit, 3, axis=1))
    avg /= np.linalg.norm(avg, axis=-1, keepdims=True)
    assert _forward_ratio(faces, x, avg) > 100 * K_F  # unit face normals averaged: no area weighting
    dropped = mc.vertex_normals(faces, x)
    dropped[:, faces[0]] = mc.vertex_normals(faces[1:], x)[:, faces[0]]
    assert _forward_ratio(faces, x, dropped) > 100 * K_F  # one incident face dropped
    g64 = _grad64(faces, x, G)
    assert _grad_ratio(faces, x, G, _grad_formula(faces, x, G, project=False), g64) > 100 * K_G
    assert _grad_ratio(faces, x, G, _grad_formula(faces, x, G, swap=True), g64) > 100 * K_G
    assert _grad_ratio(faces, x, G, _grad_formula(faces, x, G), g64) <= 1.0  # the right formula, in float64


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = _fixture("chain3")
    with pytest.raises(ValueError, match="CUDA"):
        tsk.compute_vertex_normals(ch, torch.zeros(ch.skinning.num_vertices, 3))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_forward(dc, x):
    out = torch.empty_like(x)
    dc.vertex_normals_device(x.shape[0], x.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out


def _device_backward(dc, x, G):
    g = torch.empty_like(x)
    dc.vertex_normals_backward_device(x.shape[0], x.data_ptr(), G.data_ptr(), g.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_forward_and_backward_meet_the_bounds(name):
    ch = _fixture(name)
    dc = ms.DeviceCharacter(ch, 0)
    assert dc.num_faces == ch.skinning.faces.shape[0] and dc.faces is ch.skinning.faces
    x, G = _positions(ch, 5, 41), _upstream(ch, 5, 42)
    xd, Gd = _dev(x), _dev(G)
    out, g = _device_forward(dc, xd).cpu().numpy(), _device_backward(dc, xd, Gd).cpu().numpy()
    _check(ch.skinning.faces, x, G, out, g, name)
    if name == "edges":
        assert (out[:, 3] == 0).all() and (g[:, 3] == 0).all()
        assert (out[:, 4:7] == 0).all() and (out[:, 72:74] == 0).all()


@pytest.mark.gpu
def test_results_do_not_depend_on_the_batch():
    ch = _fixture("humanoid72")
    dc = ms.DeviceCharacter(ch, 0)
    B = 4099
    x, G = _positions(ch, B, 51), _upstream(ch, B, 52)
    xd, Gd = _dev(x), _dev(G)
    o1, o2 = _device_forward(dc, xd), _device_forward(dc, xd)
    g1, g2 = _device_backward(dc, xd, Gd), _device_backward(dc, xd, Gd)
    assert torch.equal(o1, o2) and torch.equal(g1, g2)
    for b in (0, 3, 2050, B - 1):
        for size in (1, 7):
            lo = min(b, B - size)
            sl = slice(lo, lo + size)
            o = _device_forward(dc, xd[sl].contiguous())
            g = _device_backward(dc, xd[sl].contiguous(), Gd[sl].contiguous())
            assert torch.equal(o[b - lo], o1[b]) and torch.equal(g[b - lo], g1[b]), (b, size)
    sub = np.array([0, 2050, B - 1])
    _check(ch.skinning.faces, x[sub], G[sub], o1[sub].cpu().numpy(), g1[sub].cpu().numpy(), "B=4099")


@pytest.mark.gpu
def test_backward_in_several_slices_meets_the_bounds():
    """bodyhands300's 19 200 vertices take 225 KiB of h per instance, so 2400 instances need three slices of the 256 MiB scratch."""
    ch = _fixture("bodyhands300")
    dc = ms.DeviceCharacter(ch, 0)
    B, V = 2400, ch.skinning.num_vertices
    assert B * V * 3 * 4 > 2 * (256 << 20)
    gen = torch.Generator(device="cuda").manual_seed(61)
    xd = torch.from_numpy(ch.skinning.rest_vertices).cuda()[None] + 0.1 * torch.randn(B, V, 3, device="cuda", generator=gen)
    Gd = torch.randn(B, V, 3, device="cuda", generator=gen)
    g = _device_backward(dc, xd, Gd)
    sub = [0, 1164, 1165, 2330, B - 1]
    x, G = xd[sub].cpu().numpy(), Gd[sub].cpu().numpy()
    _check(ch.skinning.faces, x, G, None, g[sub].cpu().numpy(), "slices")
    alone = _device_backward(dc, xd[sub].contiguous(), Gd[sub].contiguous())
    assert torch.equal(alone, g[sub])


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_and_clones():
    ch = _fixture("edges")
    sk = ch.skinning
    V, F = sk.num_vertices, sk.faces.shape[0]
    bare = mc.Character(ch.parents, ch.offsets, ch.prerot, ch.num_params, ch.pt_outer, ch.pt_inner, ch.pt_vals, ch.pt_offsets, [], "bare")
    dc = ms.DeviceCharacter(bare, 0)
    x = _dev(_positions(ch, 2, 91))
    G = _dev(_upstream(ch, 2, 92))
    out = torch.empty_like(x)
    assert dc.num_faces == 0 and dc.faces is None
    with pytest.raises(ms.MomentumB200Error, match="no mesh faces"):
        dc.vertex_normals_device(2, x.data_ptr(), out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="no mesh faces"):
        dc.vertex_normals_backward_device(2, x.data_ptr(), G.data_ptr(), out.data_ptr())
    dc.set_skinning(sk)
    assert dc.num_faces == F
    for args in ((0, out.data_ptr()), (x.data_ptr(), 0)):
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.vertex_normals_device(2, *args)
    for args in ((0, G.data_ptr(), out.data_ptr()), (x.data_ptr(), 0, out.data_ptr()), (x.data_ptr(), G.data_ptr(), 0)):
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.vertex_normals_backward_device(2, *args)
    host = np.zeros((2, V, 3), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        dc.vertex_normals_device(2, x.data_ptr(), host.ctypes.data)
    with pytest.raises(ms.MomentumB200Error, match="negative"):
        dc.vertex_normals_device(-1, x.data_ptr(), out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="negative"):
        dc.vertex_normals_backward_device(-1, x.data_ptr(), G.data_ptr(), out.data_ptr())
    dc.vertex_normals_device(0, 0, 0)  # batch 0: nothing to do
    dc.vertex_normals_backward_device(0, 0, 0, 0)
    # a rejected face table leaves the earlier one; the library names the reason
    bad = np.ascontiguousarray(sk.faces.copy()); bad[5, 1] = V
    fb = bad.ctypes.data_as(ms._ip)
    assert dc._L.mb2_character_set_mesh_faces(dc._h, V, F, fb) == 1
    assert "outside" in dc._L.mb2_last_error().decode() and dc.num_faces == F
    assert dc._L.mb2_character_set_mesh_faces(dc._h, V, 1, None) == 1 and "null" in dc._L.mb2_last_error().decode()
    assert dc._L.mb2_character_set_mesh_faces(dc._h, 0, 1, fb) == 1 and dc.num_faces == F
    # the clone computes the same bits
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        assert dc._L.mb2_character_num_faces(clone) == F
        outs = []
        for h in (dc._h, clone):
            o, g = torch.empty_like(x), torch.empty_like(x)
            dc._check(dc._L.mb2_character_vertex_normals_device(h, 2, ms.C.c_void_p(x.data_ptr()), ms.C.c_void_p(o.data_ptr()), None))
            dc._check(dc._L.mb2_character_vertex_normals_backward_device(h, 2, ms.C.c_void_p(x.data_ptr()), ms.C.c_void_p(G.data_ptr()),
                                                                          ms.C.c_void_p(g.data_ptr()), None))
            outs.append((o, g))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    finally:
        dc._L.mb2_character_destroy(clone)
    # num_faces 0 with a null array removes the faces; a skinning without faces does too
    dc._check(dc._L.mb2_character_set_mesh_faces(dc._h, 0, 0, None))
    assert dc.num_faces == 0
    with pytest.raises(ms.MomentumB200Error, match="no mesh faces"):
        dc.vertex_normals_device(2, x.data_ptr(), out.data_ptr())
    dc.set_skinning(sk)
    assert dc.num_faces == F
    dc.set_skinning(mc.Skinning(sk.rest_vertices, sk.skin_index, sk.skin_weight, sk.inverse_bind_pose))
    assert dc.num_faces == 0 and dc.faces is None and dc.faces_error is None


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_and_gradcheck():
    from momentum_b200 import torch_skeleton as tsk

    ch = _fixture("humanoid72")
    faces, V = ch.skinning.faces, ch.skinning.num_vertices
    dev = torch.device("cuda", 0)
    x, G = _positions(ch, 3, 71), _upstream(ch, 3, 72)
    x64 = torch.from_numpy(x.astype(np.float64)).to(dev).requires_grad_(True)
    out = tsk.compute_vertex_normals(ch, x64)
    assert out.shape == (3, V, 3) and out.dtype == torch.float64
    out.backward(torch.from_numpy(G.astype(np.float64)).to(dev))
    assert x64.grad.dtype == torch.float64
    _check(faces, x, G, out.detach().cpu().numpy(), x64.grad.cpu().numpy(), "float64 in")
    o32 = tsk.compute_vertex_normals(ch, torch.from_numpy(x).to(dev))
    assert o32.dtype == torch.float32 and torch.equal(o32.double(), out.detach())
    one = tsk.compute_vertex_normals(ch, torch.from_numpy(x[1]).to(dev))
    assert one.shape == (V, 3) and torch.equal(one, o32[1])
    x0 = torch.zeros(0, V, 3, device=dev, requires_grad=True)
    tsk.compute_vertex_normals(ch, x0).sum().backward()
    assert x0.grad.shape == (0, V, 3)
    for bad in (torch.zeros(V + 1, 3, device=dev), torch.zeros(2, V, 4, device=dev), torch.zeros(1, 1, V, 3, device=dev)):
        with pytest.raises(ValueError, match="vertex_positions must be"):
            tsk.compute_vertex_normals(ch, bad)
    plain = copy.copy(ch)
    plain.skinning = mc.synthetic_skinning(ch, 3, 0)
    with pytest.raises(ValueError, match="no mesh faces"):
        tsk.compute_vertex_normals(plain, torch.zeros(plain.skinning.num_vertices, 3, device=dev))
    # gradcheck on the edge mesh minus its zero-area faces (whose clamp gradient is 1e12): the value of the float64 torch restatement, the
    # gradient of the device op
    ech = copy.copy(_fixture("edges"))
    esk = ech.skinning
    ech.skinning = mc.Skinning(esk.rest_vertices, esk.skin_index, esk.skin_weight, esk.inverse_bind_pose, esk.faces[[0] + list(range(2, 66))])

    def f(xx):
        ours = tsk.compute_vertex_normals(ech, xx)
        return _normals_torch(ech.skinning.faces, xx.detach().cpu()).to(dev) + ours - ours.detach()

    xe = torch.from_numpy(_positions(ech, 2, 73).astype(np.float64)).to(dev)
    xe = (xe + 0.01 * torch.randn_like(xe)).requires_grad_(True)
    assert torch.autograd.gradcheck(f, (xe,), eps=1e-6, atol=2e-4, rtol=2e-3)


@pytest.mark.gpu
def test_rejected_faces_leave_the_other_operations_alone():
    from momentum_b200 import torch_skeleton as tsk

    good = _fixture("chain3")
    dev = torch.device("cuda", 0)
    st = torch.from_numpy(np.concatenate([np.zeros((2, 3, 3)), np.tile([0, 0, 0, 1, 1], (2, 3, 1))], -1).astype(np.float32)).to(dev)
    V = good.skinning.num_vertices
    for faces, reason in ((np.where(good.skinning.faces == 5, V, good.skinning.faces), "outside"), (good.skinning.faces[:, :2], r"\[F, 3\]"),
                          (good.skinning.faces.astype(np.float32), r"\[F, 3\]")):
        ch = copy.copy(good)
        sk = good.skinning
        ch.skinning = mc.Skinning(sk.rest_vertices, sk.skin_index, sk.skin_weight, sk.inverse_bind_pose, faces)
        assert torch.equal(tsk.skin_points(ch, st), tsk.skin_points(good, st))
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(2, ch.num_params, device=dev))
        x = torch.from_numpy(sk.rest_vertices).to(dev)
        with pytest.raises(ValueError, match=reason):
            tsk.compute_vertex_normals(ch, x)
        dc = ms.DeviceCharacter(ch, 0)
        assert dc.faces is None and dc.num_faces == 0 and dc.skinning is ch.skinning
        with pytest.raises(ValueError, match=reason):
            tsk.compute_vertex_normals(dc, x)


@pytest.mark.gpu
def test_replacing_the_skinning_keeps_recorded_graphs_whole():
    from momentum_b200 import torch_skeleton as tsk

    ch = copy.copy(_fixture("chain3"))
    base = ch.skinning
    A = mc.Skinning(base.rest_vertices, base.skin_index, base.skin_weight, base.inverse_bind_pose, base.faces)
    flipped = base.faces[:, ::-1].copy()
    ch.skinning = A
    dev = torch.device("cuda", 0)
    x, G = _positions(ch, 2, 81), _upstream(ch, 2, 82)
    xa = torch.from_numpy(x).to(dev).requires_grad_(True)
    pa = tsk.compute_vertex_normals(ch, xa)
    ch.skinning = mc.Skinning(A.rest_vertices, A.skin_index, A.skin_weight, A.inverse_bind_pose, flipped)
    pb = tsk.compute_vertex_normals(ch, torch.from_numpy(x).to(dev))
    _check(flipped, x, None, pb.cpu().numpy(), None, "the new faces")
    pa.backward(torch.from_numpy(G).to(dev))
    _check(A.faces, x, G, pa.detach().cpu().numpy(), xa.grad.cpu().numpy(), "recorded with A")
    # replacing only the faces of the skinning gives a new handle too
    ch.skinning = A
    xc = torch.from_numpy(x).to(dev).requires_grad_(True)
    pc = tsk.compute_vertex_normals(ch, xc)
    A.faces = flipped
    assert torch.equal(tsk.compute_vertex_normals(ch, torch.from_numpy(x).to(dev)), pb)
    pc.backward(torch.from_numpy(G).to(dev))
    assert torch.equal(pc.detach(), pa.detach()) and torch.equal(xc.grad, xa.grad)
    # through one DeviceCharacter: set_skinning after the forward makes that graph's backward raise
    A.faces = base.faces
    dc = ms.DeviceCharacter(ch, 0)
    xd = torch.from_numpy(x).to(dev).requires_grad_(True)
    pd = tsk.compute_vertex_normals(dc, xd)
    dc.set_skinning(mc.Skinning(A.rest_vertices, A.skin_index, A.skin_weight, A.inverse_bind_pose, flipped))
    with pytest.raises(RuntimeError, match="replaced"):
        pd.backward(torch.from_numpy(G).to(dev))


@pytest.mark.gpu
def test_solve_ik_then_skin_points_then_normals_matches_finite_differences():
    """solve_ik -> model_parameters_to_skeleton_state -> skin_points -> compute_vertex_normals -> a loss on the normals: the gradient with
    respect to the solved model parameters against float64 central differences of the numpy restatement, and a finite, non-zero gradient
    reaching the position targets through the solver's backward."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    ch.skinning = mc.synthetic_tube_mesh(ch, 4, 6, 5)
    rng = np.random.default_rng(4)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)
    wv = rng.normal(size=(ch.skinning.num_vertices, 3))
    wvd = torch.from_numpy(wv).to(dev)

    def downstream(theta):
        return (tsk.compute_vertex_normals(ch, tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, theta))) * wvd).sum()

    def downstream64(theta):
        t, q, s = mc.forward_kinematics(ch, theta)
        pts = mc.skin_points(ch, np.concatenate([t, q, s[..., None]], -1))
        return float((mc.vertex_normals(ch.skinning.faces, pts) * wv).sum())

    tg = torch.from_numpy(targets).to(dev).double().requires_grad_(True)
    theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                        position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
    theta.retain_grad()
    loss = downstream(theta.double())
    loss.backward()
    th = theta.detach().cpu().numpy().astype(np.float64)
    gth = theta.grad.cpu().numpy()
    h = 1e-5
    for (b, i) in [(0, 0), (0, 4), (1, 7), (1, n - 1)]:
        d = np.zeros_like(th); d[b, i] = h
        fd = (downstream64(th + d) - downstream64(th - d)) / (2 * h)
        assert abs(fd - gth[b, i]) <= 2e-3 * max(abs(fd), 1.0), ("theta", b, i, fd, gth[b, i])
    assert torch.isfinite(tg.grad).all() and tg.grad.abs().max().item() > 0.0


@pytest.mark.gpu
def test_skin_with_blend_shapes_then_normals_matches_finite_differences():
    """skin_with_blend_shapes -> compute_vertex_normals -> a loss on the normals: the blend-weight gradient against float64 central
    differences of the numpy restatement."""
    from momentum_b200 import torch_skeleton as tsk

    ch = copy.copy(_fixture("chain3"))
    ch.blend_shape = mc.synthetic_blend_shape(ch, ch.skinning, 6, 7)
    ch.blend_shape = mc.BlendShape(ch.blend_shape.base_shape, ch.blend_shape.shape_vectors * np.float32(3.0))  # visible shape changes
    rng = np.random.default_rng(8)
    st = np.concatenate([np.zeros((2, 3, 3)), np.tile([0, 0, 0, 1, 1], (2, 3, 1))], -1) + rng.normal(scale=0.1, size=(2, 3, 8))
    st = st.astype(np.float32)
    w = rng.normal(scale=0.5, size=(2, 6))
    wv = rng.normal(size=(ch.skinning.num_vertices, 3))
    dev = torch.device("cuda", 0)
    wd = torch.from_numpy(w).to(dev).requires_grad_(True)
    loss = (tsk.compute_vertex_normals(ch, tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev).double(), wd)) * torch.from_numpy(wv).to(dev)).sum()
    loss.backward()
    gw = wd.grad.cpu().numpy()
    assert np.abs(gw).max() > 0.0

    def loss64(ww):
        return float((mc.vertex_normals(ch.skinning.faces, mc.skin_with_blend_shapes(ch, st, ww)) * wv).sum())

    h = 1e-5
    for b in range(2):
        for k in range(6):
            d = np.zeros_like(w); d[b, k] = h
            fd = (loss64(w + d) - loss64(w - d)) / (2 * h)
            assert abs(fd - gw[b, k]) <= 2e-3 * max(abs(fd), 1.0), (b, k, fd, gw[b, k])
