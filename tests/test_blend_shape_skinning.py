"""skin_with_blend_shapes (skinning with an identity blend shape) on the device and its backward, against float64 restatements.

References: the forward is compared with ``character.skin_with_blend_shapes`` (float64 numpy: the shaped rest mesh, then
``character.skin_points``); the skel-state gradient with torch float64 autograd of the skinning at the float64 shaped rest points
(``test_skinning._grads64``), and the weight gradient with the chain rule through the same autograd's rest-point gradient,
dL/dw_k = sum_v <S_kv, dL/dx_v>. Bounds, K pinned at about four times the worst value measured over the fixtures below on the emulator
and on an H100; x is the float64 shaped rest point:
  forward        test_skinning's forward bound at x                                                   elementwise
  skel state     test_skinning's skel-state bound at x                                                per joint
  weights        |gw_k - gw64_k| <= K_W * 2^-24 * sum_v sum_c |S_kvc| (sum_slots |w| |Lin M|^T |g_v|)_c   per instance and k
"""
import ctypes
import copy

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests import test_skinning as tsn

EPS32 = 2.0 ** -24

# worst measured ratios over these fixtures and three seeds, on the emulator / on an H100 80GB HBM3 at a 700 W power limit: forward
# 16.1 / 15.7 (chain6_edges_k8), skel state 42.6 / 41.3 (humanoid72_far_k16: the float shaped rest point 100 units out), weights
# 1.93 / 1.65 (chain3_v1_k4); each K is about four times the larger
K_F = 64.0
K_S = 170.0
K_W = 8.0


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _shaped(ch, K, seed, name):
    ch.blend_shape = mc.synthetic_blend_shape(ch, ch.skinning, K, seed)
    ch.name = name
    return ch


def _one_vertex():
    ch = copy.copy(tsn._fixture("chain3_v1"))
    return _shaped(ch, 4, 1, "chain3_v1_k4")


def _humanoid(K, seed):
    ch = copy.copy(tsn._fixture("humanoid72"))
    return _shaped(ch, K, seed, f"humanoid72_k{K}")


FIXTURES = {
    "chain3_v1_k4": (_one_vertex, 4),
    "humanoid72_k1": (lambda: _humanoid(1, 3), 1),
    "humanoid72_k16": (lambda: _humanoid(16, 4), 16),
    "humanoid72_k64": (lambda: _humanoid(64, 5), 64),
    "humanoid72_k64_first23": (lambda: _humanoid(64, 5), 23),  # K' < K
    "bodyhands300_k16": (lambda: _shaped(copy.copy(tsn._fixture("bodyhands300")), 16, 6, "bodyhands300_k16"), 16),
    "humanoid72_far_k16": (lambda: _shaped(copy.copy(tsn._fixture("humanoid72_far")), 16, 7, "humanoid72_far_k16"), 16),
    "chain6_edges_k8": (lambda: _shaped(copy.copy(tsn._fixture("chain6_edges")), 8, 8, "chain6_edges_k8"), 8),
}
_cache = {}


def _fixture(name):
    if name not in _cache:
        make, Kp = FIXTURES[name]
        _cache[name] = (make(), Kp)
    return _cache[name]


def _weights(B, Kp, seed):
    return np.random.default_rng(seed).normal(scale=1.5, size=(B, Kp)).astype(np.float32)


# ---- float64 references and bounds -------------------------------------------------------------------------------------------------
def _rest64(ch, w):
    bs = ch.blend_shape
    w = np.asarray(w, np.float64)
    return np.asarray(bs.base_shape, np.float64) + np.einsum("bk,kvc->bvc", w, np.asarray(bs.shape_vectors[:w.shape[-1]], np.float64))


def _refs(ch, st, w, G):
    """float64 (points, dL/dstate, dL/dw) of L = sum(points * G)."""
    x = _rest64(ch, w)
    gs64, gx64 = tsn._grads64(ch, st, x, G)
    gw64 = np.einsum("kvc,bvc->bk", np.asarray(ch.blend_shape.shape_vectors[:w.shape[-1]], np.float64), gx64)
    return mc.skin_with_blend_shapes(ch, st, w), gs64, gw64


def _weight_scale(ch, st, w, G):
    """per instance and k: 2^-24 sum_v sum_c |S_kvc| (sum_slots |w| |Lin M|^T |g_v|)_c"""
    sk = ch.skinning
    st64 = np.asarray(st, np.float64)
    qn = st64[..., 3:7] / np.linalg.norm(st64[..., 3:7], axis=-1, keepdims=True)
    L = np.abs((mc._quat_matrix(qn) * st64[..., 7, None, None]) @ np.asarray(sk.inverse_bind_pose, np.float64)[None, :, :, :3])
    act = tsn._active(sk)
    g = np.abs(np.asarray(G, np.float64))
    r = np.zeros_like(g)
    for k in range(mc.MAX_SKIN_JOINTS):
        j = np.where(act[:, k], sk.skin_index[:, k], 0)
        wk = np.where(act[:, k], np.abs(sk.skin_weight[:, k]), 0.0)
        r += np.einsum("bvrc,bvr->bvc", L[:, j], g) * wk[None, :, None]
    return EPS32 * np.einsum("kvc,bvc->bk", np.abs(np.asarray(ch.blend_shape.shape_vectors[:w.shape[-1]], np.float64)), r)


def _weight_ratio(ch, st, w, G, gw, gw64):
    err = np.abs(np.asarray(gw, np.float64) - gw64)
    den = _weight_scale(ch, st, w, G)
    return float(np.where(err > 0, err / np.maximum(den, 1e-300), 0.0).max())


def _ratios(ch, st, w, G, p, gs, gw):
    x = _rest64(ch, w)
    p64, gs64, gw64 = _refs(ch, st, w, G)
    out = {}
    if p is not None:
        out["forward"] = tsn._forward_ratio(ch, st, x, p)
    if gs is not None:
        out["state"] = tsn._state_ratio(ch, st, x, G, gs, gs64)
    if gw is not None:
        out["weights"] = _weight_ratio(ch, st, w, G, gw, gw64)
    return out


def _check(ratios, where):
    bound = {"forward": K_F, "state": K_S, "weights": K_W}
    for key, r in ratios.items():
        assert r <= bound[key], (where, key, r)


# ---- CPU ----------------------------------------------------------------------------------------------------------------------------
def _direct(ch, st, w):
    """skinWithBlendShapes written out per vertex with 4x4 matrices: p_rest = base + S^T w, then sum_slots w_j (T_j IBP_j) p_rest."""
    sk, bs = ch.skinning, ch.blend_shape
    J, V = ch.num_joints, sk.num_vertices
    out = np.zeros((st.shape[0], V, 3))
    for b in range(st.shape[0]):
        M = np.zeros((J, 4, 4))
        for j in range(J):
            q = st[b, j, 3:7].astype(np.float64)
            T = np.eye(4)
            T[:3, :3] = mc._quat_matrix(q / np.linalg.norm(q)) * float(st[b, j, 7])
            T[:3, 3] = st[b, j, :3]
            I = np.eye(4)
            I[:3, :] = sk.inverse_bind_pose[j]
            M[j] = T @ I
        for v in range(V):
            rest = bs.base_shape[v].astype(np.float64) + bs.shape_vectors[:len(w[b]), v].astype(np.float64).T @ w[b].astype(np.float64)
            for k in range(mc.MAX_SKIN_JOINTS):
                if sk.skin_weight[v, k] == 0.0:
                    break
                out[b, v] += float(sk.skin_weight[v, k]) * (M[sk.skin_index[v, k]] @ np.append(rest, 1.0))[:3]
    return out


def test_numpy_reference_agrees_with_direct_restatement_and_composition():
    for name in ("chain3_v1_k4", "chain6_edges_k8", "humanoid72_k64_first23"):
        ch, Kp = _fixture(name)
        st = tsn._states(ch, 2, 1)
        w = _weights(2, Kp, 2)
        p = mc.skin_with_blend_shapes(ch, st, w)
        scale = max(1.0, np.abs(p).max())
        if ch.skinning.num_vertices <= 200:
            assert np.abs(p - _direct(ch, st, w)).max() <= 1e-12 * scale, name
        rest = ch.blend_shape.base_shape.reshape(1, -1).astype(np.float64) + w.astype(np.float64) @ ch.blend_shape.shape_vectors[:Kp].reshape(Kp, -1).astype(np.float64)
        assert np.abs(p - mc.skin_points(ch, st, rest.reshape(2, -1, 3))).max() <= 1e-12 * scale, name
        # shared [K'] weights and a single state
        assert np.array_equal(mc.skin_with_blend_shapes(ch, st[0], w[0]), mc.skin_with_blend_shapes(ch, st[:1], w[:1])[0])


def test_synthetic_blend_shape():
    ch, _ = _fixture("humanoid72_k64")
    bs = ch.blend_shape
    assert bs.shape_vectors.shape == (64, ch.skinning.num_vertices, 3) and bs.shape_vectors.dtype == np.float32
    assert np.array_equal(bs.base_shape, ch.skinning.rest_vertices)
    again = mc.synthetic_blend_shape(ch, ch.skinning, 64, 5)
    assert np.array_equal(again.shape_vectors, bs.shape_vectors)
    # three bumps of at most 4 % of a bone each, and every shape moves some vertices
    t = mc.forward_kinematics(ch, np.zeros((1, ch.num_params)))[0][0]
    bone = np.linalg.norm(t[1:] - t[ch.parents[1:]], axis=-1).max()
    assert 0.0 < np.abs(bs.shape_vectors).max() <= 3 * 0.04 * bone
    assert (np.abs(bs.shape_vectors).reshape(64, -1).max(1) > 0).all()


@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _head(ch, keep, base=None, vectors=None, K=None):
    bs = ch.blend_shape
    base = np.ascontiguousarray(bs.base_shape if base is None else base, np.float32)
    vectors = np.ascontiguousarray(bs.shape_vectors if vectors is None else vectors, np.float32)
    keep.extend([base, vectors])
    K = vectors.shape[0] if K is None else K
    return tsn._head(ch, keep) + [K, base.shape[0], base.ctypes.data, vectors.ctypes.data]


def _emu_forward(L, ch, st, w, **kw):
    keep = []
    st, w = np.ascontiguousarray(st, np.float32), np.ascontiguousarray(w, np.float32)
    out = np.full((st.shape[0], ch.skinning.num_vertices, 3), np.nan, np.float32)
    rc = L.emu_skin_with_blend_shapes(*_head(ch, keep, **kw), st.shape[0], st.ctypes.data, w.ctypes.data, w.shape[1], out.ctypes.data)
    return rc, out


def _emu_backward(L, ch, st, w, G):
    keep = []
    st, w, G = (np.ascontiguousarray(a, np.float32) for a in (st, w, G))
    gs = np.full(st.shape, np.nan, np.float32)
    gw = np.full(w.shape, np.nan, np.float32)
    rc = L.emu_skin_with_blend_shapes_backward(*_head(ch, keep), st.shape[0], st.ctypes.data, w.ctypes.data, w.shape[1], G.ctypes.data,
                                               gs.ctypes.data, gw.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return gs, gw


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_forward_and_backward_meet_the_bounds(emu, name):
    ch, Kp = _fixture(name)
    B = 3
    st = tsn._states(ch, B, 11)
    w = _weights(B, Kp, 13)
    G = tsn._upstream(ch, B, 12)
    rc, p = _emu_forward(emu, ch, st, w)
    assert rc == 0, emu.emu_last_error().decode()
    gs, gw = _emu_backward(emu, ch, st, w, G)
    _check(_ratios(ch, st, w, G, p, gs, gw), name)


def test_weight_gradient_matches_central_differences(emu):
    """The reference is linear in w, so central differences of the float64 reference are exact up to rounding."""
    for name in ("chain6_edges_k8", "humanoid72_k16"):
        ch, Kp = _fixture(name)
        st = tsn._states(ch, 2, 21)
        w = _weights(2, Kp, 22).astype(np.float64)
        G = tsn._upstream(ch, 2, 23).astype(np.float64)
        _, gw = _emu_backward(emu, ch, st, w, G)
        h = 1e-3
        for b, k in ((0, 0), (1, Kp - 1), (1, Kp // 2)):
            d = np.zeros_like(w)
            d[b, k] = h
            fd = ((mc.skin_with_blend_shapes(ch, st, w + d) - mc.skin_with_blend_shapes(ch, st, w - d)) * G).sum() / (2 * h)
            assert abs(gw[b, k] - fd) <= 1e-4 * max(1.0, abs(fd)), (name, b, k, gw[b, k], fd)


def test_rejected_blend_shapes(emu):
    ch, _ = _fixture("chain3_v1_k4")
    bs = ch.blend_shape
    st = tsn._states(ch, 1, 1)
    w = _weights(1, 4, 2)
    nan_base = bs.base_shape.copy(); nan_base[0, 1] = np.nan
    inf_vec = bs.shape_vectors.copy(); inf_vec[2, 0, 0] = np.inf
    cases = ((dict(base=nan_base), "base shape must be finite"), (dict(vectors=inf_vec), "shape vectors must be finite"),
             (dict(vectors=bs.shape_vectors[:0]), "at least one shape vector"),
             (dict(base=np.zeros((0, 3), np.float32), vectors=np.zeros((4, 0, 3), np.float32)), "at least one vertex"),
             (dict(base=np.zeros((2, 3), np.float32), vectors=np.zeros((4, 2, 3), np.float32)), "vertex count differs"))
    for kw, msg in cases:
        rc, _ = _emu_forward(emu, ch, st, w, **kw)
        assert rc == 1, kw  # MB2_ERR_INVALID_ARGUMENT
        assert msg in emu.emu_last_error().decode(), (msg, emu.emu_last_error())
    for Kp in (0, 5):
        rc, _ = _emu_forward(emu, ch, st, np.zeros((1, Kp), np.float32))
        assert rc == 1 and "num_weights" in emu.emu_last_error().decode(), Kp
    # a null array with a positive count, and a rejected blend shape leaves the earlier one in place
    base, vec = np.ascontiguousarray(bs.base_shape), np.ascontiguousarray(bs.shape_vectors)
    k_after = ctypes.c_int32(-1)
    for b2, v2, msg in ((None, vec, "null"), (base, None, "null"), (nan_base, vec, "finite")):
        rc = emu.emu_blend_shape_replace(4, 1, base.ctypes.data, vec.ctypes.data, 2, 1, None if b2 is None else np.ascontiguousarray(b2).ctypes.data,
                                         None if v2 is None else v2.ctypes.data, ctypes.byref(k_after))
        assert rc == 1 and msg in emu.emu_last_error().decode() and k_after.value == 4, (msg, k_after.value)
    rc = emu.emu_blend_shape_replace(4, 1, base.ctypes.data, vec.ctypes.data, 2, 1, base.ctypes.data, vec.ctypes.data, ctypes.byref(k_after))
    assert rc == 0 and k_after.value == 2


def test_bounds_reject_wrong_blend_shapes():
    """Each bound against a mistake it is there to catch: a shape vector dropped from the rest point, the weights of a neighbouring
    instance, and the weight gradient summed against the wrong shape vector."""
    ch, Kp = _fixture("humanoid72_k16")
    B = 2
    st = tsn._states(ch, B, 31)
    w = _weights(B, Kp, 32)
    G = tsn._upstream(ch, B, 33)
    p64, gs64, gw64 = _refs(ch, st, w, G)
    w_drop = w.copy(); w_drop[:, 3] = 0.0
    assert tsn._forward_ratio(ch, st, _rest64(ch, w), mc.skin_with_blend_shapes(ch, st, w_drop)) > 100 * K_F
    _, gs_swap, _ = _refs(ch, st, w[::-1].copy(), G)
    assert tsn._state_ratio(ch, st, _rest64(ch, w), G, gs_swap, gs64) > 100 * K_S
    assert _weight_ratio(ch, st, w, G, np.roll(gw64, 1, axis=1), gw64) > 100 * K_W


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch, _ = _fixture("chain3_v1_k4")
    with pytest.raises(ValueError, match="CUDA"):
        tsk.skin_with_blend_shapes(ch, torch.zeros(ch.num_joints, 8), torch.zeros(4))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_forward(dc, st, w):
    B = st.shape[0]
    out = torch.empty(B, dc.skinning.num_vertices, 3, device=st.device)
    dc.skin_with_blend_shapes_device(B, st.data_ptr(), w.data_ptr(), w.shape[1], out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out


def _device_backward(dc, st, w, G, want_state=True, want_weights=True):
    B = st.shape[0]
    gs = torch.empty_like(st) if want_state else None
    gw = torch.empty_like(w) if want_weights else None
    dc.skin_with_blend_shapes_backward_device(B, st.data_ptr(), w.data_ptr(), w.shape[1], G.data_ptr(), 0 if gs is None else gs.data_ptr(),
                                              0 if gw is None else gw.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return gs, gw


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_forward_and_backward_meet_the_bounds(name):
    ch, Kp = _fixture(name)
    dc = ms.DeviceCharacter(ch, 0)
    B = 5
    st, w, G = tsn._states(ch, B, 41), _weights(B, Kp, 43), tsn._upstream(ch, B, 42)
    std, wd, Gd = _dev(st), _dev(w), _dev(G)
    p = _device_forward(dc, std, wd)
    gs, gw = _device_backward(dc, std, wd, Gd)
    _check(_ratios(ch, st, w, G, p.cpu().numpy(), gs.cpu().numpy(), gw.cpu().numpy()), name)
    # each output alone gives the same bits
    gs_only, _ = _device_backward(dc, std, wd, Gd, want_weights=False)
    _, gw_only = _device_backward(dc, std, wd, Gd, want_state=False)
    assert torch.equal(gs_only, gs) and torch.equal(gw_only, gw)


@pytest.mark.gpu
def test_results_do_not_depend_on_the_batch():
    ch, Kp = _fixture("humanoid72_k16")
    dc = ms.DeviceCharacter(ch, 0)
    B = 4096
    st, w, G = tsn._states(ch, B, 51), _weights(B, Kp, 52), tsn._upstream(ch, B, 53)
    std, wd, Gd = _dev(st), _dev(w), _dev(G)
    p1, p2 = _device_forward(dc, std, wd), _device_forward(dc, std, wd)
    s1, w1 = _device_backward(dc, std, wd, Gd)
    s2, w2 = _device_backward(dc, std, wd, Gd)
    assert torch.equal(p1, p2) and torch.equal(s1, s2) and torch.equal(w1, w2)
    for b in (0, 3, 1000, B - 1):
        for size in (1, 7):
            lo = min(b, B - size)
            sl = slice(lo, lo + size)
            at = b - lo
            p = _device_forward(dc, std[sl].contiguous(), wd[sl].contiguous())
            s, g = _device_backward(dc, std[sl].contiguous(), wd[sl].contiguous(), Gd[sl].contiguous())
            assert torch.equal(p[at], p1[b]) and torch.equal(s[at], s1[b]) and torch.equal(g[at], w1[b]), (b, size)
    sub = np.array([0, 1000, B - 1])
    _check(_ratios(ch, st[sub], w[sub], G[sub], p1[sub].cpu().numpy(), s1[sub].cpu().numpy(), w1[sub].cpu().numpy()), "B=4096")


@pytest.mark.gpu
def test_agrees_with_the_two_step_composition():
    from momentum_b200 import torch_skeleton as tsk

    for name in ("humanoid72_k64_first23", "bodyhands300_k16"):
        ch, Kp = _fixture(name)
        B = 4
        st, w, G = tsn._states(ch, B, 61), _weights(B, Kp, 62), tsn._upstream(ch, B, 63)
        dev = torch.device("cuda", 0)
        sf = torch.from_numpy(st).to(dev).requires_grad_(True)
        wf = torch.from_numpy(w).to(dev).requires_grad_(True)
        tsk.skin_with_blend_shapes(ch, sf, wf).backward(torch.from_numpy(G).to(dev))
        sc = torch.from_numpy(st).to(dev).requires_grad_(True)
        wc = torch.from_numpy(w).to(dev).requires_grad_(True)
        S = torch.from_numpy(ch.blend_shape.shape_vectors[:Kp]).to(dev)
        rest = torch.from_numpy(ch.blend_shape.base_shape).to(dev) + torch.einsum("bk,kvc->bvc", wc, S)
        pc = tsk.skin_points(ch, sc, rest)
        pc.backward(torch.from_numpy(G).to(dev))
        pf = tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev), torch.from_numpy(w).to(dev))
        for p, gs, gw in ((pf, sf.grad, wf.grad), (pc, sc.grad, wc.grad)):
            _check(_ratios(ch, st, w, G, p.detach().cpu().numpy(), gs.cpu().numpy(), gw.cpu().numpy()), name)


@pytest.mark.gpu
def test_torch_wrapper_shapes_shared_weights_and_gradcheck():
    from momentum_b200 import torch_skeleton as tsk

    ch, Kp = _fixture("humanoid72_k16")
    J, V = ch.num_joints, ch.skinning.num_vertices
    dev = torch.device("cuda", 0)
    B = 3
    st, w, G = tsn._states(ch, B, 71), _weights(B, Kp, 72), tsn._upstream(ch, B, 73)
    # float64 in -> float64 out; [K'] shared weights give the batch sum of the per-instance gradients
    s64 = torch.from_numpy(st.astype(np.float64)).to(dev).requires_grad_(True)
    w_shared = torch.from_numpy(w[0].astype(np.float64)).to(dev).requires_grad_(True)
    p = tsk.skin_with_blend_shapes(ch, s64, w_shared)
    assert p.shape == (B, V, 3) and p.dtype == torch.float64
    p.backward(torch.from_numpy(G.astype(np.float64)).to(dev))
    w_rep = torch.from_numpy(np.repeat(w[:1], B, 0).astype(np.float64)).to(dev).requires_grad_(True)
    tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev).double(), w_rep).backward(torch.from_numpy(G.astype(np.float64)).to(dev))
    assert w_shared.grad.shape == (Kp,) and torch.allclose(w_shared.grad, w_rep.grad.sum(0), rtol=1e-6, atol=1e-6 * float(w_rep.grad.abs().max()))
    gw64 = _refs(ch, st, np.repeat(w[:1], B, 0), G)[2].sum(0)
    den = _weight_scale(ch, st, np.repeat(w[:1], B, 0), G).sum(0)
    assert (np.abs(w_shared.grad.cpu().numpy() - gw64) <= K_W * den).all()
    # [J, 8] with [K']
    p1 = tsk.skin_with_blend_shapes(ch, torch.from_numpy(st[1]).to(dev), torch.from_numpy(w[1]).to(dev))
    assert p1.shape == (V, 3)
    assert torch.equal(p1, tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev), torch.from_numpy(w).to(dev))[1])
    # batch 0
    s0 = torch.zeros(0, J, 8, device=dev, requires_grad=True)
    w0 = torch.zeros(0, Kp, device=dev, requires_grad=True)
    tsk.skin_with_blend_shapes(ch, s0, w0).sum().backward()
    assert s0.grad.shape == (0, J, 8) and w0.grad.shape == (0, Kp)
    # ValueErrors
    for bad_w in (torch.zeros(Kp + 1, device=dev), torch.zeros(B + 1, Kp, device=dev), torch.zeros(0, device=dev)):
        with pytest.raises(ValueError, match="blend_weights must be"):
            tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev), bad_w)
    with pytest.raises(ValueError, match="no blend shape"):
        tsk.skin_with_blend_shapes(tsn._fixture("chain3"), torch.zeros(3, 8, device=dev), torch.zeros(1, device=dev))
    # gradcheck on a small rig: the value of a float64 torch restatement, the gradient of the device op
    ch3, K3 = _fixture("chain6_edges_k8")
    S3 = torch.from_numpy(ch3.blend_shape.shape_vectors.astype(np.float64)).to(dev)
    base3 = torch.from_numpy(ch3.blend_shape.base_shape.astype(np.float64)).to(dev)

    def ref64(s, ww):
        return tsn._skin64(ch3, s.cpu(), (base3 + torch.einsum("bk,kvc->bvc", ww, S3)).cpu()).to(dev)

    def f(s, ww):
        ours = tsk.skin_with_blend_shapes(ch3, s, ww)
        return ref64(s, ww).detach() + ours - ours.detach()

    s3 = torch.from_numpy(tsn._states(ch3, 2, 74).astype(np.float64)).to(dev).requires_grad_(True)
    w3 = torch.from_numpy(_weights(2, K3, 75).astype(np.float64)).to(dev).requires_grad_(True)
    assert torch.autograd.gradcheck(f, (s3, w3), eps=1e-6, atol=2e-4, rtol=2e-3, check_undefined_grad=False)


@pytest.mark.gpu
def test_replacing_the_blend_shape_keeps_recorded_graphs_whole():
    from momentum_b200 import torch_skeleton as tsk

    ch = copy.copy(tsn._fixture("humanoid72"))
    A = mc.synthetic_blend_shape(ch, ch.skinning, 8, 81)
    Bk = mc.synthetic_blend_shape(ch, ch.skinning, 12, 82)
    ch.blend_shape = A
    st, w, G = tsn._states(ch, 2, 83), _weights(2, 8, 84), tsn._upstream(ch, 2, 85)
    dev = torch.device("cuda", 0)
    sa = torch.from_numpy(st).to(dev).requires_grad_(True)
    wa = torch.from_numpy(w).to(dev).requires_grad_(True)
    pa = tsk.skin_with_blend_shapes(ch, sa, wa)
    ch.blend_shape = Bk
    pb = tsk.skin_with_blend_shapes(ch, torch.from_numpy(st).to(dev), torch.from_numpy(_weights(2, 12, 86)).to(dev))
    assert not torch.equal(pb, pa.detach())
    pa.backward(torch.from_numpy(G).to(dev))
    ch.blend_shape = A
    _check(_ratios(ch, st, w, G, pa.detach().cpu().numpy(), sa.grad.cpu().numpy(), wa.grad.cpu().numpy()), "recorded with A")
    # through one DeviceCharacter: set_blend_shape after the forward makes that graph's backward raise
    dc = ms.DeviceCharacter(ch, 0)
    sd = torch.from_numpy(st).to(dev).requires_grad_(True)
    pd = tsk.skin_with_blend_shapes(dc, sd, torch.from_numpy(w).to(dev))
    dc.set_blend_shape(Bk)
    with pytest.raises(RuntimeError, match="replaced"):
        pd.backward(torch.from_numpy(G).to(dev))
    assert dc.num_blend_shapes == 12


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_and_clones():
    ch, Kp = _fixture("chain6_edges_k8")
    J, V, K = ch.num_joints, ch.skinning.num_vertices, ch.blend_shape.num_shapes
    bare = mc.Character(ch.parents, ch.offsets, ch.prerot, ch.num_params, ch.pt_outer, ch.pt_inner, ch.pt_vals, ch.pt_offsets, [], "bare")
    dc = ms.DeviceCharacter(bare, 0)
    st = _dev(tsn._states(ch, 2, 91))
    w = _dev(_weights(2, K, 92))
    G = _dev(tsn._upstream(ch, 2, 93))
    out = torch.zeros(2, V, 3, device="cuda")
    assert dc.num_blend_shapes == 0
    with pytest.raises(ms.MomentumB200Error, match="no skinning"):
        dc.skin_with_blend_shapes_device(2, st.data_ptr(), w.data_ptr(), K, out.data_ptr())
    dc.set_skinning(ch.skinning)
    with pytest.raises(ms.MomentumB200Error, match="no blend shape"):
        dc.skin_with_blend_shapes_device(2, st.data_ptr(), w.data_ptr(), K, out.data_ptr())
    small = mc.BlendShape(ch.blend_shape.base_shape[:3], ch.blend_shape.shape_vectors[:, :3])
    dc.set_blend_shape(small)
    with pytest.raises(ms.MomentumB200Error, match="vertex count differs"):
        dc.skin_with_blend_shapes_device(2, st.data_ptr(), w.data_ptr(), K, out.data_ptr())
    dc.set_blend_shape(ch.blend_shape)
    assert dc.num_blend_shapes == K
    for bad in (0, K + 1):
        with pytest.raises(ms.MomentumB200Error, match="num_weights"):
            dc.skin_with_blend_shapes_device(2, st.data_ptr(), w.data_ptr(), bad, out.data_ptr())
        with pytest.raises(ms.MomentumB200Error, match="num_weights"):
            dc.skin_with_blend_shapes_backward_device(2, st.data_ptr(), w.data_ptr(), bad, G.data_ptr(), 0, 0)
    for args in ((0, w.data_ptr(), out.data_ptr()), (st.data_ptr(), 0, out.data_ptr()), (st.data_ptr(), w.data_ptr(), 0)):
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.skin_with_blend_shapes_device(2, args[0], args[1], K, args[2])
    with pytest.raises(ms.MomentumB200Error, match="null"):
        dc.skin_with_blend_shapes_backward_device(2, st.data_ptr(), w.data_ptr(), K, 0, st.data_ptr(), 0)
    host = np.zeros((2, V, 3), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        dc.skin_with_blend_shapes_device(2, st.data_ptr(), w.data_ptr(), K, host.ctypes.data)
    with pytest.raises(ms.MomentumB200Error, match="negative"):
        dc.skin_with_blend_shapes_device(-1, st.data_ptr(), w.data_ptr(), K, out.data_ptr())
    dc.skin_with_blend_shapes_device(0, 0, 0, K, 0)  # batch 0: nothing to do
    dc.skin_with_blend_shapes_backward_device(0, 0, 0, K, 0, 0, 0)
    nan_vec = ch.blend_shape.shape_vectors.copy(); nan_vec[0, 0, 0] = np.nan
    with pytest.raises(ms.MomentumB200Error, match="finite"):
        dc.set_blend_shape(mc.BlendShape(ch.blend_shape.base_shape, nan_vec))
    assert dc.num_blend_shapes == K  # a rejected blend shape leaves the earlier one
    # the clone skins identically
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        assert dc._L.mb2_character_num_blend_shapes(clone) == K
        outs = []
        for h in (dc._h, clone):
            p = torch.empty(2, V, 3, device="cuda")
            gs, gw = torch.empty_like(st), torch.empty_like(w)
            dc._check(dc._L.mb2_character_skin_with_blend_shapes_device(h, 2, ms.C.c_void_p(st.data_ptr()), ms.C.c_void_p(w.data_ptr()), K,
                                                                        ms.C.c_void_p(p.data_ptr()), None))
            dc._check(dc._L.mb2_character_skin_with_blend_shapes_backward_device(h, 2, ms.C.c_void_p(st.data_ptr()), ms.C.c_void_p(w.data_ptr()), K,
                                                                                 ms.C.c_void_p(G.data_ptr()), ms.C.c_void_p(gs.data_ptr()),
                                                                                 ms.C.c_void_p(gw.data_ptr()), None))
            outs.append((p, gs, gw))
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(*outs))
    finally:
        dc._L.mb2_character_destroy(clone)


@pytest.mark.gpu
def test_many_shape_vectors_take_the_narrow_tile_or_are_rejected():
    """K' = 4000 does not fit a 16-instance tile's weights in shared memory but fits a 4-instance tile, at any batch; K' = 20000 fits
    neither and is rejected by name."""
    base, _ = _fixture("chain3_v1_k4")
    ch = copy.copy(base)
    rng = np.random.default_rng(95)
    ch.blend_shape = mc.BlendShape(ch.skinning.rest_vertices.copy(), rng.normal(scale=0.01, size=(20000, 1, 3)).astype(np.float32))
    dc = ms.DeviceCharacter(ch, 0)
    B = 600  # enough tiles for the wide tile to be chosen if it fitted
    st, G = tsn._states(ch, B, 96), tsn._upstream(ch, B, 97)
    w = _weights(B, 4000, 98) * np.float32(0.02)
    p = _device_forward(dc, _dev(st), _dev(w))
    gs, gw = _device_backward(dc, _dev(st), _dev(w), _dev(G))
    # a sum of 4000 terms per rest point is outside the fixtures the bounds were pinned on: here the results only have to be right
    sub = np.array([0, 299, B - 1])
    p64, gs64, gw64 = _refs(ch, st[sub], w[sub], G[sub])
    for got, ref in ((p.cpu().numpy()[sub], p64), (gs.cpu().numpy()[sub], gs64), (gw.cpu().numpy()[sub], gw64)):
        assert np.abs(got - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    big = _dev(np.zeros((2, 20000), np.float32))
    out = torch.empty(2, 1, 3, device="cuda")
    with pytest.raises(ms.MomentumB200Error, match="too large"):
        dc.skin_with_blend_shapes_device(2, _dev(st[:2]).data_ptr(), big.data_ptr(), 20000, out.data_ptr())


@pytest.mark.gpu
def test_a_rejected_blend_shape_leaves_the_other_operations_alone():
    """A character whose blend shape the library rejects still skins with skin_points and runs forward kinematics; only the blend-shape
    call reports the rejection, with its reason."""
    from momentum_b200 import torch_skeleton as tsk

    good, Kp = _fixture("chain6_edges_k8")
    dev = torch.device("cuda", 0)
    st = torch.from_numpy(tsn._states(good, 2, 99)).to(dev)
    for bad, reason in ((mc.BlendShape(good.blend_shape.base_shape, np.full_like(good.blend_shape.shape_vectors, np.nan)), "finite"),
                        (mc.BlendShape(good.blend_shape.base_shape, good.blend_shape.shape_vectors[:, :5]), "same V")):
        ch = copy.copy(good)
        ch.blend_shape = bad
        assert torch.equal(tsk.skin_points(ch, st), tsk.skin_points(good, st))
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(2, ch.num_params, device=dev))
        with pytest.raises(ValueError, match=reason):
            tsk.skin_with_blend_shapes(ch, st, torch.zeros(Kp, device=dev))
        dc = ms.DeviceCharacter(ch, 0)
        assert dc.blend_shape is None and dc.num_blend_shapes == 0 and reason in dc.blend_shape_error
        with pytest.raises(ValueError, match=reason):
            tsk.skin_with_blend_shapes(dc, st, torch.zeros(Kp, device=dev))
