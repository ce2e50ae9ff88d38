"""skin_points (linear-blend skinning) on the device and its backward, against float64 restatements.

References: the forward is compared with ``character.skin_points`` (float64 numpy, applySSD with q normalised); the gradients with
torch float64 autograd of the same math written in torch (``_skin64``), normalisation of q included. Bounds, K pinned at about four
times the worst value measured over the fixtures below on the emulator and on an H100:
  forward        |p - p64| <= K_F * 2^-24 * sum_k |w_k| (|Lin M_k| |x| + |t_k|)                      elementwise
  skel state     ||g_j - g64_j||_inf <= K_S * 2^-24 * sum_i |w_ij| |g_i| (|y_ij| + 1) max(1, s_j / |q_j|)   per joint
  rest points    ||g - g64||_inf <= K_R * max(||g64||_inf, 1)                                         per instance (or the batch sum)
The self-checks show that each bound rejects a skinning that drops the inverse-bind-pose translation or counts an influence twice, a
backward without the normalisation Jacobian, and E_j accumulated in the uncentred form on the fixture 100 units from the origin.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "emu")
EPS32 = 2.0 ** -24

# worst measured ratios over these fixtures, three seeds and the three rest-point layouts, on the emulator / on an H100 80GB HBM3 at a
# 700 W power limit: forward 30.4 / 11.0 (chain6_edges / humanoid72), skel state 12.3 / 11.3 (humanoid72_far both times), rest points
# 3.0e-7 / 2.7e-7 (humanoid72_far / bodyhands300); each K is about four times the larger
K_F = 128.0
K_S = 50.0
K_R = 1.2e-6


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _with_skin(ch, vertices_per_joint, seed):
    ch.skinning = mc.synthetic_skinning(ch, vertices_per_joint, seed)
    return ch


def _one_vertex():
    ch = mc.create_test_character(3)
    sk = mc.synthetic_skinning(ch, 1, 3)
    ch.skinning = mc.Skinning(sk.rest_vertices[:1], sk.skin_index[:1], sk.skin_weight[:1], sk.inverse_bind_pose)
    ch.name = "chain3_v1"
    return ch


def _far_humanoid():
    ch, _ = mc.humanoid72()
    ch.offsets = ch.offsets.copy()
    ch.offsets[0] += np.float32(100.0)
    ch.name = "humanoid72_far"
    return _with_skin(ch, 139, 7)


def _edge_mesh():
    """chain6 with vertices of exactly 1 and exactly 8 influences, weights that do not sum to 1, and non-zero slots after a zero weight
    (which must be ignored)."""
    ch = mc.create_test_character(6)
    sk = mc.synthetic_skinning(ch, 8, 9)
    rng = np.random.default_rng(9)
    V = sk.num_vertices
    idx = rng.integers(0, 6, (V, 8)).astype(np.int32)
    w = rng.uniform(0.05, 0.6, (V, 8)).astype(np.float32)  # sums far from 1
    w[0:4, 1:] = 0.0  # exactly one influence
    w[4:8, 3] = 0.0  # three, then non-zero garbage (indices out of range and a NaN weight too)
    idx[4:8, 4:] = [99, -1, 7, 1000]
    w[4:8, 6] = np.nan
    # the other vertices keep all eight slots
    ch.skinning = mc.Skinning(sk.rest_vertices, idx, w, sk.inverse_bind_pose)
    ch.name = "chain6_edges"
    return ch


FIXTURES = {
    "chain3": lambda: _with_skin(mc.create_test_character(3), 3, 1),
    "chain3_v1": _one_vertex,
    "humanoid72": lambda: _with_skin(mc.humanoid72()[0], 139, 2),
    "bodyhands300": lambda: _with_skin(mc.bodyhands300()[0], 67, 4),
    "humanoid72_far": _far_humanoid,
    "chain6_edges": _edge_mesh,
}
_cache = {}


def _fixture(name):
    if name not in _cache:
        _cache[name] = FIXTURES[name]()
    return _cache[name]


def _states(ch, B, seed):
    """Skeleton states of random poses, with |q| spread over [0.8, 1.25] (the skinning normalises q)."""
    rng = np.random.default_rng(seed)
    theta = rng.uniform(-0.5, 0.5, (B, ch.num_params))
    t, q, s = mc.forward_kinematics(ch, theta)
    q = q * rng.uniform(0.8, 1.25, q.shape[:-1] + (1,))
    return np.concatenate([t, q, s[..., None]], -1).astype(np.float32)


def _upstream(ch, B, seed):
    return np.random.default_rng(seed).normal(size=(B, ch.skinning.num_vertices, 3)).astype(np.float32)


# ---- float64 references ------------------------------------------------------------------------------------------------------------
def _active(sk):
    return np.cumprod(np.asarray(sk.skin_weight) != 0.0, axis=1).astype(bool)


def _quat_matrix_t(q):
    x, y, z, w = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _skin64(ch, st, x, normalise=True, ibp_translation=True, twice=False):
    """torch float64 skinning: st [B,J,8], x [B,V,3] -> [B,V,3]. The keyword arguments build the wrong variants of the self-checks."""
    sk = ch.skinning
    q = st[..., 3:7]
    qn = q / torch.linalg.norm(q, dim=-1, keepdim=True) if normalise else q
    sR = _quat_matrix_t(qn) * st[..., 7, None, None]
    ibp = torch.from_numpy(np.asarray(sk.inverse_bind_pose, np.float64))
    L = sR @ ibp[None, :, :, :3]
    c = (sR @ ibp[None, :, :, 3:])[..., 0] * (1.0 if ibp_translation else 0.0) + st[..., :3]
    act = _active(sk)
    out = torch.zeros_like(x)
    for k in range(mc.MAX_SKIN_JOINTS):
        j = torch.from_numpy(np.where(act[:, k], sk.skin_index[:, k], 0).astype(np.int64))
        wk = torch.from_numpy(np.where(act[:, k], sk.skin_weight[:, k], 0.0).astype(np.float64))
        mult = 2.0 if (twice and k == 0) else 1.0
        out = out + mult * (torch.einsum("bvrc,bvc->bvr", L[:, j], x) + c[:, j]) * wk[None, :, None]
    return out


def _rest(ch, B, batched, seed=None):
    x = np.asarray(ch.skinning.rest_vertices, np.float32)
    if seed is not None:
        x = x + np.random.default_rng(seed).normal(scale=0.5, size=x.shape).astype(np.float32)
    return np.ascontiguousarray(np.broadcast_to(x, (B,) + x.shape)) if batched else x


def _grads64(ch, st, x, G, **variant):
    """float64 (dL/dstate [B,J,8], dL/dx in x's layout) of L = sum(skin * G)."""
    s64 = torch.from_numpy(np.asarray(st, np.float64)).requires_grad_(True)
    x64 = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    xb = x64.expand(s64.shape[0], *x64.shape[-2:]) if x64.dim() == 2 else x64
    (_skin64(ch, s64, xb, **variant) * torch.from_numpy(np.asarray(G, np.float64))).sum().backward()
    return s64.grad.numpy(), x64.grad.numpy()


def _forward_ratio(ch, st, x, p):
    """max over elements of |p - p64| / (2^-24 sum_k |w_k| (|Lin M_k| |x| + |t_k|))"""
    sk = ch.skinning
    st64 = np.asarray(st, np.float64)
    xb = np.broadcast_to(np.asarray(x, np.float64), (st64.shape[0],) + np.shape(x)[-2:])
    qn = st64[..., 3:7] / np.linalg.norm(st64[..., 3:7], axis=-1, keepdims=True)
    sR = mc._quat_matrix(qn) * st64[..., 7, None, None]
    ibp = np.asarray(sk.inverse_bind_pose, np.float64)
    L = sR @ ibp[None, :, :, :3]
    c = (sR @ ibp[None, :, :, 3:])[..., 0] + st64[..., :3]
    act = _active(sk)
    scale = np.zeros_like(xb)
    for k in range(mc.MAX_SKIN_JOINTS):
        j = np.where(act[:, k], sk.skin_index[:, k], 0)
        wk = np.where(act[:, k], np.abs(sk.skin_weight[:, k]), 0.0)
        scale += (np.einsum("bvrc,bvc->bvr", np.abs(L[:, j]), np.abs(xb)) + np.abs(c[:, j])) * wk[None, :, None]
    p64 = mc.skin_points(ch, st, x)
    return float((np.abs(np.asarray(p, np.float64) - p64) / (EPS32 * scale)).max())


def _state_scale(ch, st, x, G):
    """per instance and joint: 2^-24 sum_i |w_ij| |g_i| (|y_ij| + 1) max(1, s_j / |q_j|)"""
    sk = ch.skinning
    B, J = st.shape[0], ch.num_joints
    xb = np.broadcast_to(np.asarray(x, np.float64), (B,) + np.shape(x)[-2:])
    ibp = np.asarray(sk.inverse_bind_pose, np.float64)
    act = _active(sk)
    den = np.zeros((B, J))
    gn = np.linalg.norm(np.asarray(G, np.float64), axis=-1)
    for k in range(mc.MAX_SKIN_JOINTS):
        v = np.nonzero(act[:, k])[0]
        j = sk.skin_index[v, k]
        y = np.einsum("vrc,bvc->bvr", ibp[j, :, :3], xb[:, v]) + ibp[j, :, 3]
        contrib = np.abs(sk.skin_weight[v, k]) * gn[:, v] * (np.linalg.norm(y, axis=-1) + 1.0)
        for b in range(B):
            np.add.at(den[b], j, contrib[b])
    st64 = np.asarray(st, np.float64)
    return EPS32 * den * np.maximum(1.0, st64[..., 7] / np.linalg.norm(st64[..., 3:7], axis=-1))


def _state_ratio(ch, st, x, G, g, g64):
    err = np.abs(np.asarray(g, np.float64) - g64).max(axis=-1)
    den = _state_scale(ch, st, x, G)
    return float(np.where(err > 0, err / np.maximum(den, 1e-300), 0.0).max())


def _rest_ratio(g, g64):
    g, g64 = np.asarray(g, np.float64), np.asarray(g64, np.float64)
    if g.ndim == 2:
        g, g64 = g[None], g64[None]
    return float((np.abs(g - g64).reshape(g.shape[0], -1).max(1) / np.maximum(np.abs(g64).reshape(g.shape[0], -1).max(1), 1.0)).max())


# ---- CPU: the emulator runs the device functions pass by pass -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("emu_skinning") / "libemu_skinning.so")
    csrc = os.path.join(ROOT, "momentum_b200", "csrc")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-ffp-contract=off", "--fmad=false", "-shared", "-o", lib,
                           os.path.join(EMU_DIR, "emu_skinning.cu"), os.path.join(csrc, "ik_plan.cpp"), os.path.join(csrc, "ik_chol_sched.cpp")])
    L = ctypes.CDLL(lib)
    L.emu_skinning_last_error.restype = ctypes.c_char_p
    head = [ctypes.c_int32] + [ctypes.c_void_p] * 3 + [ctypes.c_int32] + [ctypes.c_void_p] * 4 + [ctypes.c_int32] + [ctypes.c_void_p] * 4
    L.emu_skinning_tables.argtypes = head + [ctypes.c_void_p] * 2
    L.emu_skin_points.argtypes = head + [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p]
    L.emu_skin_points_backward.argtypes = head + [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 3
    return L


def _head(ch, keep, rest=None, index=None, weight=None, ibp=None):
    sk = ch.skinning
    arrays = [np.ascontiguousarray(ch.parents, np.int32), np.ascontiguousarray(ch.offsets, np.float32), np.ascontiguousarray(ch.prerot, np.float32),
              np.ascontiguousarray(ch.pt_outer, np.int32), np.ascontiguousarray(ch.pt_inner, np.int32), np.ascontiguousarray(ch.pt_vals, np.float32),
              np.ascontiguousarray(ch.pt_offsets, np.float32),
              np.ascontiguousarray(sk.rest_vertices if rest is None else rest, np.float32),
              np.ascontiguousarray(sk.skin_index if index is None else index, np.int32),
              np.ascontiguousarray(sk.skin_weight if weight is None else weight, np.float32),
              np.ascontiguousarray(sk.inverse_bind_pose if ibp is None else ibp, np.float32)]
    keep.extend(arrays)
    p = [a.ctypes.data for a in arrays]
    V = arrays[7].shape[0] if arrays[7].ndim == 2 else 0
    return [ch.num_joints] + p[:3] + [ch.num_params] + p[3:7] + [V] + p[7:]


def _ptr(a):
    return None if a is None else a.ctypes.data


def _emu_forward(L, ch, st, rest=None, batched=False):
    keep = []
    st = np.ascontiguousarray(st, np.float32)
    out = np.full((st.shape[0], ch.skinning.num_vertices, 3), np.nan, np.float32)
    rest = None if rest is None else np.ascontiguousarray(rest, np.float32)
    rc = L.emu_skin_points(*_head(ch, keep), st.shape[0], st.ctypes.data, _ptr(rest), int(batched), out.ctypes.data)
    assert rc == 0, L.emu_skinning_last_error().decode()
    return out


def _emu_backward(L, ch, st, rest, batched, G, want_rest=True):
    keep = []
    st, G = np.ascontiguousarray(st, np.float32), np.ascontiguousarray(G, np.float32)
    gs = np.full(st.shape, np.nan, np.float32)
    gr = np.full(np.shape(rest), np.nan, np.float32) if (rest is not None and want_rest) else None
    rest = None if rest is None else np.ascontiguousarray(rest, np.float32)
    rc = L.emu_skin_points_backward(*_head(ch, keep), st.shape[0], st.ctypes.data, _ptr(rest), int(batched), G.ctypes.data, gs.ctypes.data, _ptr(gr))
    assert rc == 0, L.emu_skinning_last_error().decode()
    return gs, gr


def test_numpy_and_torch_restatements_agree():
    for name in ("chain3", "humanoid72", "chain6_edges"):
        ch = _fixture(name)
        st = _states(ch, 2, 1)
        x = _rest(ch, 2, True, seed=3)
        p = mc.skin_points(ch, st, x)
        pt = _skin64(ch, torch.from_numpy(st.astype(np.float64)), torch.from_numpy(x.astype(np.float64))).numpy()
        assert np.abs(p - pt).max() <= 1e-12 * max(1.0, np.abs(p).max()), name
        assert np.array_equal(mc.skin_points(ch, st[0]), mc.skin_points(ch, st[:1])[0])


def test_synthetic_skinning_shape_and_influences():
    for name, verts in (("humanoid72", (9000, 11000)), ("bodyhands300", (19000, 21000))):
        ch = _fixture(name)
        sk = ch.skinning
        assert verts[0] <= sk.num_vertices <= verts[1], (name, sk.num_vertices)
        counts = _active(sk).sum(1)
        assert counts.min() == 1 and counts.max() <= 8 and (counts >= 4).any(), name
        assert np.allclose(sk.skin_weight.sum(1), 1.0, atol=1e-5)
        # the inverse bind pose undoes the rest pose: skinning the rest mesh at theta = 0 returns it
        t, q, s = mc.forward_kinematics(ch, np.zeros((1, ch.num_params)))
        st = np.concatenate([t, q, s[..., None]], -1)
        assert np.abs(mc.skin_points(ch, st)[0] - sk.rest_vertices).max() <= 1e-4


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_forward_and_backward_meet_the_bounds(emu, name):
    ch = _fixture(name)
    B = 3
    st = _states(ch, B, 11)
    G = _upstream(ch, B, 12)
    assert _forward_ratio(ch, st, ch.skinning.rest_vertices, _emu_forward(emu, ch, st)) <= K_F
    for batched in (False, True):
        x = _rest(ch, B, batched, seed=5)
        assert _forward_ratio(ch, st, x, _emu_forward(emu, ch, st, x, batched)) <= K_F, (name, batched)
        gs, gr = _emu_backward(emu, ch, st, x, batched, G)
        gs64, gr64 = _grads64(ch, st, x, G)
        assert _state_ratio(ch, st, x, G, gs, gs64) <= K_S, (name, batched)
        assert _rest_ratio(gr, gr64) <= K_R, (name, batched)


def test_slots_after_the_first_zero_weight_are_ignored(emu):
    ch = _fixture("chain6_edges")
    keep = []
    counts = np.zeros(ch.skinning.num_vertices, np.int32)
    nnz = ctypes.c_int32()
    assert emu.emu_skinning_tables(*_head(ch, keep), counts.ctypes.data, ctypes.byref(nnz)) == 0
    assert list(counts[:4]) == [1] * 4 and list(counts[4:8]) == [3] * 4 and (counts[8:] == 8).all()
    assert nnz.value == counts.sum()
    clean = ch.skinning.skin_weight.copy()
    clean[4:8, 4:] = 0.0
    idx = ch.skinning.skin_index.copy()
    idx[4:8, 4:] = 0
    st = _states(ch, 2, 3)
    ref = _emu_forward(emu, ch, st)
    import dataclasses
    cleaned = dataclasses.replace(ch, skinning=mc.Skinning(ch.skinning.rest_vertices, idx, clean, ch.skinning.inverse_bind_pose))
    assert np.array_equal(_emu_forward(emu, cleaned, st), ref)


def test_rejected_skinning_inputs(emu):
    ch = _fixture("chain3")
    sk = ch.skinning
    st = _states(ch, 1, 1)
    out = np.zeros((1, sk.num_vertices, 3), np.float32)

    def rc_msg(**kw):
        keep = []
        rc = emu.emu_skin_points(*_head(ch, keep, **kw), 1, st.ctypes.data, None, 0, out.ctypes.data)
        return rc, emu.emu_skinning_last_error().decode()

    bad_idx = sk.skin_index.copy(); bad_idx[1, 0] = ch.num_joints
    neg_idx = sk.skin_index.copy(); neg_idx[0, 0] = -1
    nan_w = sk.skin_weight.copy(); nan_w[2, 0] = np.nan
    inf_x = sk.rest_vertices.copy(); inf_x[0, 1] = np.inf
    nan_ibp = sk.inverse_bind_pose.copy(); nan_ibp[1, 2, 3] = np.nan
    for kw, msg in ((dict(index=bad_idx), "out of range"), (dict(index=neg_idx), "out of range"), (dict(weight=nan_w), "weights must be finite"),
                    (dict(rest=inf_x), "vertices must be finite"), (dict(ibp=nan_ibp), "bind poses must be finite"),
                    (dict(rest=np.zeros((0, 3), np.float32), index=np.zeros((0, 8), np.int32), weight=np.zeros((0, 8), np.float32)), "at least one vertex")):
        rc, m = rc_msg(**kw)
        assert rc == 1, kw  # MB2_ERR_INVALID_ARGUMENT
        assert msg in m, (msg, m)
    # the emulator refuses a rest-point gradient without rest points, like the C-ABI
    keep = []
    G = _upstream(ch, 1, 2)
    gr = np.zeros((sk.num_vertices, 3), np.float32)
    assert emu.emu_skin_points_backward(*_head(ch, keep), 1, st.ctypes.data, None, 0, G.ctypes.data, None, gr.ctypes.data) != 0


def test_bounds_reject_wrong_skinning():
    """Each bound against the mistake it is there to catch, measured on the float64 references and float32 emulations of the wrong forms."""
    for name in ("humanoid72", "humanoid72_far"):
        ch = _fixture(name)
        B = 2
        st = _states(ch, B, 21)
        x = _rest(ch, B, False)
        xb = torch.from_numpy(np.broadcast_to(x.astype(np.float64), (B,) + x.shape).copy())
        s64 = torch.from_numpy(st.astype(np.float64))
        for variant in (dict(ibp_translation=False), dict(twice=True)):
            p_wrong = _skin64(ch, s64, xb, **variant).numpy()
            assert _forward_ratio(ch, st, x, p_wrong) > 100 * K_F, (name, variant)
        G = _upstream(ch, B, 22)
        gs64, gr64 = _grads64(ch, st, x, G)
        # without the normalisation Jacobian: the gradient with respect to q^ taken as the input
        qn = st.astype(np.float64).copy()
        qn[..., 3:7] /= np.linalg.norm(qn[..., 3:7], axis=-1, keepdims=True)
        g_hat, _ = _grads64(ch, qn, x, G, normalise=False)
        wrong = gs64.copy(); wrong[..., 3:7] = g_hat[..., 3:7]
        assert _state_ratio(ch, st, x, G, wrong, gs64) > 100 * K_S, name
        twice_s, twice_r = _grads64(ch, st, x, G, twice=True)
        assert _state_ratio(ch, st, x, G, twice_s, gs64) > 100 * K_S and _rest_ratio(twice_r, gr64) > 100 * K_R, name
    # E_j accumulated as (sum w g x^T) N^T + a c^T in float32 on the fixture 100 units out
    ch = _fixture("humanoid72_far")
    sk = ch.skinning
    st = _states(ch, 1, 23)
    G = _upstream(ch, 1, 24)
    gs64, _ = _grads64(ch, st, sk.rest_vertices, G)
    J = ch.num_joints
    act = _active(sk)
    X = np.zeros((J, 3, 3), np.float32); a = np.zeros((J, 3), np.float32)
    for k in range(mc.MAX_SKIN_JOINTS):
        v = np.nonzero(act[:, k])[0]
        j = sk.skin_index[v, k]
        wg = (sk.skin_weight[v, k, None] * G[0, v]).astype(np.float32)
        for jj, w_g, xx in zip(j, wg, sk.rest_vertices[v]):
            X[jj] += np.outer(w_g, xx).astype(np.float32)
            a[jj] += w_g
    ibp = sk.inverse_bind_pose.astype(np.float32)
    E = (X @ np.swapaxes(ibp[:, :, :3], 1, 2) + a[:, :, None] * ibp[:, None, :, 3]).astype(np.float64)
    # the final step in float64 from the uncentred E: only the accumulation differs from the reference
    q = st[0, :, 3:7].astype(np.float64)
    nq = np.linalg.norm(q, axis=-1, keepdims=True)
    u = torch.from_numpy(q / nq).requires_grad_(True)
    f = (torch.from_numpy(E) * _quat_matrix_t(u)).sum((-1, -2)) * torch.from_numpy(st[0, :, 7].astype(np.float64))
    f.sum().backward()
    gu = u.grad.numpy()
    gq = (gu - (q / nq) * (gu * q / nq).sum(-1, keepdims=True)) / nq
    uncentred = gs64.copy()
    uncentred[0, :, 3:7] = gq
    uncentred[0, :, 7] = (E * mc._quat_matrix(q / nq)).sum((-1, -2))
    assert _state_ratio(ch, st, sk.rest_vertices, G, uncentred, gs64) > K_S


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = _fixture("chain3")
    with pytest.raises(ValueError, match="CUDA"):
        tsk.skin_points(ch, torch.zeros(ch.num_joints, 8))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_forward(dc, st, rest=None, batched=False):
    B = st.shape[0]
    out = torch.empty(B, dc.skinning.num_vertices, 3, device=st.device)
    dc.skin_points_device(B, st.data_ptr(), 0 if rest is None else rest.data_ptr(), batched, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out


def _device_backward(dc, st, rest, batched, G, want_state=True, want_rest=True):
    B = st.shape[0]
    gs = torch.empty_like(st) if want_state else None
    gr = torch.empty_like(rest) if (rest is not None and want_rest) else None
    dc.skin_points_backward_device(B, st.data_ptr(), 0 if rest is None else rest.data_ptr(), batched, G.data_ptr(), 0 if gs is None else gs.data_ptr(),
                                   0 if gr is None else gr.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return gs, gr


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_forward_and_backward_meet_the_bounds(name):
    ch = _fixture(name)
    dc = ms.DeviceCharacter(ch, 0)
    B = 5
    st = _states(ch, B, 31)
    G = _upstream(ch, B, 32)
    std, Gd = _dev(st), _dev(G)
    assert _forward_ratio(ch, st, ch.skinning.rest_vertices, _device_forward(dc, std).cpu().numpy()) <= K_F, name
    gs, gr = _device_backward(dc, std, None, False, Gd)
    assert gr is None
    gs64, _ = _grads64(ch, st, ch.skinning.rest_vertices, G)
    assert _state_ratio(ch, st, ch.skinning.rest_vertices, G, gs.cpu().numpy(), gs64) <= K_S, name
    for batched in (False, True):
        x = _rest(ch, B, batched, seed=6)
        xd = _dev(x)
        assert _forward_ratio(ch, st, x, _device_forward(dc, std, xd, batched).cpu().numpy()) <= K_F, (name, batched)
        gs, gr = _device_backward(dc, std, xd, batched, Gd)
        gs64, gr64 = _grads64(ch, st, x, G)
        assert _state_ratio(ch, st, x, G, gs.cpu().numpy(), gs64) <= K_S, (name, batched)
        assert _rest_ratio(gr.cpu().numpy(), gr64) <= K_R, (name, batched)
        # each output alone gives the same bits
        gs_only, _ = _device_backward(dc, std, xd, batched, Gd, want_rest=False)
        _, gr_only = _device_backward(dc, std, xd, batched, Gd, want_state=False)
        assert torch.equal(gs_only, gs) and torch.equal(gr_only, gr)


@pytest.mark.gpu
def test_large_batch_determinism_and_bounds():
    ch = _fixture("humanoid72")
    dc = ms.DeviceCharacter(ch, 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 3 * sms * 8 + 37  # three waves of the widest launch (eight 256-thread CTAs per SM) and a remainder
    st = _states(ch, B, 41)
    G = _upstream(ch, B, 42)
    std, Gd = _dev(st), _dev(G)
    xs = _dev(_rest(ch, B, False, seed=7))
    xb = _dev(_rest(ch, B, True, seed=7))
    p1, p2 = _device_forward(dc, std), _device_forward(dc, std)
    s1, r1 = _device_backward(dc, std, xs, False, Gd)
    s2, r2 = _device_backward(dc, std, xs, False, Gd)
    sb, rb = _device_backward(dc, std, xb, True, Gd)
    assert torch.equal(p1, p2) and torch.equal(s1, s2) and torch.equal(r1, r2)
    sample = [0, 1, B // 3, B // 2, B - 38, B - 1]
    for b in sample:
        one = slice(b, b + 1)
        assert torch.equal(_device_forward(dc, std[one].contiguous()), p1[one]), b
        sg, rg = _device_backward(dc, std[one].contiguous(), xb[one].contiguous(), True, Gd[one].contiguous())
        assert torch.equal(sg, sb[one]) and torch.equal(rg, rb[one]), b
        sg, _ = _device_backward(dc, std[one].contiguous(), xs, False, Gd[one].contiguous(), want_rest=False)
        assert torch.equal(sg, s1[one]), b
    sub = np.array(sample[:4])
    x = _rest(ch, B, False, seed=7)
    assert _forward_ratio(ch, st[sub], ch.skinning.rest_vertices, p1[sub].cpu().numpy()) <= K_F
    gs64, _ = _grads64(ch, st[sub], x, G[sub])
    assert _state_ratio(ch, st[sub], x, G[sub], s1[sub].cpu().numpy(), gs64) <= K_S
    _, gr64 = _grads64(ch, st, x, G)  # the batch sum over all B instances
    assert _rest_ratio(r1.cpu().numpy(), gr64) <= K_R


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_and_counts_vertices():
    ch = _fixture("chain3")
    bare = mc.Character(ch.parents, ch.offsets, ch.prerot, ch.num_params, ch.pt_outer, ch.pt_inner, ch.pt_vals, ch.pt_offsets, [], "bare")
    dc = ms.DeviceCharacter(bare, 0)
    V, J = ch.skinning.num_vertices, ch.num_joints
    st = torch.zeros(2, J, 8, device="cuda"); st[..., 6] = 1; st[..., 7] = 1
    out = torch.zeros(2, V, 3, device="cuda")
    assert dc.num_vertices == 0
    with pytest.raises(ms.MomentumB200Error, match="no skinning"):
        dc.skin_points_device(2, st.data_ptr(), 0, False, out.data_ptr())
    dc.set_skinning(ch.skinning)
    assert dc.num_vertices == V
    host = np.zeros((2, V, 3), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        dc.skin_points_device(2, st.data_ptr(), 0, False, host.ctypes.data)
    with pytest.raises(ms.MomentumB200Error, match="null"):
        dc.skin_points_device(2, 0, 0, False, out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="negative"):
        dc.skin_points_device(-1, st.data_ptr(), 0, False, out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null"):
        dc.skin_points_backward_device(2, st.data_ptr(), 0, False, 0, st.data_ptr(), 0)
    with pytest.raises(ms.MomentumB200Error, match="must be null"):
        dc.skin_points_backward_device(2, st.data_ptr(), 0, False, out.data_ptr(), 0, out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="out of range"):
        bad = mc.Skinning(ch.skinning.rest_vertices, np.full_like(ch.skinning.skin_index, J), ch.skinning.skin_weight, ch.skinning.inverse_bind_pose)
        dc.set_skinning(bad)
    assert dc.num_vertices == V  # a rejected skinning leaves the earlier one
    dc.skin_points_device(0, 0, 0, False, 0)  # batch 0: nothing to do
    dc.skin_points_backward_device(0, 0, 0, False, 0, 0, 0)
    small = mc.Skinning(ch.skinning.rest_vertices[:2], ch.skinning.skin_index[:2], ch.skinning.skin_weight[:2], ch.skinning.inverse_bind_pose)
    dc.set_skinning(small)
    assert dc.num_vertices == 2


@pytest.mark.gpu
def test_cloned_character_skins_identically():
    ch = _fixture("chain6_edges")
    dc = ms.DeviceCharacter(ch, 0)
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        assert dc._L.mb2_character_num_vertices(clone) == ch.skinning.num_vertices
        st = _dev(_states(ch, 3, 51))
        G = _dev(_upstream(ch, 3, 52))
        x = _dev(_rest(ch, 3, False, seed=8))
        outs = []
        for h in (dc._h, clone):
            p = torch.empty(3, ch.skinning.num_vertices, 3, device="cuda")
            gs, gr = torch.empty_like(st), torch.empty_like(x)
            dc._check(dc._L.mb2_character_skin_points_device(h, 3, ms.C.c_void_p(st.data_ptr()), None, 0, ms.C.c_void_p(p.data_ptr()), None))
            dc._check(dc._L.mb2_character_skin_points_backward_device(h, 3, ms.C.c_void_p(st.data_ptr()), ms.C.c_void_p(x.data_ptr()), 0,
                                                                      ms.C.c_void_p(G.data_ptr()), ms.C.c_void_p(gs.data_ptr()), ms.C.c_void_p(gr.data_ptr()), None))
            outs.append((p, gs, gr))
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(*outs))
    finally:
        dc._L.mb2_character_destroy(clone)


@pytest.mark.gpu
def test_torch_wrapper():
    from momentum_b200 import torch_skeleton as tsk

    ch = _fixture("humanoid72")
    J, V = ch.num_joints, ch.skinning.num_vertices
    dev = torch.device("cuda", 0)
    st, G = _states(ch, 3, 61), _upstream(ch, 3, 62)
    # float64 in -> float64 out, the rest mesh by default, gradients to the skel state
    s64 = torch.from_numpy(st.astype(np.float64)).to(dev).requires_grad_(True)
    p = tsk.skin_points(ch, s64)
    assert p.shape == (3, V, 3) and p.dtype == torch.float64 and p.is_cuda
    assert _forward_ratio(ch, st, ch.skinning.rest_vertices, p.detach().cpu().numpy()) <= K_F
    p.backward(torch.from_numpy(G.astype(np.float64)).to(dev))
    gs64, _ = _grads64(ch, st, ch.skinning.rest_vertices, G)
    assert s64.grad.dtype == torch.float64 and _state_ratio(ch, st, ch.skinning.rest_vertices, G, s64.grad.cpu().numpy(), gs64) <= K_S
    # [J, 8]
    s1 = torch.from_numpy(st[1]).to(dev).requires_grad_(True)
    p1 = tsk.skin_points(ch, s1)
    assert p1.shape == (V, 3) and torch.equal(p1, p[1].float())
    p1.backward(torch.from_numpy(G[1]).to(dev))
    assert s1.grad.shape == (J, 8)
    # shared and batched rest points
    for batched in (False, True):
        x = _rest(ch, 3, batched, seed=9)
        xt = torch.from_numpy(x).to(dev).requires_grad_(True)
        sf = torch.from_numpy(st).to(dev).requires_grad_(True)
        tsk.skin_points(ch, sf, xt).backward(torch.from_numpy(G).to(dev))
        gs64, gr64 = _grads64(ch, st, x, G)
        assert xt.grad.shape == x.shape and _rest_ratio(xt.grad.cpu().numpy(), gr64) <= K_R, batched
        assert _state_ratio(ch, st, x, G, sf.grad.cpu().numpy(), gs64) <= K_S, batched
    # batch 0
    s0 = torch.zeros(0, J, 8, device=dev, requires_grad=True)
    p0 = tsk.skin_points(ch, s0)
    assert p0.shape == (0, V, 3)
    p0.sum().backward()
    assert s0.grad.shape == (0, J, 8)
    # a side stream gives the same bits
    sf = torch.from_numpy(st).to(dev).requires_grad_(True)
    ref = tsk.skin_points(ch, sf)
    ref.backward(torch.from_numpy(G).to(dev))
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        ss = torch.from_numpy(st).to(dev).requires_grad_(True)
        out = tsk.skin_points(ch, ss)
        out.backward(torch.from_numpy(G).to(dev))
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    assert torch.equal(out, ref) and torch.equal(ss.grad, sf.grad)
    # a replaced skinning is uploaded again, not served from the cached handle
    import copy
    ch2 = copy.copy(ch)
    ch2.skinning = ch.skinning
    first = tsk.skin_points(ch2, sf.detach())
    moved = mc.Skinning(ch.skinning.rest_vertices + np.float32(1.0), ch.skinning.skin_index, ch.skinning.skin_weight, ch.skinning.inverse_bind_pose)
    ch2.skinning = moved
    second = tsk.skin_points(ch2, sf.detach())
    assert torch.equal(first, ref.detach()) and not torch.equal(second, first)
    assert _forward_ratio(ch2, st, moved.rest_vertices, second.cpu().numpy()) <= K_F
    smaller = mc.Skinning(moved.rest_vertices[:10], moved.skin_index[:10], moved.skin_weight[:10], moved.inverse_bind_pose)
    ch2.skinning = smaller
    assert tsk.skin_points(ch2, sf.detach()).shape == (3, 10, 3)
    # the ValueError cases
    with pytest.raises(ValueError, match="CUDA"):
        tsk.skin_points(ch, torch.from_numpy(st))
    with pytest.raises(ValueError, match="4x4"):
        tsk.skin_points(ch, torch.zeros(3, J, 4, 4, device=dev))
    with pytest.raises(ValueError, match="must be"):
        tsk.skin_points(ch, torch.zeros(3, J + 1, 8, device=dev))
    with pytest.raises(ValueError, match="rest_points must be"):
        tsk.skin_points(ch, torch.zeros(3, J, 8, device=dev), torch.zeros(V + 1, 3, device=dev))
    with pytest.raises(ValueError, match="rest_points must be"):
        tsk.skin_points(ch, torch.zeros(3, J, 8, device=dev), torch.zeros(2, V, 3, device=dev))
    with pytest.raises(ValueError, match="no skinning"):
        tsk.skin_points(mc.create_test_character(3), torch.zeros(3, 8, device=dev))


@pytest.mark.gpu
def test_replacing_the_skinning_keeps_recorded_graphs_whole():
    """A graph recorded with skinning A back-propagates with A after character.skinning is replaced by a larger B and B is used; a graph
    recorded on a DeviceCharacter whose skinning is then replaced by set_skinning refuses its backward."""
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    A = mc.synthetic_skinning(ch, 20, 71)
    Bk = mc.synthetic_skinning(ch, 40, 72)
    ch.skinning = A
    st, G = _states(ch, 2, 73), _upstream(ch, 2, 74)
    x = _rest(ch, 2, False, seed=75)
    dev = torch.device("cuda", 0)
    sa = torch.from_numpy(st).to(dev).requires_grad_(True)
    xa = torch.from_numpy(x).to(dev).requires_grad_(True)
    pa = tsk.skin_points(ch, sa, xa)
    ch.skinning = Bk
    pb = tsk.skin_points(ch, torch.from_numpy(st).to(dev))
    assert pb.shape == (2, Bk.num_vertices, 3)
    assert _forward_ratio(ch, st, Bk.rest_vertices, pb.cpu().numpy()) <= K_F
    pa.backward(torch.from_numpy(G).to(dev))
    ch.skinning = A
    gs64, gr64 = _grads64(ch, st, x, G)
    assert _state_ratio(ch, st, x, G, sa.grad.cpu().numpy(), gs64) <= K_S
    assert _rest_ratio(xa.grad.cpu().numpy(), gr64) <= K_R
    # the same through one DeviceCharacter: set_skinning after the forward makes that graph's backward raise
    dc = ms.DeviceCharacter(ch, 0)
    sd = torch.from_numpy(st).to(dev).requires_grad_(True)
    pd = tsk.skin_points(dc, sd)
    dc.set_skinning(Bk)
    with pytest.raises(RuntimeError, match="replaced"):
        pd.backward(torch.from_numpy(G).to(dev))
    assert tsk.skin_points(dc, sd.detach()).shape == (2, Bk.num_vertices, 3)


@pytest.mark.gpu
def test_solve_ik_then_skin_points_matches_finite_differences():
    """solve_ik -> model_parameters_to_skeleton_state -> skin_points -> a loss on the vertices: the position-target gradient of the
    whole pipeline against central differences, on the zero-residual problem where the solver's implicit-function derivative is exact."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    ch.skinning = mc.synthetic_skinning(ch, 20, 5)
    rng = np.random.default_rng(4)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)
    wv = torch.from_numpy(rng.normal(size=(ch.skinning.num_vertices, 3))).to(dev)

    def pipeline(tg):
        theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                            position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
        pts = tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, theta.double()))
        return (pts * wv).sum() + 0.05 * (pts ** 2).sum()

    tg = torch.from_numpy(targets).to(dev).double().requires_grad_(True)
    pipeline(tg).backward()
    g_tg = tg.grad.clone()
    assert g_tg.abs().max().item() > 0.0
    eps = 5e-3
    with torch.no_grad():
        for (b, c, k) in [(0, 0, 0), (0, 3, 1), (1, 5, 2), (1, 7, 0)]:
            d = torch.zeros_like(tg); d[b, c, k] = eps
            fd = (pipeline(tg + d).item() - pipeline(tg - d).item()) / (2 * eps)
            assert abs(fd - g_tg[b, c, k].item()) <= 0.1 * max(abs(fd), abs(g_tg[b, c, k].item()), 0.05), ("target", b, c, k, fd, g_tg[b, c, k].item())
