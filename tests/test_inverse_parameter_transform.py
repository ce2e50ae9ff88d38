"""apply_inverse_parameter_transform on the device: theta = W (jp - o), W = P^+ the ParameterTransform's Moore-Penrose pseudo-inverse
with the absolute truncation of InverseParameterTransform (a singular value > 1e-6 is inverted, any other is 0), and its backward W^T.

The reference W64 is a float64 numpy SVD pseudo-inverse with that rule, taken per connected component of P's sparsity graph (the same
matrix as the SVD of all of P, which the matrix test also checks, without its rounding noise in the entries that are 0 by structure).
A forward passes when, per element, |theta_p - theta64_p| <= K_FWD * sum_k |W64_pk (jp_k - o_k)|, a backward when
|g_r - g64_r| <= K_BWD * sum_p |W64_pr g_p|, with theta64 = W64 (jp - o) and g64 = W64^T g on the float32 inputs. Each K is pinned at about
four times the worst value measured over the fixtures and seeds (emulator / H100, in the comments). The self-checks show that the bounds
reject a W without the truncation, a W under a relative cut-off, a forward that ignores the offsets and a backward that applies P
instead of W^T.
"""
import ctypes
import math
import time

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_joint_parameters import _fk64, _joint_params, _ref64
from tests.test_skeleton_state import FIXTURES as _SKELETON_FIXTURES
from tests.test_skeleton_state import _pt_dense

OP = "apply_inverse_parameter_transform"  # its entry in solver.JOINT_OPS
U32 = 2.0 ** -24  # float32 unit roundoff

# worst measured ratio over the fixtures and seeds, emulator / H100 80GB HBM3 at a 700 W power limit -> the pinned bound, about four
# times the larger (the coupled character both times); the wrong implementations of the self-checks reach >= 1
K_FWD = 5.5e-7  # 1.31e-7 / 9.71e-8
K_BWD = 6e-7    # 1.41e-7 / 1.41e-7


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _coupled():
    """Six joints whose ParameterTransform has every kind of component: a global scale on every scale row, one parameter on three rows
    with different coefficients, one row driven by three parameters, a 6 x 10 dense block with condition number 1e3, two identical
    columns, an empty column, singleton columns at 1e-7 (below the threshold) and 1e-5 (kept), undriven rows and non-zero offsets."""
    rng = np.random.default_rng(2024)
    J = 6
    parents = np.array([-1, 0, 1, 2, 1, 4], np.int32)
    offsets = rng.uniform(-1, 1, (J, 3)).astype(np.float32)
    prerot = np.stack([mc._random_prerot(rng) for _ in range(J)]).astype(np.float32)
    trip, p = [], 0

    def new():
        nonlocal p
        p += 1
        return p - 1

    scale = new()
    trip += [(7 * j + 6, scale, 1.0) for j in range(J)]
    three = new()
    trip += [(0, three, 1.0), (1, three, -2.5), (2, three, 30.0)]  # sigma = 30.1: a relative cut-off of 1e-6 drops the 1e-5 column
    trip += [(3 + d, new(), 1.0) for d in range(3)]
    trip += [(7 * 1 + 3, new(), c) for c in (1.0, 0.5, -0.25)]
    trip += [(7 * 1 + d, new(), 1.0) for d in range(3)]  # rows 7 + 4, 7 + 5 are driven by nothing
    Uq, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    Vq, _ = np.linalg.qr(rng.normal(size=(10, 6)))
    dense = (Uq * np.logspace(0, -3, 6)) @ Vq.T
    cols = [new() for _ in range(10)]
    trip += [(7 * 2 + r, cols[c], float(dense[r, c])) for r in range(6) for c in range(10)]
    twin = [new(), new()]
    trip += [(7 * 3 + r, t, c) for t in twin for r, c in ((0, 1.0), (1, 0.3))]
    new()  # the empty column
    trip += [(7 * 3 + 3, new(), 1e-7), (7 * 3 + 4, new(), 1e-5)]
    trip += [(7 * j + d, new(), 1.0) for j in (4, 5) for d in range(6)]
    outer, inner, vals = mc._csr_from_triplets(7 * J, p, trip)
    pt_offsets = rng.uniform(-0.2, 0.2, 7 * J).astype(np.float32)
    return mc.Character(parents, offsets, prerot, p, outer, inner, vals, pt_offsets, [], "coupled")


FIXTURES = dict(_SKELETON_FIXTURES, coupled=_coupled)
# the fixtures whose P has full column rank (checked below); two_roots' shared parameter drives two rows that have their own parameters
FULL_RANK = [name for name in _SKELETON_FIXTURES if name != "two_roots"]


def _stress():
    """bodyhands300's skeleton with P one dense random [7 J, n] block: the largest component a rig of that size can have"""
    ch = mc.bodyhands300()[0]
    rng = np.random.default_rng(7)
    J, n = ch.num_joints, ch.num_params
    dense = rng.normal(size=(7 * J, n)).astype(np.float32)
    outer = (np.arange(7 * J + 1) * n).astype(np.int32)
    inner = np.tile(np.arange(n, dtype=np.int32), 7 * J)
    return mc.Character(ch.parents, ch.offsets, ch.prerot, n, outer, inner, dense.reshape(-1), ch.pt_offsets, [], "stress_dense")


# ---- float64 reference -------------------------------------------------------------------------------------------------------------
def _pinv_abs(A, tol=1e-6):
    """Moore-Penrose pseudo-inverse with the absolute rule: sigma > tol inverted, any other 0"""
    if A.size == 0:
        return np.zeros(A.T.shape)
    U, S, Vt = np.linalg.svd(A, full_matrices=False)
    return (Vt.T * np.where(S > tol, 1.0 / np.where(S > tol, S, 1.0), 0.0)) @ U.T


def _components(ch):
    """the connected components of P's sparsity graph: [(rows, parameters)], each ascending"""
    R, n = 7 * ch.num_joints, ch.num_params
    rows = np.repeat(np.arange(R), np.diff(ch.pt_outer))
    g = scipy.sparse.coo_matrix((np.ones(rows.size), (rows, R + ch.pt_inner.astype(np.int64))), shape=(R + n, R + n))
    _, label = scipy.sparse.csgraph.connected_components(g, directed=False)
    out = []
    for c in np.unique(label[R:]):
        out.append((np.flatnonzero(label[:R] == c), np.flatnonzero(label[R:] == c)))
    return out


def _w64(ch, pinv=_pinv_abs):
    """W = P^+ [n, 7 J] float64, block by block"""
    P = _pt_dense(ch).numpy()
    W = np.zeros(P.T.shape)
    for r, c in _components(ch):
        W[np.ix_(c, r)] = pinv(P[np.ix_(r, c)])
    return W


def _fwd_ratio(ch, W64, jp, theta, offsets=True):
    """per instance: max_p |theta_p - theta64_p| / sum_k |W64_pk (jp_k - o_k)|"""
    d = np.asarray(jp, np.float64) - (ch.pt_offsets.astype(np.float64) if offsets else 0.0)
    ref, mag = d @ W64.T, np.abs(d) @ np.abs(W64).T
    return (np.abs(np.asarray(theta, np.float64) - ref) / np.maximum(mag, 1e-300)).max(1)


def _bwd_ratio(W64, g, gjp):
    """per instance: max_r |g_r - (W64^T g)_r| / sum_p |W64_pr g_p|"""
    g = np.asarray(g, np.float64)
    ref, mag = g @ W64, np.abs(g) @ np.abs(W64)
    return (np.abs(np.asarray(gjp, np.float64) - ref) / np.maximum(mag, 1e-300)).max(1)


def _inputs(ch, B, seed):
    """jp [B, 7 J] around P theta + o plus noise off the range of P, and g [B, n], float32"""
    rng = np.random.default_rng(seed)
    jp = _joint_params(ch, B, seed).reshape(B, -1) + ch.pt_offsets
    return jp.astype(np.float32), rng.normal(size=(B, ch.num_params)).astype(np.float32)


# ---- the two implementations: the CPU emulator and the device through the torch wrapper ------------------------------------------------
# the entry of tests/emu/emu_inverse_parameter_transform.cu (the nine character values, backward, batch, in, grad, out), declared here
# next to the only tests that call it
_EMU_SIGNATURE = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4 + \
    [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 3


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_inverse_parameter_transform.argtypes = _EMU_SIGNATURE
    return L


def _emu_run(L, ch, x, backward=False):
    """forward: theta [B, n] of jp x [B, 7 J]; backward: dLoss / d jp [B, 7 J] of dLoss / d theta x [B, n]"""
    keep = []
    x = np.ascontiguousarray(x, np.float32)
    B = x.shape[0]
    out = np.full((B, 7 * ch.num_joints if backward else ch.num_params), np.nan, np.float32)
    rc = L.emu_inverse_parameter_transform(*emu_lib.character_args(ch, keep), int(backward), B, None if backward else x.ctypes.data,
                                           x.ctypes.data if backward else None, out.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return out


def _dev_run(ch, x, backward=False):
    from momentum_b200 import torch_skeleton as tsk

    if not backward:
        return tsk.apply_inverse_parameter_transform(ch, torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()).cpu().numpy()
    jp = torch.zeros(x.shape[0], 7 * ch.num_joints, device="cuda", requires_grad=True)
    tsk.apply_inverse_parameter_transform(ch, jp).backward(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda())
    return jp.grad.cpu().numpy()


def _measure(run, ch, B=16, seed=31):
    W64 = _w64(ch)
    jp, g = _inputs(ch, B, seed)
    return _fwd_ratio(ch, W64, jp, run(ch, jp)).max(), _bwd_ratio(W64, g, run(ch, g, True)).max()


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_fixture_ranks():
    """FULL_RANK really has full column rank; the coupled character does not (the three parameters of one row, the 6 x 10 block, the
    identical columns, the empty and the truncated one)"""
    for name in FULL_RANK:
        ch = FIXTURES[name]()
        assert np.linalg.matrix_rank(_pt_dense(ch).numpy(), tol=1e-6) == ch.num_params, name
    ch = _coupled()
    assert np.linalg.matrix_rank(_pt_dense(ch).numpy(), tol=1e-6) == ch.num_params - 9
    ch = FIXTURES["two_roots"]()
    assert np.linalg.matrix_rank(_pt_dense(ch).numpy(), tol=1e-6) == ch.num_params - 1


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_matrix_is_the_truncated_pseudo_inverse(emu, fixture):
    """the forward on the 7 J unit vectors with zero offsets is W^T: each entry is W64's rounded to float (the Gram eigen-solve adds at
    most 1e-9 of its row's largest entry), W64 equals numpy's SVD of all of P, and W satisfies the four Moore-Penrose identities (P W P = P
    up to the truncated singular values, at most 1e-6)"""
    ch = FIXTURES[fixture]()
    ch.pt_offsets = np.zeros_like(ch.pt_offsets)
    R = 7 * ch.num_joints
    W = _emu_run(emu, ch, np.eye(R, dtype=np.float32)).T.astype(np.float64)
    W64 = _w64(ch)
    P = _pt_dense(ch).numpy()
    assert np.abs(W64 - _pinv_abs(P)).max() <= 1e-9 * max(1.0, np.abs(W64).max())
    row = np.abs(W64).max(1, keepdims=True)
    assert np.all(np.abs(W - W64) <= U32 * np.abs(W64) + 1e-9 * row), np.abs(W - W64).max()
    assert np.all((W64 == 0) <= (W == 0))  # structure: nothing outside the components
    aP, aW = np.abs(P), np.abs(W)
    assert np.all(np.abs(P @ W @ P - P) <= 4 * U32 * (aP @ aW @ aP) + 1e-6)
    assert np.all(np.abs(W @ P @ W - W) <= 4 * U32 * (aW @ aP @ aW + aW) + 1e-12)
    assert np.all(np.abs(P @ W - (P @ W).T) <= 4 * U32 * (aP @ aW + (aP @ aW).T) + 1e-12)
    assert np.all(np.abs(W @ P - (W @ P).T) <= 4 * U32 * (aW @ aP + (aW @ aP).T) + 1e-12)


def test_emulated_coupled_entries():
    """the coupled character's components as constructed: an even split of the identical columns, 1 / (J s) for the global scale, a
    zero row for the empty and the truncated column, 1e5 for the kept one"""
    L = emu_lib.load()
    L.emu_inverse_parameter_transform.argtypes = _EMU_SIGNATURE
    ch = _coupled()
    ch.pt_offsets = np.zeros_like(ch.pt_offsets)
    W = _emu_run(L, ch, np.eye(7 * ch.num_joints, dtype=np.float32)).T
    J, n = ch.num_joints, ch.num_params
    np.testing.assert_allclose(W[0, 6::7], 1.0 / J, rtol=U32)
    twin, empty, tiny, small = n - 17, n - 15, n - 14, n - 13
    np.testing.assert_array_equal(W[twin], W[twin + 1])
    np.testing.assert_allclose(W[twin, 7 * 3] * 2 * (1 + 0.09), 1.0, rtol=4 * U32)
    assert not W[empty].any() and not W[tiny].any()
    assert W[small, 7 * 3 + 4] == np.float32(1e5) and np.count_nonzero(W[small]) == 1


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_operation_meets_the_float64_bounds(emu, fixture):
    fwd, bwd = _measure(lambda ch, x, b=False: _emu_run(emu, ch, x, b), FIXTURES[fixture]())
    print(f"{fixture}: forward {fwd:.3g}, backward {bwd:.3g}")
    assert fwd <= K_FWD and bwd <= K_BWD


def test_bounds_reject_wrong_implementations():
    """no truncation, a relative cut-off, ignoring the offsets, and P in place of W^T in the backward"""
    ch = _coupled()
    W64 = _w64(ch)
    P = _pt_dense(ch).numpy()
    jp, g = _inputs(ch, 8, 41)
    d = jp.astype(np.float64) - ch.pt_offsets
    assert _fwd_ratio(ch, W64, jp, d @ W64.T).max() <= K_FWD  # the exact product passes
    untruncated = _w64(ch, lambda A: _pinv_abs(A, 0.0))
    relative = scipy.linalg.pinv(P, atol=0.0, rtol=1e-6)
    assert np.abs(untruncated).max() >= 1e7 and not relative[-13].any()
    for wrong in (d @ untruncated.T, d @ relative.T, jp.astype(np.float64) @ W64.T):
        assert _fwd_ratio(ch, W64, jp, wrong).min() > 1e3 * K_FWD
    assert _bwd_ratio(W64, g, g.astype(np.float64) @ P.T).min() > 1e3 * K_BWD


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_round_trips(emu, fixture):
    """inverse(apply(theta)) = P^+ P theta (theta on the full-rank fixtures), apply(inverse(jp)) = jp on the range of P plus o, and the
    adjoint identity <g, F(jp)> = <F^T g, jp> with zero offsets"""
    ch = FIXTURES[fixture]()
    rng = np.random.default_rng(51)
    B, n = 8, ch.num_params
    P, W64 = _pt_dense(ch).numpy(), _w64(ch)
    o = ch.pt_offsets.astype(np.float64)
    theta = rng.uniform(-0.5, 0.5, (B, n))
    jp = (theta @ P.T + o).astype(np.float32)
    back = _emu_run(emu, ch, jp).astype(np.float64)
    want = theta if fixture in FULL_RANK else theta @ (W64 @ P).T
    # the float32 rounding of jp, carried through W, is part of the tolerance
    tol = (K_FWD + 2 * U32) * (np.abs(jp.astype(np.float64)) + np.abs(o)) @ np.abs(W64).T + 1e-12
    assert np.all(np.abs(back - want) <= tol), np.abs(back - want).max()
    again = back @ P.T + o
    assert np.abs(again - jp).max() <= 1e-5 * max(1.0, np.abs(jp).max())
    # the adjoint identity
    ch.pt_offsets = np.zeros_like(ch.pt_offsets)
    x, g = _inputs(ch, B, 52)
    fx, ftg = _emu_run(emu, ch, x).astype(np.float64), _emu_run(emu, ch, g, True).astype(np.float64)
    lhs, rhs = (g * fx).sum(1), (ftg * x).sum(1)
    scale = (np.abs(g) @ np.abs(W64) * np.abs(x)).sum(1)
    assert np.all(np.abs(lhs - rhs) <= 1e-5 * scale + 1e-12)


def test_cpu_tensors_and_bad_shapes_are_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = mc.create_test_character(4)
    J = ch.num_joints
    with pytest.raises(ValueError, match="CUDA"):
        tsk.apply_inverse_parameter_transform(ch, torch.zeros(7 * J))
    with pytest.raises(ValueError, match="CUDA"):
        tsk.apply_inverse_parameter_transform(ch, torch.zeros(2, 7 * J, dtype=torch.float64))
    for bad in ((7 * J + 1,), (2, ch.num_params), (J, 7), (2, 3, 7 * J)):
        with pytest.raises(ValueError, match=r"must be \[.*\] or \[B, .*\], got"):
            tsk.apply_inverse_parameter_transform(ch, torch.zeros(bad))
    with pytest.raises(ValueError, match="tensor"):
        tsk.apply_inverse_parameter_transform(ch, np.zeros(7 * J, np.float32))


def test_planner_build_time(emu):
    """the host build of W (makeCharacter, this emulator's -O2 build of the planner), printed for humanoid72, bodyhands300 and a dense
    component at bodyhands300's size"""
    for ch in (mc.humanoid72()[0], mc.bodyhands300()[0], _stress()):
        keep = []
        args = emu_lib.character_args(ch, keep)
        best = math.inf
        for _ in range(2 if ch.name == "stress_dense" else 5):
            t = time.perf_counter()
            assert emu.emu_inverse_parameter_transform(*args, 0, 0, None, None, None) == 0, emu.emu_last_error().decode()
            best = min(best, time.perf_counter() - t)
        print(f"planner build {ch.name} (J = {ch.num_joints}, n = {ch.num_params}, nnz P = {ch.pt_inner.size}): {best * 1e3:.2f} ms")


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_device_operation_meets_the_float64_bounds(fixture):
    fwd, bwd = _measure(_dev_run, FIXTURES[fixture]())
    print(f"{fixture}: forward {fwd:.3g}, backward {bwd:.3g}")
    assert fwd <= K_FWD and bwd <= K_BWD


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", ["humanoid72", "bodyhands300"])
def test_end_to_end_recovers_the_model_parameters(fixture):
    """model_parameters_to_skeleton_state -> skeleton_state_to_joint_parameters -> flatten -> apply_inverse_parameter_transform recovers
    theta (|ry| <= 1.2, no angle wrap), and the gradient of a loss through all three matches float64 autograd"""
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES[fixture]()
    B, J = 8, ch.num_joints
    theta = np.random.default_rng(81).uniform(-0.4, 0.4, (B, ch.num_params)).astype(np.float32)
    th = torch.from_numpy(theta).cuda().requires_grad_(True)
    jp = tsk.skeleton_state_to_joint_parameters(ch, tsk.model_parameters_to_skeleton_state(ch, th)).flatten(-2)
    back = tsk.apply_inverse_parameter_transform(ch, jp)
    jp64 = _ref64(ch, "apply_parameter_transform", torch.from_numpy(theta.astype(np.float64)))
    assert np.abs(jp64.numpy().reshape(B, J, 7)[..., 3:6]).max() < math.pi / 2  # inside the principal range
    err = np.abs(back.detach().cpu().numpy() - theta).max()
    assert err <= 1e-4, err
    G = np.random.default_rng(82).normal(size=(B, ch.num_params))
    (back * torch.from_numpy(G.astype(np.float32)).cuda()).sum().backward()
    # float64 autograd through the same composition
    W64 = torch.from_numpy(_w64(ch))
    t64 = torch.from_numpy(theta.astype(np.float64)).requires_grad_(True)
    X = _fk64(ch, _ref64(ch, "apply_parameter_transform", t64).reshape(B, J, 7)).reshape(B, -1)
    j64 = _ref64(ch, "skeleton_state_to_joint_parameters", X)
    b64 = (j64 - torch.from_numpy(ch.pt_offsets.astype(np.float64))) @ W64.T
    (b64 * torch.from_numpy(G)).sum().backward()
    g, want = th.grad.cpu().numpy().astype(np.float64), t64.grad.numpy()
    ratio = (np.abs(g - want).max(1) / np.maximum(np.abs(want).max(1), 1.0)).max()
    assert ratio <= 1e-4, ratio


def _raw(dc, backward, x, out_numel):
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.empty(x.shape[0], out_numel, device="cuda")
    dc.joint_op_device(OP, backward, x.shape[0], x.data_ptr(), out.data_ptr(), stream=stream)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", ["humanoid72", "bodyhands300"])
def test_batch_independence_and_determinism(fixture):
    """one instance alone and inside batches of several sizes gives identical bits, and two runs give identical bits"""
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES[fixture]()
    R, n = 7 * ch.num_joints, ch.num_params
    B = 8192 + 37
    dc = tsk._device_character(ch, torch.device("cuda", 0))
    jp, g = (torch.from_numpy(a).cuda() for a in _inputs(ch, B, 91))
    f1, f2 = _raw(dc, False, jp, n), _raw(dc, False, jp, n)
    b1, b2 = _raw(dc, True, g, R), _raw(dc, True, g, R)
    assert torch.equal(f1, f2) and torch.equal(b1, b2)
    for lo, hi in ((0, 1), (5, 6), (B // 2, B // 2 + 300), (B - 38, B), (0, 2048)):
        assert torch.equal(_raw(dc, False, jp[lo:hi].contiguous(), n), f1[lo:hi]), (lo, hi)
        assert torch.equal(_raw(dc, True, g[lo:hi].contiguous(), R), b1[lo:hi]), (lo, hi)


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_streams_and_errors():
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES["coupled"]()
    n, R = ch.num_params, 7 * ch.num_joints
    dev = torch.device("cuda", 0)
    jp = torch.from_numpy(_inputs(ch, 3, 101)[0]).to(dev)
    out = tsk.apply_inverse_parameter_transform(ch, jp.double())
    assert out.shape == (3, n) and out.dtype == torch.float64
    one = tsk.apply_inverse_parameter_transform(ch, jp[1])
    assert one.shape == (n,) and torch.equal(one, out[1].float())
    x = jp.double().requires_grad_(True)
    tsk.apply_inverse_parameter_transform(ch, x).sum().backward()
    assert x.grad.shape == (3, R) and x.grad.dtype == torch.float64
    e = torch.zeros(0, R, device=dev, requires_grad=True)
    out0 = tsk.apply_inverse_parameter_transform(ch, e)
    assert out0.shape == (0, n)
    out0.sum().backward()
    assert e.grad.shape == (0, R)

    def run(t):
        t = t.clone().requires_grad_(True)
        o = tsk.apply_inverse_parameter_transform(ch, t)
        o.backward(torch.ones_like(o))
        return o.detach(), t.grad

    ref = run(jp)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        got = run(jp)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    dc = ms.DeviceCharacter(ch, 0)
    assert torch.equal(tsk.apply_inverse_parameter_transform(dc, jp), ref[0])
    dc.device = 1
    with pytest.raises(ValueError, match="device character"):
        tsk.apply_inverse_parameter_transform(dc, jp)


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments():
    ch = mc.create_test_character(4)
    dc = ms.DeviceCharacter(ch, 0)
    n, J = ch.num_params, ch.num_joints
    th = torch.zeros(2, n, device="cuda")
    jp = torch.zeros(2, 7 * J, device="cuda")
    host = np.zeros((2, 7 * J), np.float32)
    for backward, x, y in ((False, jp, th), (True, th, jp)):
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.joint_op_device(OP, backward, 2, 0, y.data_ptr())
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.joint_op_device(OP, backward, 2, x.data_ptr(), 0)
        with pytest.raises(ms.MomentumB200Error, match="negative"):
            dc.joint_op_device(OP, backward, -1, x.data_ptr(), y.data_ptr())
        with pytest.raises(ms.MomentumB200Error, match="device memory"):
            dc.joint_op_device(OP, backward, 2, x.data_ptr(), host.ctypes.data)
        with pytest.raises(ms.MomentumB200Error, match="device memory"):
            dc.joint_op_device(OP, backward, 2, host.ctypes.data, y.data_ptr())
        dc.joint_op_device(OP, backward, 0, 0, 0)  # batch 0: nothing to do
