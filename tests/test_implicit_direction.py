"""The direction of solve_ik's implicit-function backward on the device: v = (2 J_E^T J_E)^+ g, J v, the residual and the gradient RMS
(``mb2_solver_function_implicit_direction_device``, the reference's hessianInverseTimes).

The reference is float64 ``numpy.linalg.svd`` of the backend's own float32 J_E (the tests/f64ref.py approach): FK and Jacobian rounding
drop out and only the solve's error remains. A result passes when ||v - v64||_inf <= K_BOUND ||v64||_inf per instance, and the same for
J v. Every fixture keeps its s^2 at least 1e-3 tau away from the truncation threshold tau = 1e-5, so that none sits on the edge by
accident; one fixture sits there on purpose. The CPU emulator (tests/emu/emu_implicit_direction.cu) runs the kernel's building blocks on
the oracle's float32 Jacobian, the GPU tests run the kernel through the C-ABI.
"""
import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import add_test_limits, bodyhands_problem, chain_problem, humanoid_problem
from tests import emu_lib

TAU = 1e-5
MAX_SWEEPS = 32  # kJacobiMaxSweeps (ik_jacobi.cuh)

# worst measured max(||v - v64||_inf / ||v64||_inf, same for J v) over the fixtures below: 4.7e-8 on the emulator (humanoid72, cfg2)
# and 5.5e-8 on an H100 80GB HBM3 at a 700 W power limit (chain), the float32 rounding of the outputs; pinned about four times above.
# The likely errors of the self-check miss it by more than 100x.
K_BOUND = 2e-7


# ---- fixtures -----------------------------------------------------------------------------------------------------------------------
def _fixture(name, B, seed=5):
    """(character, error functions, enabled [n], theta [B, n] float32, g [B, n] float32, unpadded rows)"""
    rng = np.random.default_rng(seed)
    if name == "chain":
        ch, efs, _, _ = chain_problem(J=6, B=B, seed=seed)
        n = ch.num_params
        theta = rng.uniform(-0.4, 0.4, (B, n))
        enabled = np.ones(n, bool)
    elif name == "bodyhands300_cfg4":
        ch, efs, _, star = bodyhands_problem(B)
        n = ch.num_params
        theta = star + 0.05 * rng.normal(size=star.shape)
        enabled = np.ones(n, bool)
    else:
        ch, efs, _, star = humanoid_problem(B, orientation=name != "humanoid72_cfg2")
        n = ch.num_params
        theta = star + 0.05 * rng.normal(size=star.shape)
        enabled = np.ones(n, bool)
        if name == "humanoid72_all":  # Position + Orientation + Limit + Motion: more rows than parameters (k = n_E = 220)
            add_test_limits(ch, rng, ellipsoid=False)
            efs = efs + [mc.LimitErrorFunction(weight=1.0),
                         mc.ModelParametersErrorFunction(rng.uniform(0.3, 1.0, n), star + 0.1 * rng.normal(size=star.shape), weight=1.0)]
        if name == "humanoid72_subset":  # about half of the parameters: fewer enabled columns than rows (k = n_E)
            enabled[7 + rng.choice(n - 7, (n - 7) // 2, replace=False)] = False
    g = rng.normal(size=(B, n))
    rows = sum(mc.jacobian_size(ch, ef) for ef in efs)
    return ch, efs, enabled, theta.astype(np.float32), g.astype(np.float32), rows


FIXTURES = ["chain", "humanoid72_cfg2", "humanoid72_cfg3", "humanoid72_all", "humanoid72_subset", "bodyhands300_cfg4"]
K_OF = {"humanoid72_cfg2": 72, "humanoid72_cfg3": 126, "humanoid72_all": 220, "bodyhands300_cfg4": 424}


def _ref64(JE, g):
    """v64 [n_E], J v64 [rows], s^2, from float64 SVD (fully_differentiable_body_ik.cpp:78-109)"""
    J = np.asarray(JE, np.float64)
    _, S, Vt = np.linalg.svd(J, full_matrices=False)
    s2 = S * S
    tmp = Vt @ np.asarray(g, np.float64)
    tmp = np.where(s2 < TAU, 0.0, tmp / np.maximum(s2, 1e-300))
    v = 0.5 * Vt.T @ tmp
    return v, J @ v, s2


def _ratio(x, x64):
    return float(np.abs(np.asarray(x, np.float64) - x64).max() / max(np.abs(x64).max(), 1e-300))


def _assert_off_the_edge(s2):
    assert np.abs(s2 - TAU).min() >= 1e-3 * TAU, np.abs(s2 - TAU).min() / TAU


def _oracle_jacobian(ch, efs, enabled, theta_b, b, rows):
    from oracle.binding import OracleFunction

    orc = OracleFunction(ch, efs, "float32", instance=b)
    orc.set_enabled_parameters(enabled)
    _, J, r, _ = orc.get_jacobian(theta_b.astype(np.float64))
    return np.asarray(J[:rows], np.float32), np.asarray(r[:rows], np.float32)


# ---- CPU: the emulator ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _emu(L, JE, r, g):
    """(v [n_E], J v [rows], gradient RMS, sweeps) of the emulated kernel on the rows x n_E float32 matrix JE"""
    rows, nE = JE.shape
    jt = np.ascontiguousarray(np.asarray(JE, np.float32).T)
    r = np.ascontiguousarray(r, np.float32)
    g = np.ascontiguousarray(g, np.float32)
    v, jv, rms, sw = np.zeros(nE), np.zeros(rows), np.zeros(1), np.zeros(1, np.int32)
    assert L.emu_implicit_direction(rows, nE, jt.ctypes.data, r.ctypes.data, g.ctypes.data, v.ctypes.data, jv.ctypes.data, rms.ctypes.data,
                                    sw.ctypes.data) == 0
    return v, jv, float(rms[0]), int(sw[0])


@pytest.mark.parametrize("name", FIXTURES)
def test_emulated_direction_meets_the_float64_bound(emu, name):
    B = 2
    ch, efs, enabled, theta, g, rows = _fixture(name, B)
    E = np.nonzero(enabled)[0]
    for b in range(B):
        J, r = _oracle_jacobian(ch, efs, enabled, theta[b], b, rows)
        JE = J[:, E]
        if name in K_OF:
            assert min(JE.shape) == K_OF[name]
        v, jv, rms, sweeps = _emu(emu, JE, r, g[b, E])
        v64, jv64, s2 = _ref64(JE, g[b, E])
        _assert_off_the_edge(s2)
        worst = max(_ratio(v, v64), _ratio(jv, jv64))
        print(f"emu {name} b={b} rows={JE.shape[0]} n_E={JE.shape[1]}: ratio {worst:.3e}, {sweeps} sweeps")
        assert worst <= K_BOUND, (name, b, worst)
        assert sweeps < MAX_SWEEPS
        rms64 = np.sqrt(np.mean((2.0 * JE.astype(np.float64).T @ r.astype(np.float64)) ** 2))
        assert abs(rms - rms64) <= 1e-6 * rms64


@pytest.mark.parametrize("case", ["zero", "k1_rows", "k1_params", "clustered", "repeated", "odd", "zero_rows"])
def test_emulated_edge_cases_converge_and_meet_the_bound(emu, case):
    rng = np.random.default_rng(11)
    if case == "zero":
        JE = np.zeros((6, 9), np.float32)
    elif case == "k1_rows":
        JE = rng.normal(size=(1, 7)).astype(np.float32)
    elif case == "k1_params":
        JE = rng.normal(size=(8, 1)).astype(np.float32)
    elif case in ("clustered", "repeated"):  # U diag(s) V^T with clustered (1 + 1e-9 i) or exactly repeated singular values
        U, _ = np.linalg.qr(rng.normal(size=(24, 24)))
        V, _ = np.linalg.qr(rng.normal(size=(31, 24)))
        s = np.where(np.arange(24) < 12, 1.0, 0.3) * (1.0 + (1e-9 * np.arange(24) if case == "clustered" else 0.0))
        JE = (U * s) @ V.T
    elif case == "odd":
        JE = rng.normal(size=(37, 45))
    else:  # zero rows and an all-zero 2 x 2 block, as zero-weight constraints give
        JE = rng.normal(size=(20, 33))
        JE[[3, 4, 11]] = 0.0
    JE = np.asarray(JE, np.float32)
    g, r = rng.normal(size=JE.shape[1]), rng.normal(size=JE.shape[0])
    v, jv, _, sweeps = _emu(emu, JE, r, g)
    assert sweeps < MAX_SWEEPS, sweeps
    v64, jv64, s2 = _ref64(JE, g.astype(np.float32))
    if case == "zero":
        assert sweeps == 0 and not v.any() and not jv.any()
        return
    _assert_off_the_edge(s2)
    assert max(_ratio(v, v64), _ratio(jv, jv64)) <= K_BOUND, case


def _motion_edge(n=40, efw=0.8):
    """A Motion-only problem on the test chain whose weights put s_i^2 = 0.1 efw w_i^2 at tau (1 +- 1.1e-3) (and a few far from it)"""
    ch = mc.create_test_character(6)
    n = ch.num_params
    rng = np.random.default_rng(3)
    side = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    w = np.sqrt(TAU * (1.0 + 1.1e-3 * side) / (0.1 * efw))
    w[::7] = 1.0
    tgt = rng.normal(size=(1, n))
    return ch, mc.ModelParametersErrorFunction(w, tgt, weight=efw), rng.normal(size=n).astype(np.float32)


def _check_truncation_edge(JE, g, v):
    """J_E is diagonal (one row per parameter): a kept component is g_i / (2 s_i^2), a dropped one exactly 0."""
    s2 = np.diag(JE.astype(np.float64)) ** 2
    assert np.abs(s2 - TAU).min() >= 0.9e-3 * TAU  # the stored float32 entries moved the products by ~1e-7 at most
    keep = s2 >= TAU
    assert keep.any() and (~keep).any()
    assert np.array_equal(v[~keep], np.zeros((~keep).sum()))
    want = g[keep].astype(np.float64) / (2.0 * s2[keep])
    assert np.abs(v[keep] - want).max() <= 1e-6 * np.abs(want).max()


def test_emulated_truncation_edge(emu):
    ch, ef, g = _motion_edge()
    J, r = _oracle_jacobian(ch, [ef], np.ones(ch.num_params, bool), np.zeros(ch.num_params, np.float32), 0, ch.num_params)
    assert np.count_nonzero(J - np.diag(np.diag(J))) == 0
    v, _, _, _ = _emu(emu, J, r, g)
    _check_truncation_edge(J, g, v)


def test_the_bound_rejects_the_likely_errors():
    """float64 / float32 stand-ins of what a Jacobi solve most easily gets wrong, on the oracle's float32 J_E of cfg3 (rows side, nine
    rows of rank three per Orientation constraint) and of the parameter-side fixture: each misses the bound by far."""
    for name in ("humanoid72_cfg3", "humanoid72_all"):
        ch, efs, enabled, theta, g, rows = _fixture(name, 1)
        E = np.nonzero(enabled)[0]
        J, _ = _oracle_jacobian(ch, efs, enabled, theta[0], 0, rows)
        JE, gE = J[:, E].astype(np.float64), g[0, E].astype(np.float64)
        v64, jv64, s2 = _ref64(JE, gE)
        rows_side = JE.shape[0] <= JE.shape[1]

        def solve(K, y, power, tau=TAU, half=0.5):
            lam, Q = np.linalg.eigh(K)
            z = np.where(lam >= tau, (Q.T @ y) / np.where(lam >= tau, lam, 1.0) ** power, 0.0) if tau > 0 else (Q.T @ y) / lam ** power
            z = Q @ z
            v = half * (JE.T @ z if rows_side else z)
            return v, JE @ v

        K = JE @ JE.T if rows_side else JE.T @ JE
        y = JE @ gE if rows_side else gE
        p = 2 if rows_side else 1
        good = solve(K, y, p)
        assert max(_ratio(good[0], v64), _ratio(good[1], jv64)) <= K_BOUND
        K32, y32 = K.astype(np.float32), y.astype(np.float32)
        lam32, Q32 = np.linalg.eigh(K32)
        z32 = np.where(lam32 >= TAU, (Q32.T @ y32) / np.where(lam32 >= TAU, lam32, 1.0) ** p, 0.0)
        v32 = 0.5 * (JE.T @ (Q32 @ z32) if rows_side else Q32 @ z32)
        wrong = {"no 1/2": solve(K, y, p, half=1.0)}
        if rows_side:  # (on the parameter side the float32 Gram of this fixture is well enough conditioned to miss the bound by 5x only)
            wrong["float32 eigen-solve"] = (v32, JE @ v32)
            wrong["Lambda^-1 on the rows side"] = solve(K, y, 1)
            wrong["no truncation"] = solve(K, y, p, tau=0.0)  # the rank-deficient Orientation blocks: exact-zero eigenvalues
            assert (s2 < 1e-12).any()
        for what, (v, jv) in wrong.items():
            worst = max(_ratio(v, v64), _ratio(jv, jv64))
            assert not worst <= 100 * K_BOUND, (name, what, worst)


# ---- GPU: the kernel through the C-ABI ---------------------------------------------------------------------------------------------------
def _dev_function(ch, efs, enabled, B):
    fn = ms.SkeletonSolverFunction(ch, B, efs, device=0)
    fn.upload_targets()
    fn.set_enabled_parameters(enabled)
    return fn


def _dev_direction(fn, theta, g, outputs=(True, True, True), stream=None):
    """(v [B, n], J v [B, rows8], r [B, rows8], rms [B]) as torch tensors; a skipped output stays NaN"""
    B, n = theta.shape
    st = stream or torch.cuda.current_stream()
    with torch.cuda.stream(st):
        th, gg = torch.as_tensor(theta).cuda(), torch.as_tensor(g).cuda()
        v = torch.full((B, n), float("nan"), device="cuda")
        rest = [torch.full((B, fn.jacobian_rows), float("nan"), device="cuda"), torch.full((B, fn.jacobian_rows), float("nan"), device="cuda"),
                torch.full((B,), float("nan"), device="cuda")]
        ptrs = [o.data_ptr() if want else 0 for o, want in zip(rest, outputs)]
        fn.implicit_direction_device(th.data_ptr(), gg.data_ptr(), v.data_ptr(), *ptrs, stream=st.cuda_stream)
    st.synchronize()
    return [v] + rest


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_kernel_direction_meets_the_float64_bound(name):
    B = 3 if name == "bodyhands300_cfg4" else 5
    ch, efs, enabled, theta, g, rows = _fixture(name, B)
    fn = _dev_function(ch, efs, enabled, B)
    v, jv, r, rms = [t.cpu().numpy() for t in _dev_direction(fn, theta, g)]
    _, J, res, _ = fn.get_jacobian(theta)  # the backend's own float32 Jacobian and residual
    E = np.nonzero(enabled)[0]
    for b in range(B):
        JE = J[b, :rows][:, E]
        if name in K_OF:
            assert min(JE.shape) == K_OF[name]
        v64, jv64, s2 = _ref64(JE, g[b, E])
        _assert_off_the_edge(s2)
        worst = max(_ratio(v[b, E], v64), _ratio(jv[b, :rows], jv64))
        print(f"kernel {name} b={b} rows={JE.shape[0]} n_E={JE.shape[1]}: ratio {worst:.3e}")
        assert worst <= K_BOUND, (name, b, worst)
        assert not v[b, ~enabled].any()
        assert np.array_equal(r[b], res[b]) and not jv[b, rows:].any()
        rms64 = np.sqrt(np.mean((2.0 * JE.astype(np.float64).T @ res[b, :rows].astype(np.float64)) ** 2))
        assert abs(rms[b] - rms64) <= 1e-6 * rms64


@pytest.mark.gpu
def test_kernel_truncation_edge():
    ch, ef, g = _motion_edge()
    n = ch.num_params
    fn = _dev_function(ch, [ef], np.ones(n, bool), 1)
    theta = np.zeros((1, n), np.float32)
    v = _dev_direction(fn, theta, g[None])[0].cpu().numpy()[0]
    _, J, _, _ = fn.get_jacobian(theta)
    _check_truncation_edge(J[0, :n], g, v)


@pytest.mark.gpu
def test_kernel_is_deterministic_and_independent_of_the_batch():
    """cfg3 over at least three waves plus a remainder for any launch shape (at most 8 CTAs of 256 threads per SM)"""
    B = 3 * torch.cuda.get_device_properties(0).multi_processor_count * 8 + 37
    ch, efs, enabled, theta, g, rows = _fixture("humanoid72_cfg3", B, seed=7)
    fn = _dev_function(ch, efs, enabled, B)
    a, b = _dev_direction(fn, theta, g), _dev_direction(fn, theta, g)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for i in (0, 1, B // 3, B - 38, B - 1):  # B - 37 .. B - 1 is the remainder
        one_efs = [type(e)(e.parents, e.offsets, e.weights, np.asarray(e.targets)[i:i + 1], weight=e.weight) for e in efs]
        one = _dev_direction(_dev_function(ch, one_efs, enabled, 1), theta[i:i + 1], g[i:i + 1])
        assert all(torch.equal(x, y[i:i + 1]) for x, y in zip(one, a)), i


@pytest.mark.gpu
def test_c_abi_errors_null_outputs_and_a_side_stream():
    ch, efs, enabled, theta, g, rows = _fixture("chain", 2)
    fn = _dev_function(ch, efs, enabled, 2)
    th, gg = torch.from_numpy(theta).cuda(), torch.from_numpy(g).cuda()
    v = torch.zeros_like(th)
    with pytest.raises(ms.MomentumB200Error, match="null"):
        fn.implicit_direction_device(0, gg.data_ptr(), v.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null"):
        fn.implicit_direction_device(th.data_ptr(), 0, v.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null direction"):
        fn.implicit_direction_device(th.data_ptr(), gg.data_ptr(), 0)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        fn.implicit_direction_device(theta.ctypes.data, gg.data_ptr(), v.data_ptr())
    host = np.zeros(2, np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        fn.implicit_direction_device(th.data_ptr(), gg.data_ptr(), v.data_ptr(), 0, 0, host.ctypes.data)
    full = _dev_direction(fn, theta, g)
    for mask in ((True, False, False), (False, True, False), (False, False, True), (False, False, False)):
        part = _dev_direction(fn, theta, g, mask)
        assert torch.equal(part[0], full[0])
        for want, x, y in zip(mask, part[1:], full[1:]):
            assert torch.equal(x, y) if want else bool(torch.isnan(x).all())
    side = torch.cuda.Stream()
    on_side = _dev_direction(fn, theta, g, stream=side)
    assert all(torch.equal(x, y) for x, y in zip(on_side, full))
    # an empty enabled set gives v = 0
    fn.set_enabled_parameters(np.zeros(ch.num_params, bool))
    z = _dev_direction(fn, theta, g)
    assert not z[0].any() and not z[1].any() and not z[3].any()
    # a handle's batch is positive: a zero batch never reaches the entry
    with pytest.raises(ms.MomentumB200Error):
        ms.SkeletonSolverFunction(ch, 0, efs, device=0)


# ---- GPU: solve_ik end to end against the float64 SVD path ------------------------------------------------------------------------------
def _svd_direction(fn, active, theta_ptr, g_ptr, v_ptr, jv_ptr, r_ptr, rms_ptr, stream):
    """The backward's former algorithm, restated: the device Jacobian, float64 torch.linalg.svd of its enabled columns, the RMS in
    float64; written to the same buffers the device entry fills."""
    from momentum_b200 import torch_ik as ti

    dev = torch.device("cuda", 0)
    B, n, rows8 = fn.batch, fn.num_parameters, fn.jacobian_rows
    theta = ti._device_view(theta_ptr, (B, n), dev)
    ptr, ld = fn.get_jacobian_device(theta_ptr, stream)
    torch.cuda.synchronize()
    J_all = ti._device_view(ptr, (B, n + 1, ld), dev).clone()
    J = J_all[:, :n, :rows8].transpose(1, 2).double()
    r = J_all[:, n, :rows8].double()
    act = torch.as_tensor(np.nonzero(active)[0], device=dev)
    Ja = J[:, :, act]
    g = ti._device_view(g_ptr, (B, n), dev).double()[:, act]
    rms = torch.sqrt(((2.0 * torch.einsum("brk,br->bk", Ja, r)) ** 2).mean(dim=1))
    _, S, Vh = torch.linalg.svd(Ja, full_matrices=False)
    s2 = S * S
    tmp = torch.einsum("bkn,bn->bk", Vh, g)
    tmp = torch.where(s2 < TAU, torch.zeros_like(tmp), tmp / s2.clamp_min(1e-30))
    v = torch.zeros(B, n, dtype=torch.float64, device=dev)
    v[:, act] = 0.5 * torch.einsum("bkn,bk->bn", Vh, tmp)
    ti._device_view(v_ptr, (B, n), dev).copy_(v.float())
    ti._device_view(jv_ptr, (B, rows8), dev).copy_(torch.einsum("brn,bn->br", J, v).float())
    ti._device_view(r_ptr, (B, rows8), dev).copy_(r.float())
    ti._device_view(rms_ptr, (B,), dev).copy_(rms.float())
    torch.cuda.synchronize()
    del theta


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [False, True])
def test_solve_ik_gradients_match_the_float64_svd_path(monkeypatch, shared):
    from momentum_b200 import torch_ik as ti

    dev = torch.device("cuda", 0)
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 17  # k = 220: one CTA per SM, so two waves and more
    ch, sets = mc.humanoid72()
    rng = np.random.default_rng(21)
    add_test_limits(ch, rng, ellipsoid=False)
    n = ch.num_params
    star = np.zeros((B, n))
    star[:, 7:] = rng.uniform(-0.4, 0.4, (B, n - 7))
    pp, op = np.array(sets["position_joints"], np.int32), np.array(sets["orientation_joints"], np.int32)
    po = rng.uniform(-3, 3, (len(pp), 3))
    oo = rng.normal(size=(len(op), 4)); oo /= np.linalg.norm(oo, axis=-1, keepdims=True)
    pt = mc.world_points(ch, star, pp, po) + 0.02 * rng.normal(size=(B, len(pp), 3))
    ot = mc.world_rotations(ch, star, op, oo)
    mt = star + 0.05 * rng.normal(size=star.shape)
    mw = rng.uniform(0.3, 1.0, n)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(dev).requires_grad_(True)
    leaves = dict(efw=t(np.ones((B, 4))), pt=t(pt), pw=t(rng.uniform(0.5, 1.5, (B, len(pp)))),
                  po=t(po if shared else np.broadcast_to(po, (B,) + po.shape)), ot=t(ot), ow=t(rng.uniform(0.5, 1.5, (B, len(op)))),
                  oo=t(oo if shared else np.broadcast_to(oo, (B,) + oo.shape)), mt=t(mt), mw=t(mw if shared else np.broadcast_to(mw, (B, n))))
    kinds = [ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation, ti.ErrorFunctionType.Limit, ti.ErrorFunctionType.Motion]
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=20, max_iter=20, threshold=1.0)
    active = np.ones(n, bool)
    theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), kinds, leaves["efw"], opts, position_cons_parents=pp, position_cons_offsets=leaves["po"],
                        position_cons_weights=leaves["pw"], position_cons_targets=leaves["pt"], orientation_cons_parents=op,
                        orientation_cons_offsets=leaves["oo"], orientation_cons_weights=leaves["ow"], orientation_cons_targets=leaves["ot"],
                        motion_targets=leaves["mt"], motion_weights=leaves["mw"])
    loss = (theta.double() * torch.from_numpy(rng.normal(size=(B, n))).to(dev)).sum()
    loss.backward(retain_graph=True)
    got = {k: x.grad.clone() for k, x in leaves.items()}
    for x in leaves.values():
        x.grad = None
    fn = theta.grad_fn.cfg["fn"]  # the handle this solve used
    monkeypatch.setattr(fn, "implicit_direction_device", lambda *a, **kw: _svd_direction(fn, active, *a, **kw), raising=False)
    loss.backward()
    assert any(got[k].abs().max() > 0 for k in got)
    for k, x in leaves.items():
        ref = x.grad
        err = (got[k] - ref).abs().max().item()
        assert err <= 1e-4 * max(ref.abs().max().item(), 1.0), (k, err, ref.abs().max().item())
