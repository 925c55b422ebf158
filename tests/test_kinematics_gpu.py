"""Forward kinematics and linear point Jacobians on the H100 (DESIGN.md section 7.13): the KIN instances of the world-frame kernel as nvcc
builds them, against the host build of the same source and the C oracle, on ragged and chunked batches, with installed parameters,
through torch.autograd (backward, forward_ad, torch.func.jvp, a loss after a rollout of steps), a batched inverse kinematics at 4096
environments, pytinydiffsim.point_jacobian, and every argument check of the C-ABI.  The CPU twins are in tests/test_kinematics_on_host.py."""
import ctypes
import os

import numpy as np
import pytest

import tds_b200
from tds_b200.model import fixture_path, load_model, param_values
from test_mass_matrix_on_host import GOLDEN, ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, rel
from test_params_on_host import all_ids, perturbed
from test_kinematics_on_host import LAIKAGO_TOES, laikago_ik, laikago_targets, oracle_outputs, tables

pytestmark = pytest.mark.gpu

ALL = ORACLE_FIXTURES + OTHER_FIXTURES


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return q


def _xf(R, p):
    n, nl = p.shape[:2]
    return np.concatenate([R.reshape(n, nl, 9), p], axis=2)


@pytest.mark.parametrize("name", ALL)
def test_device_against_the_host_build_and_the_oracle(name):
    import emu_kin
    model, q = fixture(name)
    sim = _sim(model, q.shape[0])
    for lk, lc in tables(model):
        R, p, x, J = sim.kinematics_host(q, lk, lc)
        xh, xxh, Jh = emu_kin.kinematics(model, q, lk, lc)
        assert rel(_xf(R, p), xh) <= 1e-12 and rel(x, xxh) <= 1e-12 and rel(J, Jh) <= 1e-12
        if name in ORACLE_FIXTURES:
            for e in range(2):
                xo, xxo, Jo = oracle_outputs(model, f32(q[e]), lk, lc)
                for a, b in ((_xf(R, p)[e], xo), (x[e], xxo), (J[e], Jo)):
                    assert np.all(np.abs(a - b) <= 1e-10 * np.maximum(1.0, np.abs(b))), name


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 100, 3)
    lk, lc = tables(model)[0]
    full = _sim(model, 100).kinematics_host(q, lk, lc)
    for n in (1, 31, 33, 100):
        part = _sim(model, n).kinematics_host(q[-n:], lk, lc)
        for a, b in zip(part, full):
            assert np.array_equal(a, b[-n:]), n


def test_device_layout_and_host_layout_agree():
    import torch
    model, q = fixture("laikago")
    n = q.shape[0]
    sim = _sim(model, n)
    lk, lc = tables(model)[0]
    K, ns = len(lk), sim.n_stride
    R, p, x, J = sim.kinematics_host(q, lk, lc)
    qs = torch.zeros((sim.n_q, ns), dtype=torch.float32, device="cuda")
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    z = dict(dtype=torch.float64, device="cuda")
    xf_d, x_d, J_d = torch.zeros((sim.n_links * 12, ns), **z), torch.zeros((3 * K, ns), **z), torch.zeros((3 * K * sim.n_qd, ns), **z)
    sim.kinematics_device(qs, lk, lc, xf_d, x_d, J_d)
    torch.cuda.synchronize()
    assert np.array_equal(xf_d[:, :n].t().cpu().numpy().reshape(n, -1, 12), _xf(R, p))
    assert np.array_equal(x_d[:, :n].t().cpu().numpy().reshape(n, K, 3), x)
    assert np.array_equal(J_d[:, :n].t().cpu().numpy().reshape(n, K, 3, sim.n_qd), J)


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_kin
    model, q = fixture(name)
    sim = _sim(model, q.shape[0])
    lk, lc = tables(model)[0]
    rng = np.random.default_rng(4)
    V = rng.normal(size=(q.shape[0], sim.n_q, 3))
    d = sim.kinematics_jvp_host(q, lk, lc, V)
    dh = emu_kin.kinematics_jvp(model, q, lk, lc, V)
    for a, b in zip(d, dh):
        assert rel(a.reshape(b.shape), b) <= 1e-12
    G = [rng.normal(size=(q.shape[0], r)) for r in emu_kin.rows(model, len(lk))]
    g = sim.kinematics_vjp_host(q, lk, lc, *G)
    assert rel(g, emu_kin.kinematics_vjp(model, q, lk, lc, *G)) <= 1e-12
    # a NULL cotangent is zero
    g0 = sim.kinematics_vjp_host(q, lk, lc, None, G[1], None)
    assert rel(g0, emu_kin.kinematics_vjp(model, q, lk, lc, 0 * G[0], G[1], 0 * G[2])) <= 1e-12


def test_humanoid_jvp_in_several_chunks_equals_one_chunk():
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    warps = probe.jacobian_chunk() // 3 + 1
    n = 32 * warps
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    m = sim.n_q
    assert 1 <= chunk < m, (chunk, m)
    q = _q(model, n, 5)
    lk, lc = tables(model)[0]
    V = np.random.default_rng(6).normal(size=(n, sim.n_q, m))
    d = sim.kinematics_jvp_host(q, lk, lc, V)
    for j0 in range(0, m, chunk):
        part = sim.kinematics_jvp_host(q, lk, lc, V[:, :, j0:j0 + chunk])
        for a, b in zip(part, d):
            assert np.array_equal(a, b[..., j0:j0 + chunk]), j0


def test_parameter_sets_and_step_outputs_are_untouched():
    """Outputs are bit-identical with and without an installed set; the step's outputs are bit-identical before and after kinematics
    calls, while a set is installed and after it is cleared."""
    model, q = fixture("laikago")
    n = q.shape[0]
    sim = _sim(model, n)
    qd = np.load(os.path.join(GOLDEN, "laikago.npz"))["qd_in"][:n]
    lk, lc = tables(model)[0]
    before = sim.step_host(2, q, qd)
    K0 = sim.kinematics_host(q, lk, lc)
    V = np.random.default_rng(1).normal(size=(n, sim.n_q, 2))
    D0 = sim.kinematics_jvp_host(q, lk, lc, V)
    assert all(np.array_equal(a["q"], before["q"]) for a in [sim.step_host(2, q, qd)])
    ids = all_ids(model)
    sim.set_physical_params(ids, perturbed(model, ids, n, 14, 0.5, 0.0))
    with_set = sim.step_host(2, q, qd)
    for a, b in zip(sim.kinematics_host(q, lk, lc), K0):
        assert np.array_equal(a, b)
    for a, b in zip(sim.kinematics_jvp_host(q, lk, lc, V), D0):
        assert np.array_equal(a, b)
    again = sim.step_host(2, q, qd)
    assert np.array_equal(again["q"], with_set["q"]) and np.array_equal(again["qd"], with_set["qd"])
    sim.set_physical_params(None)
    for a, b in zip(sim.kinematics_host(q, lk, lc), K0):
        assert np.array_equal(a, b)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


def test_autograd_backward_and_forward_mode():
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture("humanoid")
    n = q.shape[0]
    sim = _sim(model, n)
    lk, lc = tables(model)[0]
    K = len(lk)
    qt = torch.tensor(q, dtype=torch.float32, device="cuda")
    rng = np.random.default_rng(16)
    GR, Gp, Gx, GJ = (rng.normal(size=s) for s in ((n, sim.n_links, 3, 3), (n, sim.n_links, 3), (n, K, 3), (n, K, 3, sim.n_qd)))
    qr = qt.clone().requires_grad_(True)
    R, p, x, J = tds_b200.autograd.forward_kinematics(sim, qr, lk, lc)
    ref = sim.kinematics_host(f32(q), lk, lc)
    for a, b in zip((R, p, x, J), ref):
        assert a.dtype == torch.float64 and np.array_equal(a.detach().cpu().numpy(), b)
    loss = sum((a * torch.tensor(g, device="cuda")).sum() for a, g in zip((R, p, x, J), (GR, Gp, Gx, GJ)))
    loss.backward()
    g_q = sim.kinematics_vjp_host(f32(q), lk, lc, np.concatenate([GR.reshape(n, -1, 9), Gp], axis=2), Gx, GJ)
    assert qr.grad.dtype == torch.float32
    assert rel(qr.grad.cpu().numpy().astype(np.float64), g_q.astype(np.float32).astype(np.float64)) <= 1e-12
    vq = rng.normal(size=(n, sim.n_q))
    dxf, dx, dJ = sim.kinematics_jvp_host(f32(q), lk, lc, vq.astype(np.float32))
    want = (dxf[..., :9].reshape(n, -1, 3, 3), dxf[..., 9:], dx, dJ)
    tq = torch.tensor(vq, dtype=torch.float32, device="cuda")
    with fwAD.dual_level():
        outs = tds_b200.autograd.forward_kinematics(sim, fwAD.make_dual(qt, tq), lk, lc)
        tans = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in outs]
    for a, b in zip(tans, want):
        assert rel(a, b) <= 1e-12
    _, ft = torch.func.jvp(lambda a: tds_b200.autograd.forward_kinematics(sim, a, lk, lc), (qt,), (tq,))
    for a, b in zip(ft, want):
        assert rel(a.cpu().numpy(), b) <= 1e-12


@pytest.mark.parametrize("name", ["cartpole", "pendulum5", "laikago_pd"])
def test_loss_on_points_after_a_rollout_equals_the_chain_of_vjps(name):
    import torch
    from test_vjp_gpu import _case
    n, steps = 16, 5
    sim, mode, q, qd, t, pd = _case(name, n)
    if t is None:
        t = np.zeros((n, sim.n_act if pd else sim.n_tau))
    md = 2 if mode == 0 else mode
    lk, lc = {"cartpole": ([1], [[0.0, 0.0, 0.5]]), "pendulum5": ([4], [[0.0, 0.0, -0.5]]),
              "laikago_pd": (LAIKAGO_TOES, np.zeros((4, 3)))}[name]
    dev = "cuda:0"
    q0 = torch.tensor(q, dtype=torch.float32, device=dev, requires_grad=True)
    qd0 = torch.tensor(qd, dtype=torch.float32, device=dev, requires_grad=True)
    tau = torch.tensor(t, dtype=torch.float32, device=dev, requires_grad=True)
    W = np.random.default_rng(8).normal(size=(n, len(lk), 3))
    states = []
    xq, xd = q0, qd0
    for _ in range(steps):
        states.append((xq.detach().cpu().numpy().astype(np.float64), xd.detach().cpu().numpy().astype(np.float64)))
        xq, xd = tds_b200.autograd.step(sim, xq, xd, tau, mode=md, use_pd=pd)
    qT = xq.detach().cpu().numpy().astype(np.float64)
    _, _, x, _ = tds_b200.autograd.forward_kinematics(sim, xq, lk, lc)
    (x * torch.tensor(W, device=dev)).sum().backward()
    # the same chain through the C-ABI: the kinematics VJP, then the step VJPs, cotangents rounded to float32 between calls
    g_q = sim.kinematics_vjp_host(qT, lk, lc, None, W, None).astype(np.float32).astype(np.float64)
    g = np.concatenate([g_q, np.zeros((n, sim.n_qd))], axis=1)
    g_tau = np.zeros(t.shape, dtype=np.float32)
    nx = sim.n_q + sim.n_qd
    for k in reversed(range(steps)):
        gin = sim.step_vjp_host(md, states[k][0], states[k][1], t, g, use_pd=pd)
        g_tau = g_tau + gin[:, nx:nx + t.shape[1]].astype(np.float32)
        g = gin[:, :nx].astype(np.float32).astype(np.float64)
    assert rel(q0.grad.cpu().numpy().astype(np.float64), g[:, :sim.n_q]) <= 1e-6
    assert rel(qd0.grad.cpu().numpy().astype(np.float64), g[:, sim.n_q:]) <= 1e-6
    assert rel(tau.grad.cpu().numpy().astype(np.float64), g_tau.astype(np.float64)) <= 1e-6


def test_batched_inverse_kinematics_at_4096_environments():
    model, qt, rng = laikago_targets(4096, 22)
    sim = _sim(model, 4096)
    lc = np.zeros((4, 3))

    def kin(q):
        _, _, x, J = sim.kinematics_host(q, LAIKAGO_TOES, lc)
        return x, J
    err, it = laikago_ik(kin, qt, rng)
    print(f"laikago IK at 4096 environments: {it} iterations, largest toe error {err.max():.2e} m")
    assert err.max() <= 1e-4 and it <= 15


def test_pytinydiffsim_point_jacobian_on_the_laikago_urdf():
    import emu_kin
    import pytinydiffsim as pd
    from oracle import ref
    model = load_model(fixture_path("laikago"))
    mb = pd.TinyMultiBody(False)
    mb._model = model
    mb._bind(tds_b200.BatchSim(model, 1, precision=1))
    q = f32(fixture("laikago")[1][0])
    mb.q[:] = q
    live = ref.RefSim.from_model(model) if ref.available() else None
    R, p, _, _ = mb._sim.kinematics_host(q[None], [], np.zeros((0, 3)))
    for link in (-1, 0, 5, 9, 17, 21):
        local = np.array([0.03, -0.02, 0.05])
        J_local = pd.point_jacobian(mb, link, local, True)
        world = local if link < 0 else R[0, link] @ local + p[0, link]
        J_world = pd.point_jacobian(mb, link, world)
        Jo = emu_kin.oracle_point_jacobian(model, q, link, world)
        assert J_local.shape == (3, 18)
        for J in (J_local, J_world):
            assert np.abs(J - Jo).max() <= 1e-10 * max(1.0, np.abs(Jo).max()), link
        if live is not None:
            assert np.abs(J_world - live.point_jacobian(q, link, world)).max() <= 1e-8 * max(1.0, np.abs(Jo).max())


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n = q.shape[0]
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    ip = lambda a: ctypes.c_void_p(a.ctypes.data)
    qh = np.ascontiguousarray(q)
    lk, lc = np.array([0, 1], dtype=np.int32), np.zeros((2, 3))
    bad = np.array([0, 2], dtype=np.int32)
    xf, x, J = np.zeros((n, 2, 12)), np.zeros((n, 2, 3)), np.zeros((n, 2, 3, 2))
    assert L.tds_b200_kinematics_host(h, dp(qh), 2, ip(lk), dp(lc), dp(xf), dp(x), dp(J)) == 0
    assert L.tds_b200_kinematics_host(None, dp(qh), 2, ip(lk), dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, None, 2, ip(lk), dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), -1, ip(lk), dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 65, ip(lk), dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 2, ip(bad), dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 2, None, dp(lc), dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 2, ip(lk), None, dp(xf), dp(x), dp(J)) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 2, ip(lk), dp(lc), None, None, None) == -1
    assert L.tds_b200_kinematics_host(h, dp(qh), 0, None, None, dp(xf), None, None) == 0
    assert L.tds_b200_kinematics_device(h, None, 2, ip(lk), dp(lc), None, None, None, None) == -1
    t, tx = np.zeros((n, 2, 1)), np.zeros((n, 6, 1))
    assert L.tds_b200_kinematics_jvp_host(h, dp(qh), 2, ip(lk), dp(lc), 0, dp(t), None, dp(tx), None) == -1
    assert L.tds_b200_kinematics_jvp_host(h, dp(qh), 2, ip(lk), dp(lc), 1, None, None, dp(tx), None) == -1
    assert L.tds_b200_kinematics_jvp_host(h, dp(qh), 2, ip(lk), dp(lc), 1, dp(t), None, None, None) == -1
    assert L.tds_b200_kinematics_jvp_host(h, dp(qh), 2, ip(bad), dp(lc), 1, dp(t), None, dp(tx), None) == -1
    assert L.tds_b200_kinematics_jvp_device(h, None, 2, ip(lk), dp(lc), 1, None, None, None, None, None) == -1
    G, g = np.zeros((n, 6)), np.zeros((n, 2))
    assert L.tds_b200_kinematics_vjp_host(h, dp(qh), 2, ip(lk), dp(lc), None, dp(G), None, dp(g)) == 0
    assert L.tds_b200_kinematics_vjp_host(h, dp(qh), 2, ip(lk), dp(lc), None, None, None, dp(g)) == -1
    assert L.tds_b200_kinematics_vjp_host(h, dp(qh), 2, ip(lk), dp(lc), None, dp(G), None, None) == -1
    assert L.tds_b200_kinematics_vjp_host(h, dp(qh), 65, ip(lk), dp(lc), None, dp(G), None, dp(g)) == -1
    assert L.tds_b200_kinematics_vjp_device(h, None, 2, ip(lk), dp(lc), None, None, None, None, None) == -1
    with pytest.raises(ValueError):
        tds_b200.autograd.forward_kinematics(sim, torch.zeros((n, 2), dtype=torch.float64, device="cuda"), lk, lc)
    with pytest.raises(ValueError):
        sim.kinematics_host(qh, [0, 1], np.zeros((3, 3)))
    with pytest.raises(RuntimeError):
        sim.kinematics_host(qh, [0, 2], np.zeros((2, 3)))
