"""The derivatives of the forward dynamics d qdd / dq, d qdd / dqd, d qdd / dtau on the H100 (DESIGN.md section 7.24): the product kernel
and the DER instances reading qdd in fp64 as nvcc builds them, composed by the C-ABI, against the host build of the same source, on ragged
and chunked batches, with installed parameters, through torch.autograd (backward, forward_ad, torch.func.jvp), every argument check of
the C-ABI, and at 4096 Laikago and humanoid environments against the device constrained-dynamics JVP (K = 0) along dq_dt and unit
tangents.  The CPU twins are in tests/test_fd_derivatives_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, rel
from test_params_on_host import all_ids, perturbed
from test_point_motion_on_host import dq_dt

pytestmark = pytest.mark.gpu


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return f32(q)


def _v(model, n, seed, scale=0.7):
    return f32(np.random.default_rng(seed).normal(size=(n, int(model[4]))) * scale)


def within(X, ref, sim, q, tol=1e-12):
    """|X - ref| <= tol kappa_2(M_e) max|ref_e| in every environment e (M from the device mass matrix): the solves with M amplify the
    rounding differences between two builds or two routes by M's condition number."""
    k = np.linalg.cond(sim.mass_matrix_host(q))
    n = X.shape[0]
    err = np.abs(X - ref).reshape(n, -1).max(1)
    return bool(np.all(err <= tol * k * np.maximum(np.abs(ref).reshape(n, -1).max(1), 1e-300)))


@pytest.mark.parametrize("name", ORACLE_FIXTURES + OTHER_FIXTURES)
def test_device_against_the_host_build(name):
    import emu_fd_derivatives as ef
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, tau = _v(model, n, 3), _v(model, n, 4, 3.0)
    sim = _sim(model, n)
    ref = ef.forward_dynamics_derivatives(model, q, qd, tau)
    got = sim.forward_dynamics_derivatives_host(q, qd, tau)
    assert np.array_equal(got[3], sim.mass_inverse_host(q)[0])
    assert all(within(a, b, sim, q) for a, b in zip(got, ref)), [rel(a, b) for a, b in zip(got, ref)]
    rng = np.random.default_rng(12)
    tq, tqd, tt = rng.normal(size=(n, n_q, 2)), rng.normal(size=(n, nd, 2)), rng.normal(size=(n, nd, 2))
    out = sim.forward_dynamics_derivatives_jvp_host(q, qd, tau, tq, tqd, tt)
    rt = ef.forward_dynamics_derivatives_jvp(model, q, qd, tau, tq, tqd, tt)
    assert all(np.array_equal(a, b) for a, b in zip(out[:4], got))
    assert all(within(a, b, sim, q) for a, b in zip(out[4:], rt)), [rel(a, b) for a, b in zip(out[4:], rt)]


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q, qd, tau = _q(model, 4096, 3), _v(model, 4096, 4), _v(model, 4096, 5, 3.0)
    full = _sim(model, 4096).forward_dynamics_derivatives_host(q, qd, tau)
    for n in (1, 31, 33, 100):
        got = _sim(model, n).forward_dynamics_derivatives_host(q[-n:], qd[-n:], tau[-n:])
        assert all(np.array_equal(a, b[-n:]) for a, b in zip(got, full)), n


def test_humanoid_jvp_in_several_chunks_equals_one_call():
    """A humanoid batch sized so that m = n_q + 2 n_qd tangents run in several launches of the DER JVP's chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_in = probe.n_q + 2 * probe.n_qd
    n = 32 * (probe.jacobian_chunk() * 3 // n_in + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    q, qd, tau = _q(model, n, 5), _v(model, n, 6), _v(model, n, 7, 3.0)
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    nq, nd = sim.n_q, sim.n_qd
    whole = sim.forward_dynamics_derivatives_jvp_host(q, qd, tau, V[:, :nq], V[:, nq:nq + nd], V[:, nq + nd:])[4:]
    assert n_in > 2 * chunk, (chunk, n_in)
    for j0 in range(0, n_in, chunk):
        s_ = slice(j0, j0 + chunk)
        part = sim.forward_dynamics_derivatives_jvp_host(q, qd, tau, V[:, :nq, s_], V[:, nq:nq + nd, s_], V[:, nq + nd:, s_])[4:]
        assert all(np.array_equal(a, b[..., s_]) for a, b in zip(part, whole)), j0


def test_parameters_installed_changed_cleared_and_steps_around_calls():
    from tds_b200.model import set_param_values
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, tau = _v(model, n, 3), _v(model, n, 4, 3.0)
    sim = _sim(model, n)
    sim.step_host(2, q, qd)
    D0 = sim.forward_dynamics_derivatives_host(q, qd, tau)
    ids = [i for i in all_ids(model) if i >= 2]
    for seed in (15, 16):
        vals = perturbed(model, ids, n, seed, 0.2, 0.0)
        sim.set_physical_params(ids, vals)
        D1 = sim.forward_dynamics_derivatives_host(q, qd, tau)
        sim.step_host(2, q, qd)
        for e in range(n):
            ref = _sim(set_param_values(model, ids, vals[e]), 1).forward_dynamics_derivatives_host(q[e:e + 1], qd[e:e + 1], tau[e:e + 1])
            assert all(np.array_equal(a[e:e + 1], b) for a, b in zip(D1, ref)), (seed, e)
    sim.set_physical_params(None)
    sim.step_host(2, q, qd)
    D2 = sim.forward_dynamics_derivatives_host(q, qd, tau)
    assert all(np.array_equal(a, b) for a, b in zip(D0, D2))


def test_vjp_is_the_adjoint_of_the_jvp():
    model, q = fixture("laikago")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, tau = _v(model, n, 3), _v(model, n, 4, 3.0)
    sim = _sim(model, n)
    ids = [i for i in all_ids(model) if i >= 2][:8]
    sim.set_physical_params(ids, perturbed(model, ids, n, 7, 0.2, 0.0))
    rng = np.random.default_rng(5)
    tq, tqd, tt, tp = rng.normal(size=(n, n_q)), rng.normal(size=(n, nd)), rng.normal(size=(n, nd)), rng.normal(size=(n, len(ids)))
    G = [rng.normal(size=(n, nd))] + [rng.normal(size=(n, nd, nd)) for _ in range(3)]
    tans = sim.forward_dynamics_derivatives_jvp_host(q, qd, tau, tq, tqd, tt, tp)[4:]
    g_q, g_qd, g_tau, g_par = sim.forward_dynamics_derivatives_vjp_host(q, qd, tau, *G)
    lhs = sum((a * b).reshape(n, -1).sum(1) for a, b in zip(G, tans))
    rhs = (g_q * tq).sum(1) + (g_qd * tqd).sum(1) + (g_tau * tt).sum(1) + (g_par * tp).sum(1)
    assert np.abs(lhs - rhs).max() <= 1e-10 * max(1.0, np.abs(lhs).max())


def test_autograd_against_the_c_abi():
    import torch
    from tds_b200 import autograd as ag
    model, _ = fixture("humanoid_spherical")
    n, n_q, nd = 64, int(model[3]), int(model[4])
    sim = _sim(model, n)
    q, qd, tau = _q(model, n, 1), _v(model, n, 2), _v(model, n, 3, 3.0)
    Q, QD, T = (torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True) for x in (q, qd, tau))
    outs = ag.forward_dynamics_derivatives(sim, Q, QD, T)
    ref = sim.forward_dynamics_derivatives_host(q, qd, tau)
    assert all(rel(a.detach().cpu().numpy(), b) <= 1e-12 for a, b in zip(outs, ref))
    rng = np.random.default_rng(4)
    G = [rng.normal(size=(n, nd))] + [rng.normal(size=(n, nd, nd)) for _ in range(3)]
    sum((a * torch.tensor(g, device="cuda")).sum() for a, g in zip(outs, G)).backward()
    g_q, g_qd, g_tau, _ = sim.forward_dynamics_derivatives_vjp_host(q, qd, tau, *G)
    for t, r in ((Q, g_q), (QD, g_qd), (T, g_tau)):
        assert rel(t.grad.double().cpu().numpy(), f32(r)) <= 1e-6
    tq, tqd, tt = (f32(rng.normal(size=s)) for s in ((n, n_q), (n, nd), (n, nd)))
    tref = sim.forward_dynamics_derivatives_jvp_host(q, qd, tau, tq, tqd, tt)[4:]
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        ins = [fwAD.make_dual(torch.tensor(x, dtype=torch.float32, device="cuda"), torch.tensor(t, dtype=torch.float32, device="cuda"))
               for x, t in ((q, tq), (qd, tqd), (tau, tt))]
        tans = [fwAD.unpack_dual(o).tangent for o in ag.forward_dynamics_derivatives(sim, *ins)]
    assert all(rel(a.cpu().numpy(), b) <= 1e-12 for a, b in zip(tans, tref))
    prim = tuple(torch.tensor(x, dtype=torch.float32, device="cuda") for x in (q, qd, tau))
    tang = tuple(torch.tensor(x, dtype=torch.float32, device="cuda") for x in (tq, tqd, tt))
    _, tans = torch.func.jvp(lambda x, y, z: ag.forward_dynamics_derivatives(sim, x, y, z), prim, tang)
    assert all(rel(a.cpu().numpy(), b) <= 1e-12 for a, b in zip(tans, tref))


def test_argument_checks():
    import torch
    model, _ = fixture("laikago")
    n, n_q, nd = 4, int(model[3]), int(model[4])
    sim = _sim(model, n)
    L, h = sim._L, sim._h
    ns = sim.n_stride
    q = torch.zeros(n_q, ns, device="cuda")
    out = torch.zeros(nd * nd, ns, dtype=torch.float64, device="cuda")
    t = torch.zeros(n_q, ns, dtype=torch.float64, device="cuda")
    g = torch.zeros(n_q, ns, dtype=torch.float64, device="cuda")
    p = lambda x: ctypes.c_void_p(None if x is None else x.data_ptr())
    z = p(None)
    D = L.tds_b200_forward_dynamics_derivatives_device
    assert D(h, z, z, z, p(out), p(out), z, z, None) == -1
    assert D(h, p(q), z, z, z, z, z, z, None) == -1
    J = L.tds_b200_forward_dynamics_derivatives_jvp_device
    assert J(h, p(q), z, z, 1, p(t), z, z, z, z, z, z, z, z, z, z, z, None) == -1                 # no tangent output
    assert J(h, p(q), z, z, 0, p(t), z, z, z, z, z, z, z, z, p(out), z, z, None) == -1            # m < 1
    assert J(h, p(q), z, z, 1, z, z, z, z, z, z, z, z, z, p(out), z, z, None) == -1               # no tangent
    assert J(h, p(q), z, z, 1, z, z, z, p(t), z, z, z, z, z, p(out), z, z, None) == -4            # t_par without a set
    V = L.tds_b200_forward_dynamics_derivatives_vjp_device
    assert V(h, p(q), z, z, z, z, z, z, p(g), z, z, z, None) == -1                                # no cotangent
    assert V(h, p(q), z, z, z, p(out), z, z, z, z, z, z, None) == -1                              # no gradient output
    assert V(h, p(q), z, z, z, p(out), z, z, z, z, z, p(g), None) == -4                           # g_par without a set
    qh = np.zeros((n, n_q))
    oh = np.zeros((n, nd * nd))
    dp = lambda x: None if x is None else x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert L.tds_b200_forward_dynamics_derivatives_host(h, dp(None), None, None, dp(oh), None, None, None) == -1
    assert L.tds_b200_forward_dynamics_derivatives_host(h, dp(qh), None, None, None, None, None, None) == -1
    assert L.tds_b200_forward_dynamics_derivatives_jvp_host(h, dp(qh), None, None, 1, None, None, None, dp(qh), None, None, None, None,
                                                            None, dp(oh), None, None) == -4
    assert L.tds_b200_forward_dynamics_derivatives_vjp_host(h, dp(qh), None, None, None, dp(oh), None, None, None, None, None,
                                                            dp(qh)) == -4
    with pytest.raises(ValueError):
        sim.forward_dynamics_derivatives_jvp_host(qh)
    with pytest.raises(ValueError):
        sim.forward_dynamics_derivatives_vjp_host(qh)


@pytest.mark.parametrize("name", ["laikago", "humanoid"])
def test_columns_against_the_device_constrained_dynamics_jvp(name):
    """At 4096 environments: column k of d qdd / dq is constrained_dynamics_jvp (K = 0) along dq_dt(q, e_k), of d qdd / dqd and
    d qdd / dtau along e_k in qd and tau."""
    model, _ = fixture(name)
    n, nd = 4096, int(model[4])
    sim = _sim(model, n)
    q, qd, tau = _q(model, n, 9), _v(model, n, 10), _v(model, n, 11, 3.0)
    _, a, b, c = sim.forward_dynamics_derivatives_host(q, qd, tau)
    tq = np.stack([np.stack([dq_dt(model, x, e) for e in np.eye(nd)], axis=1) for x in q.astype(np.float64)])
    eye = np.broadcast_to(np.eye(nd), (n, nd, nd)).copy()
    for X, t in ((a, dict(t_q=tq)), (b, dict(t_qd=eye)), (c, dict(t_tau=eye))):
        ref = sim.constrained_dynamics_jvp_host(q, qd, tau, **t)[2]
        assert within(X, ref, sim, q), (name, list(t), rel(X, ref))
