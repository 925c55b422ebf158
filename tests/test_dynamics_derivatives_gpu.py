"""The derivatives d tau / dq and d tau / dqd of the inverse dynamics on the H100 (DESIGN.md section 7.23): the DER instances of the
world-frame kernel as nvcc builds them, against the host build of the same source, on ragged and chunked batches, with installed
parameters, through torch.autograd (backward, forward_ad, torch.func.jvp), every argument check of the C-ABI, and at 4096 Laikago and
humanoid environments against the device inverse-dynamics JVP along dq_dt tangents.  The CPU twins are in
tests/test_dynamics_derivatives_on_host.py."""
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


def _v(model, n, seed):
    return f32(np.random.default_rng(seed).normal(size=(n, int(model[4]))) * 0.7)


@pytest.mark.parametrize("name", ORACLE_FIXTURES + OTHER_FIXTURES)
def test_device_against_the_host_build(name):
    import emu_dynamics_derivatives as ed
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = _v(model, n, 3), _v(model, n, 4)
    sim = _sim(model, n)
    ref = ed.inverse_dynamics_derivatives(model, q, qd, qdd)
    got = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
    assert rel(got[0], ref[0]) <= 1e-12 and rel(got[1], ref[1]) <= 1e-12
    rng = np.random.default_rng(12)
    tq, tqd, tqdd = rng.normal(size=(n, n_q, 2)), rng.normal(size=(n, nd, 2)), rng.normal(size=(n, nd, 2))
    a, b, ta, tb = sim.inverse_dynamics_derivatives_jvp_host(q, qd, qdd, tq, tqd, tqdd)
    ra, rb = ed.inverse_dynamics_derivatives_jvp(model, q, qd, qdd, tq, tqd, tqdd)
    assert rel(a, ref[0]) <= 1e-12 and rel(b, ref[1]) <= 1e-12
    assert rel(ta, ra) <= 1e-12 and rel(tb, rb) <= 1e-12


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q, qd, qdd = _q(model, 4096, 3), _v(model, 4096, 4), _v(model, 4096, 5)
    full = _sim(model, 4096).inverse_dynamics_derivatives_host(q, qd, qdd)
    for n in (1, 31, 33, 100):
        got = _sim(model, n).inverse_dynamics_derivatives_host(q[-n:], qd[-n:], qdd[-n:])
        assert np.array_equal(got[0], full[0][-n:]) and np.array_equal(got[1], full[1][-n:]), n


def test_humanoid_jvp_in_several_chunks_equals_one_call():
    """A humanoid batch sized so that m = n_q + 2 n_qd tangents run in at least three launches of the chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_in = probe.n_q + 2 * probe.n_qd
    n = 32 * (probe.jacobian_chunk() * 3 // n_in + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    q, qd, qdd = _q(model, n, 5), _v(model, n, 6), _v(model, n, 7)
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    nq, nd = sim.n_q, sim.n_qd
    _, _, wa, wb = sim.inverse_dynamics_derivatives_jvp_host(q, qd, qdd, V[:, :nq], V[:, nq:nq + nd], V[:, nq + nd:])
    assert n_in > 2 * chunk, (chunk, n_in)
    for j0 in range(0, n_in, chunk):
        s_ = slice(j0, j0 + chunk)
        _, _, pa, pb = sim.inverse_dynamics_derivatives_jvp_host(q, qd, qdd, V[:, :nq, s_], V[:, nq:nq + nd, s_], V[:, nq + nd:, s_])
        assert np.array_equal(pa, wa[..., s_]) and np.array_equal(pb, wb[..., s_]), j0


def test_parameters_installed_changed_cleared_and_steps_around_calls():
    from tds_b200.model import set_param_values
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, qdd = _v(model, n, 3), _v(model, n, 4)
    sim = _sim(model, n)
    sim.step_host(2, q, qd)
    D0 = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
    ids = [i for i in all_ids(model) if i >= 2]
    for seed in (15, 16):
        vals = perturbed(model, ids, n, seed, 0.5, 0.0)
        sim.set_physical_params(ids, vals)
        D1 = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
        sim.step_host(2, q, qd)
        for e in range(n):
            ref = _sim(set_param_values(model, ids, vals[e]), 1).inverse_dynamics_derivatives_host(q[e:e + 1], qd[e:e + 1], qdd[e:e + 1])
            assert np.array_equal(D1[0][e:e + 1], ref[0]) and np.array_equal(D1[1][e:e + 1], ref[1]), (seed, e)
    sim.set_physical_params(None)
    sim.step_host(2, q, qd)
    D2 = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
    assert np.array_equal(D0[0], D2[0]) and np.array_equal(D0[1], D2[1])


def test_vjp_is_the_adjoint_of_the_jvp():
    model, q = fixture("laikago")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = _v(model, n, 3), _v(model, n, 4)
    sim = _sim(model, n)
    rng = np.random.default_rng(5)
    tq, tqd, tqdd = rng.normal(size=(n, n_q)), rng.normal(size=(n, nd)), rng.normal(size=(n, nd))
    Ga, Gb = rng.normal(size=(n, nd, nd)), rng.normal(size=(n, nd, nd))
    _, _, ta, tb = sim.inverse_dynamics_derivatives_jvp_host(q, qd, qdd, tq, tqd, tqdd)
    g_q, g_qd, g_qdd, _ = sim.inverse_dynamics_derivatives_vjp_host(q, qd, qdd, Ga, Gb)
    lhs = (Ga * ta).sum(axis=(1, 2)) + (Gb * tb).sum(axis=(1, 2))
    rhs = (g_q * tq).sum(1) + (g_qd * tqd).sum(1) + (g_qdd * tqdd).sum(1)
    assert np.abs(lhs - rhs).max() <= 1e-10 * max(1.0, np.abs(lhs).max())


def test_autograd_against_the_c_abi():
    import torch
    from tds_b200 import autograd as ag
    model, _ = fixture("humanoid_spherical")
    n, n_q, nd = 64, int(model[3]), int(model[4])
    sim = _sim(model, n)
    q, qd, qdd = _q(model, n, 1), _v(model, n, 2), _v(model, n, 3)
    Q, QD, QDD = (torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True) for x in (q, qd, qdd))
    a, b = ag.inverse_dynamics_derivatives(sim, Q, QD, QDD)
    ra, rb = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
    assert rel(a.detach().cpu().numpy(), ra) <= 1e-12 and rel(b.detach().cpu().numpy(), rb) <= 1e-12
    rng = np.random.default_rng(4)
    Ga, Gb = rng.normal(size=(n, nd, nd)), rng.normal(size=(n, nd, nd))
    ((a * torch.tensor(Ga, device="cuda")).sum() + (b * torch.tensor(Gb, device="cuda")).sum()).backward()
    g_q, g_qd, g_qdd, _ = sim.inverse_dynamics_derivatives_vjp_host(q, qd, qdd, Ga, Gb)
    for t, ref in ((Q, g_q), (QD, g_qd), (QDD, g_qdd)):
        assert rel(t.grad.double().cpu().numpy(), f32(ref)) <= 1e-6
    tq, tqd, tqdd = (f32(rng.normal(size=s)) for s in ((n, n_q), (n, nd), (n, nd)))
    _, _, ta, tb = sim.inverse_dynamics_derivatives_jvp_host(q, qd, qdd, tq, tqd, tqdd)
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        ins = [fwAD.make_dual(torch.tensor(x, dtype=torch.float32, device="cuda"), torch.tensor(t, dtype=torch.float32, device="cuda"))
               for x, t in ((q, tq), (qd, tqd), (qdd, tqdd))]
        a2, b2 = ag.inverse_dynamics_derivatives(sim, *ins)
        da, db = fwAD.unpack_dual(a2).tangent, fwAD.unpack_dual(b2).tangent
    assert rel(da.cpu().numpy(), ta) <= 1e-12 and rel(db.cpu().numpy(), tb) <= 1e-12
    prim = [torch.tensor(x, dtype=torch.float32, device="cuda") for x in (q, qd, qdd)]
    tans = [torch.tensor(x, dtype=torch.float32, device="cuda") for x in (tq, tqd, tqdd)]
    _, (da, db) = torch.func.jvp(lambda x, y, z: ag.inverse_dynamics_derivatives(sim, x, y, z), tuple(prim), tuple(tans))
    assert rel(da.cpu().numpy(), ta) <= 1e-12 and rel(db.cpu().numpy(), tb) <= 1e-12


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
    D = L.tds_b200_inverse_dynamics_derivatives_device
    assert D(h, p(None), p(None), p(None), p(out), p(out), None) == -1
    assert D(h, p(q), p(None), p(None), p(None), p(None), None) == -1
    J = L.tds_b200_inverse_dynamics_derivatives_jvp_device
    assert J(h, p(q), p(None), p(None), 1, p(t), p(None), p(None), p(None), p(None), p(None), p(None), p(None), None) == -1
    assert J(h, p(q), p(None), p(None), 0, p(t), p(None), p(None), p(None), p(None), p(None), p(out), p(None), None) == -1
    assert J(h, p(q), p(None), p(None), 1, p(None), p(None), p(None), p(None), p(None), p(None), p(out), p(None), None) == -1
    assert J(h, p(q), p(None), p(None), 1, p(None), p(None), p(None), p(t), p(None), p(None), p(out), p(None), None) == -4
    V = L.tds_b200_inverse_dynamics_derivatives_vjp_device
    assert V(h, p(q), p(None), p(None), p(None), p(None), p(g), p(None), p(None), p(None), None) == -1
    assert V(h, p(q), p(None), p(None), p(out), p(None), p(None), p(None), p(None), p(None), None) == -1
    assert V(h, p(q), p(None), p(None), p(out), p(None), p(None), p(None), p(None), p(g), None) == -4
    qh = np.zeros((n, n_q))
    oh = np.zeros((n, nd * nd))
    dp = lambda x: None if x is None else x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert L.tds_b200_inverse_dynamics_derivatives_host(h, dp(None), None, None, dp(oh), dp(oh)) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_host(h, dp(qh), None, None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_jvp_host(h, dp(qh), None, None, 1, None, None, None, dp(qh), None, None, dp(oh), None) == -4
    assert L.tds_b200_inverse_dynamics_derivatives_vjp_host(h, dp(qh), None, None, dp(oh), None, None, None, None, dp(qh)) == -4


@pytest.mark.parametrize("name", ["laikago", "humanoid"])
def test_columns_against_the_device_inverse_dynamics_jvp(name):
    """At 4096 environments: column k of d tau / dq is inverse_dynamics_jvp along dq_dt(q, e_k), of d tau / dqd along e_k."""
    model, _ = fixture(name)
    n, n_q, nd = 4096, int(model[3]), int(model[4])
    sim = _sim(model, n)
    q, qd, qdd = _q(model, n, 9), _v(model, n, 10), _v(model, n, 11)
    a, b = sim.inverse_dynamics_derivatives_host(q, qd, qdd)
    tq = np.stack([np.stack([dq_dt(model, x, e) for e in np.eye(nd)], axis=1) for x in q.astype(np.float64)])
    _, Jq = sim.inverse_dynamics_jvp_host(q, qd, qdd, t_q=tq)
    _, Jqd = sim.inverse_dynamics_jvp_host(q, qd, qdd, t_qd=np.broadcast_to(np.eye(nd), (n, nd, nd)).copy())
    assert rel(a, Jq) <= 1e-10
    assert rel(b, Jqd) <= 1e-10
