"""Inverse dynamics tau = ID(q, qd, qdd) on the H100 (DESIGN.md section 7.14): the INV instances of the world-frame kernel as nvcc builds
them, against the host build of the same source and the C oracle, on ragged and chunked batches, with installed parameters, through
torch.autograd (backward, forward_ad, torch.func.jvp), the round trip through the MODE_FD step, system identification at 4096
environments, pytinydiffsim.inverse_dynamics / bias_forces, and every argument check of the C-ABI.  The CPU twins are in
tests/test_inverse_dynamics_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from tds_b200.model import fixture_path, load_model, param_names, param_values, set_param_values
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, rel
from test_params_on_host import all_ids, perturbed
from test_inverse_dynamics_on_host import links_of, state

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


def _ids(model):
    return [i for i in all_ids(model) if param_names(model)[i] not in ("friction", "restitution")]


@pytest.mark.parametrize("name", ALL)
def test_device_against_the_host_build_and_the_oracle(name):
    import emu_invdyn
    model, q = fixture(name)
    qd, qdd = state(model, q)
    sim = _sim(model, q.shape[0])
    tau = sim.inverse_dynamics_host(q, qd, qdd)
    assert rel(tau, emu_invdyn.inverse_dynamics(model, q, qd, qdd)) <= 1e-12
    assert rel(sim.inverse_dynamics_host(q, qd), emu_invdyn.inverse_dynamics(model, q, qd)) <= 1e-12
    assert rel(sim.inverse_dynamics_host(q), emu_invdyn.inverse_dynamics(model, q)) <= 1e-12
    if name in ORACLE_FIXTURES:
        to = np.array([emu_invdyn.oracle(model, a, b, c) for a, b, c in zip(f32(q), qd, qdd)])
        assert np.all(np.abs(tau - to) <= 1e-10 * np.maximum(1.0, np.abs(to)))


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 100, 3)
    qd, qdd = state(model, q, 4)
    full = _sim(model, 100).inverse_dynamics_host(q, qd, qdd)
    for n in (1, 31, 33, 100):
        assert np.array_equal(_sim(model, n).inverse_dynamics_host(q[-n:], qd[-n:], qdd[-n:]), full[-n:]), n


def test_device_layout_and_host_layout_agree():
    import torch
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, qdd = state(model, q)
    sim = _sim(model, n)

    def soa(x):
        t = torch.zeros((x.shape[1], sim.n_stride), dtype=torch.float32, device="cuda")
        t[:, :n] = torch.tensor(x.T, dtype=torch.float32)
        return t
    tau = torch.zeros((sim.n_qd, sim.n_stride), dtype=torch.float64, device="cuda")
    sim.inverse_dynamics_device(soa(q), soa(qd), soa(qdd), tau)
    torch.cuda.synchronize()
    assert np.array_equal(tau[:, :n].t().cpu().numpy(), sim.inverse_dynamics_host(q, qd, qdd))


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_invdyn
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, q)
    sim = _sim(model, n)
    ids = _ids(model)
    vals = perturbed(model, ids, n, 12, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(13)
    vin, vp = rng.normal(size=(n, n_q + 2 * nd, 2)), rng.normal(size=(n, len(ids), 2))
    tau, dtau = sim.inverse_dynamics_jvp_host(q, qd, qdd, vin[:, :n_q], vin[:, n_q:n_q + nd], vin[:, n_q + nd:], vp)
    assert rel(tau, emu_invdyn.inverse_dynamics(model, q, qd, qdd, ids=ids, values=vals)) <= 1e-12
    assert rel(dtau, emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, vin, vp, ids=ids, values=vals)) <= 1e-12
    Gc = rng.normal(size=(n, nd))
    g_q, g_qd, g_qdd, g_par = sim.inverse_dynamics_vjp_host(q, qd, qdd, Gc)
    h_in, h_par = emu_invdyn.inverse_dynamics_vjp(model, q, qd, qdd, Gc, ids=ids, values=vals)
    assert rel(np.concatenate([g_q, g_qd, g_qdd], axis=1), h_in) <= 1e-12 and rel(g_par, h_par) <= 1e-12
    fwd = np.einsum("ei,ei->e", Gc, dtau[..., 0])
    rev = np.einsum("ec,ec->e", np.concatenate([g_q, g_qd, g_qdd], axis=1), vin[:, :, 0]) + np.einsum("ek,ek->e", g_par, vp[:, :, 0])
    assert rel(fwd, rev) <= 1e-10


def test_humanoid_jvp_in_several_chunks_equals_one_chunk():
    """A humanoid batch sized so that m = n_in tangents run in at least three launches of the chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_in = probe.n_q + 2 * probe.n_qd
    warps = probe.jacobian_chunk() * 3 // n_in + 1
    n = 32 * warps
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    assert 1 <= chunk and n_in >= 3 * chunk - 2, (chunk, n_in)
    q = _q(model, n, 5)
    qd, qdd = state(model, q, 6)
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    split = lambda v: (v[:, :sim.n_q], v[:, sim.n_q:sim.n_q + sim.n_qd], v[:, sim.n_q + sim.n_qd:])
    _, dtau = sim.inverse_dynamics_jvp_host(q, qd, qdd, *split(V))
    for j0 in range(0, n_in, chunk):
        _, part = sim.inverse_dynamics_jvp_host(q, qd, qdd, *split(V[:, :, j0:j0 + chunk]))
        assert np.array_equal(part, dtau[..., j0:j0 + chunk]), j0


def test_parameter_sets_installed_changed_and_cleared():
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, qdd = state(model, q)
    sim = _sim(model, n)
    before = sim.step_host(2, q, qd)
    t0 = sim.inverse_dynamics_host(q, qd, qdd)
    ids = _ids(model)
    sim.set_physical_params(ids, param_values(model)[ids])
    assert np.array_equal(sim.inverse_dynamics_host(q, qd, qdd), t0)
    vals = perturbed(model, ids, n, 14, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    t1 = sim.inverse_dynamics_host(q, qd, qdd)
    for e in range(n):
        assert np.array_equal(t1[e:e + 1], _sim(set_param_values(model, ids, vals[e]), 1).inverse_dynamics_host(q[e:e + 1], qd[e:e + 1],
                                                                                                                qdd[e:e + 1]))
    sim.set_physical_params(None)
    assert np.array_equal(sim.inverse_dynamics_host(q, qd, qdd), t0)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_and_forward_mode(with_params):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture("humanoid")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, q)
    q = f32(q)
    sim = _sim(model, n)
    ids = _ids(model)[:20] if with_params else []
    vals = perturbed(model, ids, n, 15, 0.5, 0.0) if with_params else None
    if with_params:
        sim.set_physical_params(ids, vals)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    xs = [cu(q), cu(qd), cu(qdd)]
    pt = cu(vals, torch.float64) if with_params else None
    rng = np.random.default_rng(16)
    Gc = rng.normal(size=(n, nd))
    xr = [x.clone().requires_grad_(True) for x in xs]
    pr = pt.clone().requires_grad_(True) if with_params else None
    tau = tds_b200.autograd.inverse_dynamics(sim, *xr, params=pr)
    assert tau.dtype == torch.float64 and tuple(tau.shape) == (n, nd)
    assert np.array_equal(tau.detach().cpu().numpy(), sim.inverse_dynamics_host(q, qd, qdd))
    (tau * cu(Gc, torch.float64)).sum().backward()
    ref = sim.inverse_dynamics_vjp_host(q, qd, qdd, Gc)
    for x, g in zip(xr, ref[:3]):
        assert x.grad.dtype == torch.float32 and rel(x.grad.cpu().numpy().astype(np.float64), g.astype(np.float32).astype(np.float64)) <= 1e-12
    if with_params:
        assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), ref[3]) <= 1e-12
    v = [f32(rng.normal(size=x.shape)) for x in (q, qd, qdd)]
    vp = rng.normal(size=(n, len(ids))) if with_params else None
    _, want = sim.inverse_dynamics_jvp_host(q, qd, qdd, *v, vp)
    ts = [cu(x) for x in v]
    tp = cu(vp, torch.float64) if with_params else None
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x, t) for x, t in zip(xs, ts)]
        dp = fwAD.make_dual(pt, tp) if with_params else None
        tan = fwAD.unpack_dual(tds_b200.autograd.inverse_dynamics(sim, *duals, params=dp)).tangent.cpu().numpy()
    assert rel(tan, want) <= 1e-12
    if with_params:
        _, (ft,) = torch.func.jvp(lambda a, b, c, d: (tds_b200.autograd.inverse_dynamics(sim, a, b, c, d),), (*xs, pt), (*ts, tp))
    else:
        _, (ft,) = torch.func.jvp(lambda a, b, c: (tds_b200.autograd.inverse_dynamics(sim, a, b, c),), tuple(xs), tuple(ts))
    assert rel(ft.cpu().numpy(), want) <= 1e-12


@pytest.mark.parametrize("name", ["laikago", "ant", "pendulum5spherical"])
def test_step_round_trip_in_forward_dynamics_mode(name):
    """ID's tau for a target qdd, fed to autograd.step in MODE_FD, reproduces qdd (fixed base; fp32 step inputs and outputs)."""
    import torch
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    qd, qdd = state(model, q, 7, 0.5)
    sim = _sim(model, n)
    tau = sim.inverse_dynamics_host(q, qd, qdd)
    cu = lambda x: torch.tensor(x, dtype=torch.float32, device="cuda")
    got = tds_b200.autograd.step(sim, cu(q), cu(qd), cu(tau), mode=tds_b200.MODE_FD).detach().cpu().numpy().astype(np.float64)
    M = sim.mass_matrix_host(q)
    bound = 8 * 2.0 ** -24 * (np.abs(tau).max() + np.abs(M).max() * np.abs(qdd).max()) * np.abs(np.linalg.inv(M)).max() * nd
    assert np.abs(got - qdd).max() <= bound, (np.abs(got - qdd).max(), bound)


def test_system_identification_at_4096_environments():
    """Laikago, 4096 environments each with its own masses and damping off by +-20 %: one Gauss-Newton step per environment on the
    torque residual of 6 samples, the Jacobian from the parameter JVP on the device, recovers the true values within 1e-8."""
    model, _ = fixture("laikago")
    names, L = param_names(model), links_of(model)
    link = lambda i: int(names[i][4:].split(".")[0])
    ids = [i for i, nm in enumerate(names) if nm.startswith("link") and
           ((nm.endswith(".mass") and L[link(i), 19] > 0) or (nm.endswith(".damping") and L[link(i), 1] >= 0))]
    rng = np.random.default_rng(21)
    E, S, k = 4096, 6, len(ids)
    n_q, nd = int(model[3]), int(model[4])
    truth = param_values(model)[ids]
    damping = np.array([names[i].endswith(".damping") for i in ids])
    truth[damping] = f32(rng.uniform(0.1, 0.5, int(damping.sum())))
    guess = f32(truth * (1.0 + rng.uniform(-0.2, 0.2, size=(E, k))))
    sim = _sim(model, E)
    A = np.zeros((E, S * nd, k))
    r = np.zeros((E, S * nd))
    eye = np.broadcast_to(np.eye(k), (E, k, k))
    for s in range(S):
        q = f32(rng.uniform(-0.5, 0.5, size=(E, n_q)))
        qd, qdd = f32(rng.normal(size=(E, nd))), f32(rng.normal(size=(E, nd)) * 3.0)
        sim.set_physical_params(ids, np.broadcast_to(truth, (E, k)))
        measured = sim.inverse_dynamics_host(q, qd, qdd)
        sim.set_physical_params(ids, guess)
        tau0, J = sim.inverse_dynamics_jvp_host(q, qd, qdd, t_par=eye)
        A[:, s * nd:(s + 1) * nd] = J
        r[:, s * nd:(s + 1) * nd] = measured - tau0
    assert np.all(np.linalg.matrix_rank(A[:64]) == k)
    est = guess + np.stack([np.linalg.lstsq(A[e], r[e], rcond=None)[0] for e in range(E)])
    assert np.all(np.abs(est - truth) <= 1e-8 * np.abs(truth)), np.abs(est / truth - 1).max()


def test_pytinydiffsim_inverse_dynamics_and_bias_forces_on_the_laikago_model():
    import emu_invdyn
    import pytinydiffsim as pd
    model = load_model(fixture_path("laikago"))
    mb = pd.TinyMultiBody(False)
    mb._world = pd.TinyWorld()   # as UrdfToMultiBody2.convert2 binds it
    mb._model = model
    mb._bind(tds_b200.BatchSim(model, 1, precision=1))
    q = f32(fixture("laikago")[1][0])
    rng = np.random.default_rng(9)
    qd, qdd = f32(rng.normal(size=18)), f32(rng.normal(size=18))
    mb.q[:] = q
    q0, qd0 = mb.q.copy(), mb.qd.copy()
    for g in ((0.0, 0.0, -9.81), (0.0, 0.0, -1.62)):
        tau = pd.inverse_dynamics(mb, q, qd, qdd, g)
        assert tau.shape == (18,) and tau.dtype == np.float64
        to = emu_invdyn.oracle(model, q, qd, qdd, g)
        assert np.all(np.abs(tau - to) <= 1e-10 * np.maximum(1.0, np.abs(to)))
        h = pd.bias_forces(mb, q, qd, g)
        ho = emu_invdyn.oracle(model, q, qd, None, g)
        assert np.all(np.abs(h - ho) <= 1e-10 * np.maximum(1.0, np.abs(ho)))
    assert np.array_equal(mb.q, q0) and np.array_equal(mb.qd, qd0)


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n = q.shape[0]
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    qh, tau = np.ascontiguousarray(q), np.zeros((n, 2))
    t, tt, G, g = np.zeros((n, 2, 1)), np.zeros((n, 2, 1)), np.zeros((n, 2)), np.zeros((n, 2))
    assert L.tds_b200_inverse_dynamics_host(None, dp(qh), None, None, dp(tau)) == -1
    assert L.tds_b200_inverse_dynamics_host(h, None, None, None, dp(tau)) == -1
    assert L.tds_b200_inverse_dynamics_host(h, dp(qh), None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_device(h, None, None, None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_jvp_host(h, dp(qh), None, None, 0, dp(t), None, None, None, None, dp(tt)) == -1
    assert L.tds_b200_inverse_dynamics_jvp_host(h, dp(qh), None, None, 1, None, None, None, None, None, dp(tt)) == -1
    assert L.tds_b200_inverse_dynamics_jvp_host(h, dp(qh), None, None, 1, dp(t), None, None, None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_jvp_host(None, dp(qh), None, None, 1, dp(t), None, None, None, None, dp(tt)) == -1
    assert L.tds_b200_inverse_dynamics_jvp_host(h, dp(qh), None, None, 1, None, None, None, dp(t), None, dp(tt)) == -4
    assert L.tds_b200_inverse_dynamics_jvp_device(h, None, None, None, 1, None, None, None, None, None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_vjp_host(h, dp(qh), None, None, dp(G), None, None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_vjp_host(h, dp(qh), None, None, None, dp(g), None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_vjp_host(h, None, None, None, dp(G), dp(g), None, None, None) == -1
    assert L.tds_b200_inverse_dynamics_vjp_host(h, dp(qh), None, None, dp(G), None, None, None, dp(g)) == -4
    assert L.tds_b200_inverse_dynamics_vjp_device(h, None, None, None, None, None, None, None, None, None) == -1
    # a NULL qd / qdd is zero
    assert np.array_equal(sim.inverse_dynamics_host(q), sim.inverse_dynamics_host(q, np.zeros((n, 2)), np.zeros((n, 2))))
    # the Python layer
    z32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        tds_b200.autograd.inverse_dynamics(sim, torch.zeros((n, 2), dtype=torch.float64, device="cuda"), z32(n, 2))
    with pytest.raises(ValueError):
        tds_b200.autograd.inverse_dynamics(sim, z32(n, 2), z32(n, 3))
    with pytest.raises(ValueError):
        tds_b200.autograd.inverse_dynamics(sim, z32(n, 2), z32(n, 2), None, torch.zeros((n, 1), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        sim.inverse_dynamics_jvp_host(q, None, None, np.zeros((n, 3, 1)))
    with pytest.raises(ValueError):
        sim.inverse_dynamics_jvp_host(q, None, None)
