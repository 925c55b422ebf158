"""The dynamics queries' shared C-ABI path on the H100 (DESIGN.md section 7.12): the mass matrix, forward kinematics and inverse dynamics
run their values, JVPs and VJPs through one value launch, the Jacobian's chunk loop and one VJP by identity tangents.  The device and
host entry points of every JVP and VJP agree bit for bit, with and without installed parameters; a NULL input or cotangent is zero and
a NULL output is not computed; and a VJP whose directions run in several chunks of the 1 GB loop matches the host build."""
import ctypes

import numpy as np
import pytest

import tds_b200
from test_inverse_dynamics_on_host import state
from test_mass_matrix_on_host import fixture, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu

MODELS = ["laikago", "humanoid", "mb_three_bodies"]


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return np.asarray(q, dtype=np.float32).astype(np.float64)


def _ids(model):
    from tds_b200.model import param_names
    return [i for i in all_ids(model) if param_names(model)[i] not in ("friction", "restitution")]


def _setup(name, params, n=100):
    model, _ = fixture(name)
    q = _q(model, n, 3)
    qd, qdd = state(model, q, 4)
    sim = tds_b200.BatchSim(model, n, precision=1)
    if params:
        ids = _ids(model)
        sim.set_physical_params(ids, perturbed(model, ids, n, 5, 0.5, 0.0))
    return model, sim, q, qd, qdd


def _dev(x, sim, dtype=None):
    """host [n, ...] -> device [prod(...), n_stride] (float64, or float32 for the state), entry (r, j) of [n, rows, m] at row r m + j"""
    import torch
    if x is None:
        return None
    n = x.shape[0]
    t = torch.zeros((int(np.prod(x.shape[1:])), sim.n_stride), dtype=dtype or torch.float64, device="cuda")
    t[:, :n] = torch.from_numpy(np.ascontiguousarray(x.reshape(n, -1).T)).to(t.dtype).cuda()
    return t


def _zeros(sim, rows):
    import torch
    return torch.zeros((rows, sim.n_stride), dtype=torch.float64, device="cuda")


def _host(t, sim, shape):
    import torch
    torch.cuda.synchronize()
    return t[:, :sim.n_envs].t().cpu().numpy().reshape((sim.n_envs,) + tuple(shape))


def _f32(sim, x):
    import torch
    return _dev(x, sim, torch.float32)


@pytest.mark.parametrize("params", [False, True])
@pytest.mark.parametrize("name", MODELS)
def test_mass_matrix_device_and_host_agree_bitwise(name, params):
    model, sim, q, _, _ = _setup(name, params)
    n, n_q, nd, k, m = sim.n_envs, sim.n_q, sim.n_qd, len(sim.param_ids), 3
    rng = np.random.default_rng(7)
    tq, tp = rng.normal(size=(n, n_q, m)), rng.normal(size=(n, k, m)) if params else None
    M, dM = sim.mass_matrix_jvp_host(q, tq, tp)
    Md, tMd = _zeros(sim, nd * nd), _zeros(sim, nd * nd * m)
    sim.mass_matrix_jvp_device(_f32(sim, q), m, _dev(tq, sim), _dev(tp, sim), tMd, Md)
    assert np.array_equal(_host(Md, sim, (nd, nd)), M) and np.array_equal(_host(tMd, sim, (nd, nd, m)), dM)
    G = rng.normal(size=(n, nd, nd))
    g_q, g_par = sim.mass_matrix_vjp_host(q, G)
    gq_d, gp_d = _zeros(sim, n_q), _zeros(sim, k) if params else None
    sim.mass_matrix_vjp_device(_f32(sim, q), _dev(G, sim), gq_d, gp_d)
    assert np.array_equal(_host(gq_d, sim, (n_q,)), g_q)
    if params:
        assert np.array_equal(_host(gp_d, sim, (k,)), g_par)
        # g_par NULL: the parameter directions are not computed, and g_q does not change
        gq_only = _zeros(sim, n_q)
        sim.mass_matrix_vjp_device(_f32(sim, q), _dev(G, sim), gq_only, None)
        assert np.array_equal(_host(gq_only, sim, (n_q,)), g_q)
        gq_h = np.zeros((n, n_q))
        dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        Gc = np.ascontiguousarray(G)
        assert sim._L.tds_b200_mass_matrix_vjp_host(sim._h, dp(q), dp(Gc), dp(gq_h), None) == 0
        assert np.array_equal(gq_h, g_q)


@pytest.mark.parametrize("params", [False, True])
@pytest.mark.parametrize("name", MODELS)
def test_kinematics_device_and_host_agree_bitwise(name, params):
    model, sim, q, _, _ = _setup(name, params)
    n, n_q, nl, nd, m = sim.n_envs, sim.n_q, sim.n_links, sim.n_qd, 2
    rng = np.random.default_rng(8)
    links, local = np.array([-1, 0, nl - 1, nl // 2]), rng.normal(size=(4, 3)) * 0.1
    K = len(links)
    shapes = [(nl, 12), (K, 3), (K, 3, nd)]
    tq = rng.normal(size=(n, n_q, m))
    dh = sim.kinematics_jvp_host(q, links, local, tq)
    dd = [_zeros(sim, int(np.prod(s)) * m) for s in shapes]
    sim.kinematics_jvp_device(_f32(sim, q), links, local, m, _dev(tq, sim), *dd)
    for a, b, s in zip(dh, dd, shapes):
        assert np.array_equal(_host(b, sim, s + (m,)), a)
    G = [rng.normal(size=(n,) + s) for s in shapes]
    for keep in [(0, 1, 2), (0,), (1,), (2,), (0, 1), (0, 2), (1, 2)]:
        Gk = [g if i in keep else None for i, g in enumerate(G)]
        g_h = sim.kinematics_vjp_host(q, links, local, *Gk)
        g_d = _zeros(sim, n_q)
        sim.kinematics_vjp_device(_f32(sim, q), links, local, *(_dev(g, sim) for g in Gk), g_d)
        assert np.array_equal(_host(g_d, sim, (n_q,)), g_h), keep
        # a NULL cotangent is zero
        assert np.array_equal(sim.kinematics_vjp_host(q, links, local, *(g if i in keep else 0 * G[i] for i, g in enumerate(G))), g_h)


@pytest.mark.parametrize("params", [False, True])
@pytest.mark.parametrize("name", MODELS)
def test_inverse_dynamics_device_and_host_agree_bitwise(name, params):
    model, sim, q, qd, qdd = _setup(name, params)
    n, n_q, nd, k, m = sim.n_envs, sim.n_q, sim.n_qd, len(sim.param_ids), 2
    rng = np.random.default_rng(9)
    t = [rng.normal(size=(n, d, m)) for d in (n_q, nd, nd)]
    tp = rng.normal(size=(n, k, m)) if params else None
    G = rng.normal(size=(n, nd))
    for qd_, qdd_ in [(qd, qdd), (None, qdd), (qd, None), (None, None)]:
        tangent_sets = [(t[0], t[1], t[2], tp), (t[0], None, t[2], None), (None, t[1], None, tp)]
        if params:
            tangent_sets.append((None, None, None, tp))
        for ts in tangent_sets:
            tau, dtau = sim.inverse_dynamics_jvp_host(q, qd_, qdd_, *ts)
            tau_d, dtau_d = _zeros(sim, nd), _zeros(sim, nd * m)
            sim.inverse_dynamics_jvp_device(_f32(sim, q), _f32(sim, qd_), _f32(sim, qdd_), m, *(_dev(x, sim) for x in ts), dtau_d, tau_d)
            assert np.array_equal(_host(tau_d, sim, (nd,)), tau) and np.array_equal(_host(dtau_d, sim, (nd, m)), dtau)
        gh = sim.inverse_dynamics_vjp_host(q, qd_, qdd_, G)
        gd = [_zeros(sim, d) for d in (n_q, nd, nd)] + ([_zeros(sim, k)] if params else [None])
        sim.inverse_dynamics_vjp_device(_f32(sim, q), _f32(sim, qd_), _f32(sim, qdd_), _dev(G, sim), *gd)
        for a, b, d in zip(gh, gd, (n_q, nd, nd, k)):
            if a is not None:
                assert np.array_equal(_host(b, sim, (d,)), a)
        # a NULL output is not written and does not change the others
        g_qdd = _zeros(sim, nd)
        sim.inverse_dynamics_vjp_device(_f32(sim, q), _f32(sim, qd_), _f32(sim, qdd_), _dev(G, sim), None, None, g_qdd, None)
        assert np.array_equal(_host(g_qdd, sim, (nd,)), gh[2])


def test_mass_matrix_vjp_in_several_chunks_matches_the_host_build():
    """The humanoid with every parameter installed at 1024 environments: the n_q + k identity directions of the mass matrix's VJP do
    not fit into one 1 GB chunk."""
    import emu_mass
    model, sim, q, _, _ = _setup("humanoid", True, n=1024)
    ids, n, n_q, nd, k, ns = sim.param_ids, sim.n_envs, sim.n_q, sim.n_qd, len(sim.param_ids), sim.n_stride
    vals = perturbed(model, ids, n, 5, 0.5, 0.0)
    total = n_q + k
    chunk = min(total, max(1, (1 << 30) // (8 * (nd * nd + total) * ns)))
    assert -(-total // chunk) >= 2, (total, chunk)
    G = np.random.default_rng(10).normal(size=(n, nd, nd))
    g_q, g_par = sim.mass_matrix_vjp_host(q, G)
    e = slice(0, 48)
    h_q, h_par = emu_mass.mass_vjp(model, q[e], G[e], ids=ids, values=vals[e])
    assert rel(g_q[e], h_q) <= 1e-12 and rel(g_par[e], h_par) <= 1e-12
