"""The step that reports its contacts on the H100 (DESIGN.md section 7.15): the CF instances of the world-frame kernel as nvcc builds them,
against the host build of the same source and against tds_b200_step_device on the world-frame kernel, on ragged and chunked batches,
with installed parameters, the impulse identity at 4096 environments, torch.autograd (backward, forward_ad, torch.func.jvp), a rollout
loss on foot impulses, and every argument check of the C-ABI.  The CPU twins are in tests/test_contacts_on_host.py."""
import ctypes
import os

import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
from tds_b200.sim import MODE_FULL, MODE_NOCONTACT, MODE_WORLD, MODE_FD
from tds_b200.model import fixture_path, load_model, param_names, param_values
from test_mass_matrix_on_host import fixture, f32, rel
from test_params_on_host import all_ids

pytestmark = pytest.mark.gpu

ENV = dict(friction=1.0, keep_all_points=True)


def _laikago(n, precision=1, **kw):
    return tds_b200.laikago_sim(n, precision=precision, **kw)


def _world_sim(make):
    """A simulator whose tds_b200_step_device runs the world-frame kernel (TDS_B200_KERNEL=world is read at creation)."""
    old = os.environ.get("TDS_B200_KERNEL")
    os.environ["TDS_B200_KERNEL"] = "world"
    try:
        return make()
    finally:
        if old is None:
            del os.environ["TDS_B200_KERNEL"]
        else:
            os.environ["TDS_B200_KERNEL"] = old


def _laikago_state(n, seed=11):
    w = wl.laikago_perturbed(n, seed=seed)
    return w["q"], w["qd"], w["action"]


def _host_env(sim):
    """The env tuple of emu_contacts for a laikago_sim."""
    from tds_b200.envs import LAIKAGO_INITIAL_POSES, LAIKAGO_KP, LAIKAGO_KD, LAIKAGO_MAX_FORCE
    return (12, 6, LAIKAGO_KP, LAIKAGO_KD, LAIKAGO_MAX_FORCE, 0.4) + tuple(LAIKAGO_INITIAL_POSES)


# q', qd' and the records are fp32, and the device contracts products into FMAs where the host build rounds them apart: at fp64 the two
# builds agree to a few fp32 roundings of those outputs; mixed and fp32 within the parity tests' bound for those precisions
@pytest.mark.parametrize("precision,tol", [(1, 1e-6), (0, 5e-5), (2, 5e-5)])
def test_device_against_the_host_build(precision, tol):
    import emu_contacts
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, precision)
    qo, qdo, C = sim.step_contacts_host(MODE_FULL, q, qd, act, use_pd=True)
    hq, hqd, hC = emu_contacts.step_contacts(sim.model, MODE_FULL, q, qd, act, precision=precision, use_pd=True, env=_host_env(sim), **ENV)
    assert rel(qo, hq) <= tol and rel(qdo, hqd) <= tol
    assert rel(C, hC) <= 10 * tol, rel(C, hC)


def test_jvp_device_against_the_host_build():
    """The fp64 derivatives: the dual-number instance on the device against its host build, 1e-12."""
    import emu_contacts
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, 1)
    rows, cols = sim.contact_rows(MODE_FULL, True)
    v = np.random.default_rng(6).normal(size=(64, cols, 2))
    d = sim.step_contacts_jvp_host(MODE_FULL, q, qd, act, v, use_pd=True)
    h = emu_contacts.step_contacts_jvp(sim.model, MODE_FULL, q, qd, act, t_in=v, use_pd=True, env=_host_env(sim), **ENV)
    assert d.shape == h.shape == (64, rows, 2)
    assert rel(d, h) <= 1e-12, rel(d, h)


def _bitwise_case(name, n):
    """(simulator factory, q, qd, tau or actions, use_pd) at n environments: Laikago with PD, the humanoid (capsules on a floating base)
    and a world of three multibodies (contacts between multibodies)."""
    if name == "laikago":
        q, qd, act = _laikago_state(n)
        return (lambda p: _laikago(n, p)), q, qd, act, True
    model, _ = fixture(name)
    if name == "humanoid":
        w = wl.humanoid(n)
        q, qd = w["q"], w["qd"]
    else:
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
        reps = -(-n // g["q_in"].shape[0])
        q, qd = np.tile(g["q_in"], (reps, 1))[:n], np.tile(g["qd_in"], (reps, 1))[:n]
    tau = np.random.default_rng(12).uniform(-1.0, 1.0, size=(n, int(model[4]) - (6 if int(model[2]) else 0)))
    return (lambda p: tds_b200.BatchSim(model, n, precision=p)), q, qd, tau, False


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("with_params", [False, True])
@pytest.mark.parametrize("name", ["laikago", "humanoid", "mb_three_bodies"])
def test_q_and_qd_bitwise_equal_to_the_world_frame_step(name, precision, with_params):
    import torch
    n = 4096
    make, q, qd, u, pd = _bitwise_case(name, n)
    sims = [_world_sim(lambda: make(precision)), make(precision)]
    if with_params:
        ids = all_ids(sims[0].model)
        vals = np.broadcast_to(param_values(sims[0].model, friction=1.0)[ids], (n, len(ids))) * 1.01
        for s in sims:
            s.set_physical_params(ids, vals)
    s_ref, s_cf = sims
    ns = s_ref.n_stride
    soa = lambda x: torch.tensor(np.ascontiguousarray(np.pad(np.asarray(x, dtype=np.float64).T, ((0, 0), (0, ns - n)))),
                                 dtype=torch.float32, device="cuda")
    qs, qds, us = soa(q), soa(qd), soa(u)
    for mode in (MODE_FULL, MODE_WORLD):
        q1, qd1 = torch.zeros_like(qs), torch.zeros_like(qds)
        s_ref.step_device(mode, qs, qds, us, q_out=q1, qd_out=qd1, use_pd=pd)
        torch.cuda.synchronize()
        assert s_ref.kernel_name().startswith("tds_stepw_kernel")
        q2, qd2 = torch.zeros_like(qs), torch.zeros_like(qds)
        C = torch.zeros((10 * s_cf.n_contact_points, ns), dtype=torch.float32, device="cuda")
        s_cf.step_contacts_device(mode, qs, qds, us, q2, qd2, C, use_pd=pd)
        torch.cuda.synchronize()
        assert torch.equal(q1[:, :n], q2[:, :n]) and torch.equal(qd1[:, :n], qd2[:, :n])
        if mode == MODE_FULL:
            assert any(torch.any(C[r::10, :n] != 0) for r in (7, 8, 9))   # active contacts


@pytest.mark.parametrize("name", ["laikago", "humanoid", "mb_three_bodies"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    reps = -(-100 // g["q_in"].shape[0])
    q, qd = np.tile(g["q_in"], (reps, 1))[:100], np.tile(g["qd_in"], (reps, 1))[:100]
    full = tds_b200.BatchSim(model, 100, precision=1).step_contacts_host(MODE_FULL, q, qd)
    for n in (1, 31, 33, 100):
        part = tds_b200.BatchSim(model, n, precision=1).step_contacts_host(MODE_FULL, q[-n:], qd[-n:])
        for a, b in zip(part, full):
            assert np.array_equal(a, b[-n:]), n


def test_humanoid_jvp_in_chunks_equals_one_call():
    model, _ = fixture("humanoid")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "humanoid.npz"))
    n = 64
    q, qd = g["q_in"][:n], g["qd_in"][:n]
    sim = tds_b200.BatchSim(model, n, precision=1)
    rows, cols = sim.contact_rows(MODE_FULL)
    eye = np.broadcast_to(np.eye(cols), (n, cols, cols))
    J = sim.step_contacts_jvp_host(MODE_FULL, q, qd, None, eye)
    assert J.shape == (n, rows, cols)
    for c0 in range(0, cols, 7):
        part = sim.step_contacts_jvp_host(MODE_FULL, q, qd, None, np.ascontiguousarray(eye[:, :, c0:c0 + 7]))
        assert np.array_equal(part, J[:, :, c0:c0 + 7])
    # the q' | qd' rows are the step's Jacobian
    assert np.array_equal(J[:, :sim.n_q + sim.n_qd], sim.step_jacobian_host(MODE_FULL, q, qd))


def test_vjp_is_the_adjoint_of_the_jvp():
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, 1)
    rows, cols = sim.contact_rows(MODE_FULL, True)
    rng = np.random.default_rng(4)
    G, v = rng.normal(size=(64, rows)), rng.normal(size=(64, cols))
    g_in, g_par = sim.step_contacts_vjp_host(MODE_FULL, q, qd, act, G, use_pd=True)
    assert g_par is None
    Jv = sim.step_contacts_jvp_host(MODE_FULL, q, qd, act, v, use_pd=True)
    lhs, r = np.einsum("er,er->e", G, Jv), np.einsum("ec,ec->e", g_in, v)
    assert np.all(np.abs(lhs - r) <= 1e-10 * np.maximum(1.0, np.abs(r)))


def test_impulse_identity_at_4096_environments():
    """M (qd'_FULL - qd'_NOCONTACT) = sum_c J_c^T F_c on Laikago (fixed base: every candidate is on a leg link, the plane has no dofs),
    fp64, with M from mass_matrix_host and J from the records' points through kinematics_host, link by link."""
    n = 4096
    q, qd, act = _laikago_state(n, 5)
    sim = _laikago(n, 1)
    _, qd_full, C = sim.step_contacts_host(MODE_FULL, q, qd, act, use_pd=True)
    qd_nc = sim.step_host(MODE_NOCONTACT, q, qd, act, use_pd=True)["qd"]
    M = sim.mass_matrix_host(q)
    lhs = np.einsum("eij,ej->ei", M, qd_full - qd_nc)
    m = np.ascontiguousarray(sim.model)
    t = np.zeros((128, 4), dtype=np.int32)
    k = tds_b200._lib.lib().tds_b200_model_contact_pairs(m.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), m.size,
                                                         ctypes.c_void_p(t.ctypes.data), 128)
    R_all, p_all, _, _ = sim.kinematics_host(q, [0], np.zeros((1, 3)))
    rhs, mag = np.zeros_like(lhs), np.zeros_like(lhs)
    for c in range(k):
        link = t[c, 3]
        local = np.einsum("eji,ej->ei", R_all[:, link], C[:, c, 3:6] - p_all[:, link])   # the point in the link frame, per environment
        # the Jacobian of a point is affine in its local coordinates: J(local) = J(0) + sum_a local_a (J(e_a) - J(0))
        J0 = sim.kinematics_host(q, [link], np.zeros((1, 3)))[3][:, 0]
        JJ = [sim.kinematics_host(q, [link], np.eye(3)[a][None])[3][:, 0] - J0 for a in range(3)]
        J = J0 + sum(local[:, a, None, None] * JJ[a] for a in range(3))
        rhs += np.einsum("eij,ei->ej", J, C[:, c, 7:10])
        mag += np.einsum("eij,ei->ej", np.abs(J), np.abs(C[:, c, 7:10]))
    assert np.any(C[:, :, 7:10])
    # the magnitudes whose fp32 roundings (qd' and the records are fp32) enter the two sides
    scale = max(1.0, float(np.max(np.einsum("eij,ej->ei", np.abs(M), np.abs(qd_full) + np.abs(qd_nc)) + mag)))
    assert np.abs(lhs - rhs).max() <= 2e-5 * scale


def _autograd_case(n=64, with_params=False):
    import torch
    q, qd, act = _laikago_state(n, 8)
    sim = _laikago(n, 1)
    params = None
    if with_params:
        ids = [0] + [i for i in all_ids(sim.model) if param_names(sim.model)[i].endswith(".mass")][:3]
        vals = np.broadcast_to(param_values(sim.model, friction=1.0)[ids], (n, len(ids))).copy()
        sim.set_physical_params(ids, vals)
        params = torch.tensor(vals, dtype=torch.float64, device="cuda", requires_grad=True)
    t = lambda x: torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    return sim, t(q), t(qd), t(act), params


@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_against_the_vjp(with_params):
    import torch
    sim, q, qd, a, params = _autograd_case(with_params=with_params)
    q1, qd1, C = tds_b200.autograd.step_contacts(sim, q, qd, a, use_pd=True, params=params)
    rng = np.random.default_rng(1)
    wq, wqd, wC = (torch.tensor(rng.normal(size=x.shape), dtype=torch.float32, device="cuda") for x in (q1, qd1, C))
    ((q1 * wq).sum() + (qd1 * wqd).sum() + (C * wC).sum()).backward()
    n = sim.n_envs
    G = np.concatenate([wq.double().cpu().numpy(), wqd.double().cpu().numpy(), wC.double().cpu().numpy().reshape(n, -1)], axis=1)
    if with_params:
        sim.set_physical_params(sim.param_ids, params.detach())
    g_in, g_par = sim.step_contacts_vjp_host(MODE_FULL, q.detach().cpu().numpy(), qd.detach().cpu().numpy(), a.detach().cpu().numpy(), G,
                                             use_pd=True)
    nq, nd = sim.n_q, sim.n_qd
    assert rel(q.grad.double().cpu().numpy(), f32(g_in[:, :nq])) <= 1e-12
    assert rel(qd.grad.double().cpu().numpy(), f32(g_in[:, nq:nq + nd])) <= 1e-12
    assert rel(a.grad.double().cpu().numpy(), f32(g_in[:, nq + nd:nq + nd + 12])) <= 1e-12
    if with_params:
        assert rel(params.grad.cpu().numpy(), g_par) <= 1e-12


def test_forward_ad_and_func_jvp_against_the_jvp():
    import torch
    import torch.autograd.forward_ad as fwAD
    sim, q, qd, a, _ = _autograd_case()
    rng = np.random.default_rng(2)
    tq, tqd, ta = (torch.tensor(rng.normal(size=x.shape), dtype=torch.float32, device="cuda") for x in (q, qd, a))
    with fwAD.dual_level():
        outs = tds_b200.autograd.step_contacts(sim, fwAD.make_dual(q.detach(), tq), fwAD.make_dual(qd.detach(), tqd),
                                               fwAD.make_dual(a.detach(), ta), use_pd=True)
        tang = [fwAD.unpack_dual(o).tangent for o in outs]
    _, tang2 = torch.func.jvp(lambda x, y, z: tds_b200.autograd.step_contacts(sim, x, y, z, use_pd=True), (q.detach(), qd.detach(), a.detach()),
                              (tq, tqd, ta))
    n = sim.n_envs
    rows, cols = sim.contact_rows(MODE_FULL, True)
    v = np.zeros((n, cols))
    v[:, :sim.n_q], v[:, sim.n_q:sim.n_q + sim.n_qd] = tq.double().cpu().numpy(), tqd.double().cpu().numpy()
    v[:, sim.n_q + sim.n_qd:sim.n_q + sim.n_qd + 12] = ta.double().cpu().numpy()
    ref = sim.step_contacts_jvp_host(MODE_FULL, q.detach().cpu().numpy(), qd.detach().cpu().numpy(), a.detach().cpu().numpy(), v, use_pd=True)
    got = np.concatenate([tang[0].double().cpu().numpy(), tang[1].double().cpu().numpy(), tang[2].double().cpu().numpy().reshape(n, -1)], 1)
    got2 = np.concatenate([tang2[0].double().cpu().numpy(), tang2[1].double().cpu().numpy(), tang2[2].double().cpu().numpy().reshape(n, -1)], 1)
    assert rel(got, f32(ref)) <= 1e-12 and rel(got2, f32(ref)) <= 1e-12


def test_foot_impulse_loss_through_a_rollout_against_chained_vjps():
    """loss = sum over 5 steps of the normal impulses p_n = -F . n_b of every candidate (Laikago's toes), with PD, through
    autograd.step_contacts; the same gradient by chaining the C-ABI's VJPs backwards at the float32 cotangents autograd hands over."""
    import torch
    n, T = 256, 5
    sim, q0, qd0, _, _ = _autograd_case(n)
    rng = np.random.default_rng(9)
    acts = [torch.tensor(rng.uniform(-0.3, 0.3, size=(n, 12)), dtype=torch.float32, device="cuda", requires_grad=True) for _ in range(T)]
    q, qd = q0, qd0
    loss = 0.0
    states = []
    for t in range(T):
        states.append((q.detach().cpu().numpy(), qd.detach().cpu().numpy()))
        q, qd, C = tds_b200.autograd.step_contacts(sim, q, qd, acts[t], use_pd=True)
        loss = loss - (C[:, :, 7:10] * C[:, :, 0:3]).sum()
    loss.backward()
    # by hand: d(-F . n)/dF = -n, d/dn = -F, then q' and qd' carry the cotangents of the later steps
    npts, nq, nd = sim.n_contact_points, sim.n_q, sim.n_qd
    gq, gqd = np.zeros((n, nq), np.float32), np.zeros((n, nd), np.float32)
    g_act = [None] * T
    for t in reversed(range(T)):
        qs, qds = states[t]
        _, _, Ct = sim.step_contacts_host(MODE_FULL, qs, qds, acts[t].detach().cpu().numpy(), use_pd=True)
        Ct = Ct.astype(np.float32)
        GC = np.zeros((n, npts, 10), np.float32)
        GC[:, :, 0:3], GC[:, :, 7:10] = -Ct[:, :, 7:10], -Ct[:, :, 0:3]
        G = np.concatenate([gq, gqd, GC.reshape(n, -1)], axis=1).astype(np.float64)
        g_in, _ = sim.step_contacts_vjp_host(MODE_FULL, qs, qds, acts[t].detach().cpu().numpy(), G, use_pd=True)
        gq, gqd = g_in[:, :nq].astype(np.float32), g_in[:, nq:nq + nd].astype(np.float32)
        g_act[t] = g_in[:, nq + nd:nq + nd + 12].astype(np.float32)
    assert rel(q0.grad.cpu().numpy().astype(np.float64), gq.astype(np.float64)) <= 1e-5
    for t in range(T):
        assert rel(acts[t].grad.cpu().numpy().astype(np.float64), g_act[t].astype(np.float64)) <= 1e-5, t


def test_argument_checks():
    import torch
    q, qd, act = _laikago_state(8)
    sim = _laikago(8, 1)
    L, h = sim._L, sim._h
    dp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    C = np.zeros((8, sim.n_contact_points, 10))
    qo, qdo = np.zeros_like(q), np.zeros_like(qd)
    q, qd, act = (np.ascontiguousarray(x, dtype=np.float64) for x in (q, qd, act))
    assert L.tds_b200_step_contacts_host(None, MODE_FULL, 0, dp(q), dp(qd), None, dp(qo), dp(qdo), dp(C)) == -1
    assert L.tds_b200_step_contacts_host(h, MODE_FULL, 0, None, dp(qd), None, dp(qo), dp(qdo), dp(C)) == -1
    assert L.tds_b200_step_contacts_host(h, MODE_FULL, 0, dp(q), dp(qd), None, dp(qo), dp(qdo), None) == -1
    assert L.tds_b200_step_contacts_host(h, MODE_FULL, 1, dp(q), dp(qd), None, dp(qo), dp(qdo), dp(C)) == -1   # PD without actions
    for mode in (MODE_FD, MODE_NOCONTACT):
        assert L.tds_b200_step_contacts_host(h, mode, 0, dp(q), dp(qd), None, dp(qo), dp(qdo), dp(C)) == -2
    assert L.tds_b200_step_contacts_host(h, MODE_WORLD, 0, dp(q), dp(qd), None, dp(qo), dp(qdo), dp(C)) == 0
    rows, cols = sim.contact_rows(MODE_FULL, True)
    t_in, t_out = np.zeros((8, cols, 1)), np.zeros((8, rows, 1))
    assert L.tds_b200_step_contacts_jvp_host(h, MODE_WORLD, 1, dp(q), dp(qd), dp(act), 1, dp(t_in), None, dp(t_out)) == -2
    assert L.tds_b200_step_contacts_jvp_host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 0, dp(t_in), None, dp(t_out)) == -1
    assert L.tds_b200_step_contacts_jvp_host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 1, None, None, dp(t_out)) == -1
    assert L.tds_b200_step_contacts_jvp_host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 1, dp(t_in), dp(t_in), dp(t_out)) == -4
    G, g_in = np.zeros((8, rows)), np.zeros((8, cols))
    assert L.tds_b200_step_contacts_vjp_host(h, MODE_WORLD, 1, dp(q), dp(qd), dp(act), dp(G), dp(g_in), None) == -2
    assert L.tds_b200_step_contacts_vjp_host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), dp(G), None, None) == -1
    assert L.tds_b200_step_contacts_vjp_host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), dp(G), dp(g_in), dp(g_in)) == -4
    # PD without tds_b200_set_env: -3
    plain = tds_b200.BatchSim(sim.model, 8, precision=1)
    assert plain._L.tds_b200_step_contacts_host(plain._h, MODE_FULL, 1, dp(q), dp(qd), dp(act), dp(qo), dp(qdo), dp(C)) == -3
    assert plain._L.tds_b200_step_contacts_jvp_host(plain._h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 1, dp(t_in), None, dp(t_out)) == -3
    assert plain._L.tds_b200_step_contacts_vjp_host(plain._h, MODE_FULL, 1, dp(q), dp(qd), dp(act), dp(G), dp(g_in), None) == -3
    # device entry points
    ns = sim.n_stride
    z = lambda rows, dt=torch.float32: torch.zeros((rows, ns), dtype=dt, device="cuda")
    qs, qds, acts, Cd = z(sim.n_q), z(sim.n_qd), z(12), z(10 * sim.n_contact_points)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.tds_b200_step_contacts_device(h, MODE_FULL, 1, vp(qs), vp(qds), vp(acts), vp(qs), vp(qds), None, st) == -1
    assert L.tds_b200_step_contacts_device(h, MODE_FD, 1, vp(qs), vp(qds), vp(acts), vp(qs), vp(qds), vp(Cd), st) == -2
    assert L.tds_b200_step_contacts_device(h, MODE_FULL, 1, vp(qs), vp(qds), None, vp(qs), vp(qds), vp(Cd), st) == -1
    assert L.tds_b200_step_contacts_device(h, MODE_FULL, 1, vp(qs), vp(qds), vp(acts), vp(qs), vp(qds), vp(Cd), st) == 0
    assert plain._L.tds_b200_step_contacts_device(plain._h, MODE_FULL, 1, vp(qs), vp(qds), vp(acts), vp(qs), vp(qds), vp(Cd), st) == -3
    ti, to = z(cols, torch.float64), z(rows, torch.float64)
    jvp = lambda sm, hh, mode, m, t_in, t_par, t_out: sm._L.tds_b200_step_contacts_jvp_device(
        hh, mode, 1, vp(qs), vp(qds), vp(acts), m, t_in, t_par, t_out, st)
    assert jvp(sim, h, MODE_FULL, 1, vp(ti), None, None) == -1
    assert jvp(sim, h, MODE_FULL, 0, vp(ti), None, vp(to)) == -1
    assert jvp(sim, h, MODE_FULL, 1, None, None, vp(to)) == -1
    assert jvp(sim, h, MODE_WORLD, 1, vp(ti), None, vp(to)) == -2
    assert jvp(plain, plain._h, MODE_FULL, 1, vp(ti), None, vp(to)) == -3
    assert jvp(sim, h, MODE_FULL, 1, vp(ti), vp(ti), vp(to)) == -4
    assert jvp(sim, h, MODE_FULL, 1, vp(ti), None, vp(to)) == 0
    Gd, gi = z(rows, torch.float64), z(cols, torch.float64)
    vjp = lambda sm, hh, mode, g_out, g_in, g_par: sm._L.tds_b200_step_contacts_vjp_device(
        hh, mode, 1, vp(qs), vp(qds), vp(acts), g_out, g_in, g_par, st)
    assert vjp(sim, h, MODE_FULL, None, vp(gi), None) == -1
    assert vjp(sim, h, MODE_FULL, vp(Gd), None, None) == -1
    assert vjp(sim, h, MODE_FD, vp(Gd), vp(gi), None) == -2
    assert vjp(plain, plain._h, MODE_FULL, vp(Gd), vp(gi), None) == -3
    assert vjp(sim, h, MODE_FULL, vp(Gd), vp(gi), vp(gi)) == -4
    assert vjp(sim, h, MODE_FULL, vp(Gd), vp(gi), None) == 0
    torch.cuda.synchronize()
