"""The step with external wrenches on the H100 (DESIGN.md section 7.18): the EXT instances of the world-frame kernel as nvcc builds them,
against the host build of the same source and against tds_b200_step_contacts_device at zero wrenches, on ragged and chunked batches,
the VJP as the JVP's adjoint, torch.autograd (backward, forward_ad, torch.func.jvp), a rollout gradient and the identification of a push
on Laikago, steps around the calls, and every argument check of the C-ABI.  The CPU twins are in tests/test_wrench_on_host.py."""
import ctypes
import os

import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
from tds_b200.sim import MODE_FULL, MODE_NOCONTACT, MODE_WORLD, MODE_FD
from tds_b200.model import param_names, param_values
from test_mass_matrix_on_host import fixture, f32, rel
from test_params_on_host import all_ids

pytestmark = pytest.mark.gpu

ENV = dict(friction=1.0, keep_all_points=True)
TRUNK = 5                            # Laikago's trunk (the last link of its six root joints); q[0:3] is its position
HANDS_AND_FEET = [13, 22, 27, 32]    # the humanoid's end links


def _laikago(n, precision=1):
    return tds_b200.laikago_sim(n, precision=precision)


def _laikago_state(n, seed=11):
    w = wl.laikago_perturbed(n, seed=seed)
    return w["q"], w["qd"], w["action"]


def _host_env(sim):
    from tds_b200.envs import LAIKAGO_INITIAL_POSES, LAIKAGO_KP, LAIKAGO_KD, LAIKAGO_MAX_FORCE
    return (12, 6, LAIKAGO_KP, LAIKAGO_KD, LAIKAGO_MAX_FORCE, 0.4) + tuple(LAIKAGO_INITIAL_POSES)


def _push(n, K, seed=3, scale=20.0):
    return f32(np.random.default_rng(seed).normal(size=(n, K, 6)) * scale)


TRUNK_PTS = ([TRUNK, TRUNK], np.array([[0.0, 0.0, 0.0], [0.1, -0.05, 0.02]]))


# q', qd' and qdd are fp32, and the device contracts products into FMAs where the host build rounds them apart: at fp64 the two builds
# agree to a few fp32 roundings of those outputs; mixed and fp32 within the parity tests' bound for those precisions.  The PD torques are
# fp32 in every precision, and qdd carries their roundings through M^-1 (Laikago's light toes): qdd is compared per environment, relative
# to its largest entry.
@pytest.mark.parametrize("precision,tol", [(1, 1e-6), (0, 5e-5), (2, 5e-5)])
def test_device_against_the_host_build(precision, tol):
    import emu_wrench
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, precision)
    links, local = TRUNK_PTS
    W = _push(64, 2)
    for mode in (MODE_FD, MODE_NOCONTACT, MODE_FULL):
        d = sim.step_wrench_host(mode, q, qd, act, links, local, W, use_pd=True)
        h = emu_wrench.step_wrench(sim.model, mode, q, qd, act, links, local, W, precision=precision, use_pd=True, env=_host_env(sim), **ENV)
        if mode == MODE_FD:
            err = np.abs(d - h).max(axis=1) / np.maximum(1.0, np.abs(h).max(axis=1))
            assert err.max() <= tol, (mode, err.max())
            continue
        for a, b in zip(d, h):
            assert rel(a, b) <= tol, (mode, rel(a, b))


def test_jvp_device_against_the_host_build():
    """The fp64 derivatives: the dual-number instance on the device against its host build, 1e-12."""
    import emu_wrench
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, 1)
    links, local = TRUNK_PTS
    W = _push(64, 2)
    rows, cols = sim.jacobian_dims(MODE_FULL, True)
    rng = np.random.default_rng(6)
    ti, tw = rng.normal(size=(64, cols, 2)), rng.normal(size=(64, 2, 6, 2))
    d = sim.step_wrench_jvp_host(MODE_FULL, q, qd, act, links, local, W, t_in=ti, t_W=tw, use_pd=True)
    h = emu_wrench.step_wrench_jvp(sim.model, MODE_FULL, q, qd, act, links, local, W, t_in=ti, t_W=tw, use_pd=True, env=_host_env(sim),
                                   **ENV)
    assert d.shape == h.shape == (64, rows, 2)
    assert rel(d, h) <= 1e-12, rel(d, h)


def _case(name, n):
    """(simulator factory, q, qd, tau or actions, use_pd, links, local) at n environments."""
    if name == "laikago":
        q, qd, act = _laikago_state(n)
        return (lambda p: _laikago(n, p)), q, qd, act, True, TRUNK_PTS[0], TRUNK_PTS[1]
    model, _ = fixture(name)
    if name == "humanoid":
        w = wl.humanoid(n)
        q, qd = w["q"], w["qd"]
        links, local = [-1] + HANDS_AND_FEET, np.array([[0.0, 0.05, 0.1]] + [[0.0, 0.0, 0.0]] * 4)
    else:
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
        reps = -(-n // g["q_in"].shape[0])
        q, qd = np.tile(g["q_in"], (reps, 1))[:n], np.tile(g["qd_in"], (reps, 1))[:n]
        links, local = list(range(int(model[1]))), np.full((int(model[1]), 3), 0.03)
    tau = np.random.default_rng(12).uniform(-1.0, 1.0, size=(n, int(model[4]) - (6 if int(model[2]) else 0)))
    return (lambda p: tds_b200.BatchSim(model, n, precision=p)), q, qd, tau, False, links, local


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("with_params", [False, True])
@pytest.mark.parametrize("name", ["laikago", "humanoid", "mb_three_bodies"])
def test_zero_wrenches_bitwise_equal_to_the_contact_step(name, precision, with_params):
    import torch
    n = 4096
    make, q, qd, u, pd, links, local = _case(name, n)
    sim = make(precision)
    if with_params:
        ids = all_ids(sim.model)
        sim.set_physical_params(ids, np.broadcast_to(param_values(sim.model, friction=1.0)[ids], (n, len(ids))) * 1.01)
    ns = sim.n_stride
    soa = lambda x: torch.tensor(np.ascontiguousarray(np.pad(np.asarray(x, dtype=np.float64).T, ((0, 0), (0, ns - n)))),
                                 dtype=torch.float32, device="cuda")
    qs, qds, us = soa(q), soa(qd), soa(u)
    q1, qd1 = torch.zeros_like(qs), torch.zeros_like(qds)
    C = torch.zeros((max(10 * sim.n_contact_points, 1), ns), dtype=torch.float32, device="cuda")
    sim.step_contacts_device(MODE_FULL, qs, qds, us, q1, qd1, C, use_pd=pd)
    W0 = torch.zeros((6 * len(links), ns), dtype=torch.float32, device="cuda")
    for lk, lc in ((links, local), ([], np.zeros((0, 3)))):
        q2, qd2 = torch.zeros_like(qs), torch.zeros_like(qds)
        sim.step_wrench_device(MODE_FULL, qs, qds, us, lk, lc, W0, q2, qd2, use_pd=pd)
        torch.cuda.synchronize()
        assert torch.equal(q1[:, :n], q2[:, :n]) and torch.equal(qd1[:, :n], qd2[:, :n])
    # and a push moves the robot
    W = torch.tensor(np.ascontiguousarray(_push(n, len(links)).reshape(n, -1).T), dtype=torch.float32, device="cuda")
    W = torch.nn.functional.pad(W, (0, ns - n))
    sim.step_wrench_device(MODE_FULL, qs, qds, us, links, local, W, q2, qd2, use_pd=pd)
    torch.cuda.synchronize()
    assert not torch.equal(qd1[:, :n], qd2[:, :n])


@pytest.mark.parametrize("name", ["laikago", "humanoid"])
def test_ragged_batches_equal_their_rows_of_a_4096_batch(name):
    N = 4096
    make, q, qd, u, pd, links, local = _case(name, N)
    W = _push(N, len(links))
    full = make(1).step_wrench_host(MODE_FULL, q, qd, u, links, local, W, use_pd=pd)
    for n in (1, 31, 33, 100):
        if name == "laikago":
            sim = _laikago(n, 1)
        else:
            sim = tds_b200.BatchSim(fixture(name)[0], n, precision=1)
        part = sim.step_wrench_host(MODE_FULL, q[-n:], qd[-n:], u[-n:], links, local, W[-n:], use_pd=pd)
        for a, b in zip(part, full):
            assert np.array_equal(a, b[-n:]), n


def test_humanoid_jvp_in_chunks_equals_one_call():
    n = 64
    make, q, qd, u, pd, links, local = _case("humanoid", n)
    sim = make(1)
    W = _push(n, len(links))
    rows, cols = sim.jacobian_dims(MODE_FULL)
    K = len(links)
    eye = np.broadcast_to(np.eye(cols + 6 * K), (n, cols + 6 * K, cols + 6 * K))
    ti, tw = np.ascontiguousarray(eye[:, :cols]), np.ascontiguousarray(eye[:, cols:].reshape(n, K, 6, -1))
    J = sim.step_wrench_jvp_host(MODE_FULL, q, qd, u, links, local, W, t_in=ti, t_W=tw)
    assert J.shape == (n, rows, cols + 6 * K)
    for c0 in range(0, cols + 6 * K, 7):
        part = sim.step_wrench_jvp_host(MODE_FULL, q, qd, u, links, local, W, t_in=np.ascontiguousarray(ti[..., c0:c0 + 7]),
                                        t_W=np.ascontiguousarray(tw[..., c0:c0 + 7]))
        assert np.array_equal(part, J[:, :, c0:c0 + 7])
    # with the wrenches at zero, the step's columns are the step's Jacobian
    J0 = sim.step_wrench_jvp_host(MODE_FULL, q, qd, u, links, local, np.zeros_like(W), t_in=np.ascontiguousarray(ti[..., :cols]))
    assert rel(J0, sim.step_jacobian_host(MODE_FULL, q, qd, u)) <= 1e-12


@pytest.mark.parametrize("with_params", [False, True])
def test_vjp_is_the_adjoint_of_the_jvp(with_params):
    q, qd, act = _laikago_state(64)
    sim = _laikago(64, 1)
    if with_params:
        ids = [0] + [i for i in all_ids(sim.model) if param_names(sim.model)[i].endswith(".mass")][:3]
        sim.set_physical_params(ids, np.broadcast_to(param_values(sim.model, friction=1.0)[ids], (64, len(ids))))
    links, local = TRUNK_PTS
    W = _push(64, 2)
    rng = np.random.default_rng(4)
    for mode in (MODE_FD, MODE_FULL):
        rows, cols = sim.jacobian_dims(mode, True)
        G, v, vw = rng.normal(size=(64, rows)), rng.normal(size=(64, cols)), rng.normal(size=(64, 2, 6))
        vp = rng.normal(size=(64, len(sim.param_ids))) if with_params else None
        g_in, g_W, g_par = sim.step_wrench_vjp_host(mode, q, qd, act, links, local, W, G, use_pd=True)
        Jv = sim.step_wrench_jvp_host(mode, q, qd, act, links, local, W, t_in=v, t_W=vw, t_par=vp, use_pd=True)
        lhs = np.einsum("er,er->e", G, Jv)
        r = np.einsum("ec,ec->e", g_in, v) + np.einsum("ekr,ekr->e", g_W, vw)
        if with_params:
            r += np.einsum("ek,ek->e", g_par, vp)
        assert np.all(np.abs(lhs - r) <= 1e-10 * np.maximum(1.0, np.abs(r))), mode


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
    return sim, t(q), t(qd), t(act), t(_push(n, 2)), params


@pytest.mark.parametrize("mode", [MODE_FD, MODE_FULL])
@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_against_the_vjp(with_params, mode):
    import torch
    sim, q, qd, a, W, params = _autograd_case(with_params=with_params)
    links, local = TRUNK_PTS
    out = tds_b200.autograd.step_wrench(sim, q, qd, a, links, local, W, mode=mode, use_pd=True, params=params)
    out = (out,) if mode == MODE_FD else out
    rng = np.random.default_rng(1)
    ws = [torch.tensor(rng.normal(size=x.shape), dtype=torch.float32, device="cuda") for x in out]
    sum((o * w).sum() for o, w in zip(out, ws)).backward()
    G = np.concatenate([w.double().cpu().numpy() for w in ws], axis=1)
    if with_params:
        sim.set_physical_params(sim.param_ids, params.detach())
    npy = lambda t: t.detach().cpu().numpy()
    g_in, g_W, g_par = sim.step_wrench_vjp_host(mode, npy(q), npy(qd), npy(a), links, local, npy(W), G, use_pd=True)
    nq, nd = sim.n_q, sim.n_qd
    assert rel(q.grad.double().cpu().numpy(), f32(g_in[:, :nq])) <= 1e-12
    assert rel(qd.grad.double().cpu().numpy(), f32(g_in[:, nq:nq + nd])) <= 1e-12
    assert rel(a.grad.double().cpu().numpy(), f32(g_in[:, nq + nd:nq + nd + 12])) <= 1e-12
    assert rel(W.grad.double().cpu().numpy(), f32(g_W)) <= 1e-12
    if with_params:
        assert rel(params.grad.cpu().numpy(), g_par) <= 1e-12


def test_forward_ad_and_func_jvp_against_the_jvp():
    import torch
    import torch.autograd.forward_ad as fwAD
    sim, q, qd, a, W, _ = _autograd_case()
    links, local = TRUNK_PTS
    rng = np.random.default_rng(2)
    tq, tqd, ta, tW = (torch.tensor(rng.normal(size=x.shape), dtype=torch.float32, device="cuda") for x in (q, qd, a, W))
    with fwAD.dual_level():
        outs = tds_b200.autograd.step_wrench(sim, fwAD.make_dual(q.detach(), tq), fwAD.make_dual(qd.detach(), tqd),
                                             fwAD.make_dual(a.detach(), ta), links, local, fwAD.make_dual(W.detach(), tW), use_pd=True)
        tang = [fwAD.unpack_dual(o).tangent for o in outs]
    _, tang2 = torch.func.jvp(lambda x, y, z, w: tds_b200.autograd.step_wrench(sim, x, y, z, links, local, w, use_pd=True),
                              (q.detach(), qd.detach(), a.detach(), W.detach()), (tq, tqd, ta, tW))
    n = sim.n_envs
    rows, cols = sim.jacobian_dims(MODE_FULL, True)
    v = np.zeros((n, cols))
    v[:, :sim.n_q], v[:, sim.n_q:sim.n_q + sim.n_qd] = tq.double().cpu().numpy(), tqd.double().cpu().numpy()
    v[:, sim.n_q + sim.n_qd:sim.n_q + sim.n_qd + 12] = ta.double().cpu().numpy()
    npy = lambda t: t.detach().cpu().numpy()
    ref = sim.step_wrench_jvp_host(MODE_FULL, npy(q), npy(qd), npy(a), links, local, npy(W), t_in=v, t_W=tW.double().cpu().numpy(),
                                   use_pd=True)
    got = np.concatenate([t.double().cpu().numpy() for t in tang], 1)
    got2 = np.concatenate([t.double().cpu().numpy() for t in tang2], 1)
    assert rel(got, f32(ref)) <= 1e-12 and rel(got2, f32(ref)) <= 1e-12


def test_trunk_loss_through_a_rollout_against_chained_vjps():
    """loss = the trunk position after 5 steps with PD and a per-environment push on the trunk, through autograd.step_wrench; W.grad
    of every step by chaining the C-ABI's VJPs backwards at the float32 cotangents autograd hands over."""
    import torch
    n, T = 256, 5
    sim, q0, qd0, _, _, _ = _autograd_case(n)
    links, local = [TRUNK], np.zeros((1, 3))
    rng = np.random.default_rng(9)
    acts = [torch.tensor(rng.uniform(-0.3, 0.3, size=(n, 12)), dtype=torch.float32, device="cuda") for _ in range(T)]
    Ws = [torch.tensor(_push(n, 1, seed=20 + t), dtype=torch.float32, device="cuda", requires_grad=True) for t in range(T)]
    q, qd = q0, qd0
    states = []
    for t in range(T):
        states.append((q.detach().cpu().numpy(), qd.detach().cpu().numpy()))
        q, qd = tds_b200.autograd.step_wrench(sim, q, qd, acts[t], links, local, Ws[t], use_pd=True)
    q[:, 0:3].sum().backward()
    nq, nd = sim.n_q, sim.n_qd
    gq, gqd = np.zeros((n, nq), np.float32), np.zeros((n, nd), np.float32)
    gq[:, 0:3] = 1.0
    for t in reversed(range(T)):
        qs, qds = states[t]
        G = np.concatenate([gq, gqd], axis=1).astype(np.float64)
        g_in, g_W, _ = sim.step_wrench_vjp_host(MODE_FULL, qs, qds, acts[t].cpu().numpy(), links, local, Ws[t].detach().cpu().numpy(), G,
                                                use_pd=True)
        gq, gqd = g_in[:, :nq].astype(np.float32), g_in[:, nq:nq + nd].astype(np.float32)
        assert rel(Ws[t].grad.cpu().numpy().astype(np.float64), f32(g_W)) <= 1e-6, t
    assert rel(q0.grad.cpu().numpy().astype(np.float64), gq.astype(np.float64)) <= 1e-6


def test_identification_of_a_trunk_push_at_4096_environments():
    """A constant unknown push on the trunk (a different one per environment) from a 3-step trajectory with PD: L-BFGS through
    autograd.step_wrench recovers its force."""
    import torch
    n, T = 4096, 3
    q0, qd0, _ = _laikago_state(n, 13)
    sim = _laikago(n, 1)
    links, local = [TRUNK], np.zeros((1, 3))
    rng = np.random.default_rng(14)
    acts = [torch.tensor(rng.uniform(-0.2, 0.2, size=(n, 12)), dtype=torch.float32, device="cuda") for _ in range(T)]
    f_true = np.zeros((n, 1, 6))
    f_true[:, 0, 3:] = rng.uniform(-60.0, 60.0, size=(n, 3))
    W_true = torch.tensor(f_true, dtype=torch.float32, device="cuda")
    q0t, qd0t = (torch.tensor(x, dtype=torch.float32, device="cuda") for x in (q0, qd0))

    def rollout(W):
        q, qd, out = q0t, qd0t, []
        for t in range(T):
            q, qd = tds_b200.autograd.step_wrench(sim, q, qd, acts[t], links, local, W, mode=MODE_NOCONTACT, use_pd=True)
            out.append(qd)
        return torch.cat(out, 1)

    with torch.no_grad():
        obs = rollout(W_true)
    f = torch.zeros((n, 3), dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.LBFGS([f], lr=1.0, max_iter=40, line_search_fn="strong_wolfe", tolerance_grad=1e-12, tolerance_change=1e-14)

    def closure():
        opt.zero_grad()
        W = torch.cat([torch.zeros((n, 3), device="cuda"), f], 1).reshape(n, 1, 6)
        loss = ((rollout(W) - obs) ** 2).sum()
        loss.backward()
        return loss

    for _ in range(3):
        opt.step(closure)
    err = np.abs(f.detach().cpu().numpy() - f_true[:, 0, 3:]).max()
    assert err <= 1e-2 * 60.0, err


def test_steps_around_wrench_calls_are_unchanged():
    import torch
    n = 256
    q, qd, act = _laikago_state(n)
    sim = _laikago(n, 0)
    ns = sim.n_stride
    soa = lambda x: torch.tensor(np.ascontiguousarray(np.pad(np.asarray(x, dtype=np.float64).T, ((0, 0), (0, ns - n)))),
                                 dtype=torch.float32, device="cuda")
    qs, qds, us = soa(q), soa(qd), soa(act)

    def step():
        q1, qd1 = torch.zeros_like(qs), torch.zeros_like(qds)
        sim.step_device(MODE_FULL, qs, qds, us, q_out=q1, qd_out=qd1, use_pd=True)
        torch.cuda.synchronize()
        return q1, qd1

    a = step()
    links, local = TRUNK_PTS
    W = torch.tensor(np.ascontiguousarray(_push(n, 2).reshape(n, -1).T), dtype=torch.float32, device="cuda")
    W = torch.nn.functional.pad(W, (0, ns - n))
    q2, qd2 = torch.zeros_like(qs), torch.zeros_like(qds)
    sim.step_wrench_device(MODE_FULL, qs, qds, us, links, local, W, q2, qd2, use_pd=True)
    sim.step_wrench_vjp_host(MODE_FULL, q, qd, act, links, local, _push(n, 2), np.ones((n, sim.n_q + sim.n_qd)), use_pd=True)
    b = step()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_argument_checks():
    import torch
    q, qd, act = _laikago_state(8)
    sim = _laikago(8, 1)
    L, h = sim._L, sim._h
    dp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    q, qd, act = (np.ascontiguousarray(x, dtype=np.float64) for x in (q, qd, act))
    qo, qdo, qddo = np.zeros_like(q), np.zeros_like(qd), np.zeros_like(qd)
    lk = np.array([TRUNK, -1], dtype=np.int32)
    lc = np.zeros((2, 3))
    W = np.zeros((8, 2, 6))
    ip = lambda a: ctypes.c_void_p(a.ctypes.data)
    bad = np.array([TRUNK, sim.n_links], dtype=np.int32)
    host = lambda *a: L.tds_b200_step_wrench_host(*a)
    assert host(None, MODE_FULL, 1, dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, None, dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), None, 2, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1   # PD without actions
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 65, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), -1, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 2, ip(bad), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 2, None, dp(lc), dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 2, ip(lk), None, dp(W), dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), None, dp(qo), dp(qdo), None) == -1
    assert host(h, MODE_FD, 1, dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -1      # no qdd_out
    assert host(h, MODE_WORLD, 1, dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W), dp(qo), dp(qdo), None) == -2
    assert host(h, MODE_FULL, 1, dp(q), dp(qd), dp(act), 0, None, None, None, dp(qo), dp(qdo), None) == 0        # K = 0
    assert host(h, MODE_FD, 1, dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W), None, None, dp(qddo)) == 0
    rows, cols = sim.jacobian_dims(MODE_FULL, True)
    t_in, t_W, t_out = np.zeros((8, cols, 1)), np.zeros((8, 2, 6, 1)), np.zeros((8, rows, 1))
    jvp = lambda *a: L.tds_b200_step_wrench_jvp_host(*a)
    args = (dp(q), dp(qd), dp(act), 2, ip(lk), dp(lc), dp(W))
    assert jvp(h, MODE_WORLD, 1, *args, 1, dp(t_in), None, None, dp(t_out)) == -2
    assert jvp(h, MODE_FULL, 1, *args, 0, dp(t_in), None, None, dp(t_out)) == -1
    assert jvp(h, MODE_FULL, 1, *args, 1, None, None, None, dp(t_out)) == -1
    assert jvp(h, MODE_FULL, 1, *args, 1, dp(t_in), None, None, None) == -1
    assert jvp(h, MODE_FULL, 1, *args, 1, None, dp(t_W), dp(t_in), dp(t_out)) == -4
    assert jvp(h, MODE_FULL, 1, *args, 1, None, dp(t_W), None, dp(t_out)) == 0
    G, g_in, g_W = np.zeros((8, rows)), np.zeros((8, cols)), np.zeros((8, 2, 6))
    vjp = lambda *a: L.tds_b200_step_wrench_vjp_host(*a)
    assert vjp(h, MODE_WORLD, 1, *args, dp(G), dp(g_in), None, None) == -2
    assert vjp(h, MODE_FULL, 1, *args, None, dp(g_in), None, None) == -1
    assert vjp(h, MODE_FULL, 1, *args, dp(G), None, None, None) == -1
    assert vjp(h, MODE_FULL, 1, *args, dp(G), None, None, dp(g_in)) == -4
    assert vjp(h, MODE_FULL, 1, *args, dp(G), None, dp(g_W), None) == 0
    # PD without tds_b200_set_env: -3
    plain = tds_b200.BatchSim(sim.model, 8, precision=1)
    P, ph = plain._L, plain._h
    assert P.tds_b200_step_wrench_host(ph, MODE_FULL, 1, *args, dp(qo), dp(qdo), None) == -3
    assert P.tds_b200_step_wrench_jvp_host(ph, MODE_FULL, 1, *args, 1, dp(t_in), None, None, dp(t_out)) == -3
    assert P.tds_b200_step_wrench_vjp_host(ph, MODE_FULL, 1, *args, dp(G), dp(g_in), None, None) == -3
    # device entry points
    ns = sim.n_stride
    z = lambda rows, dt=torch.float32: torch.zeros((rows, ns), dtype=dt, device="cuda")
    qs, qds, acts, Wd = z(sim.n_q), z(sim.n_qd), z(12), z(12)
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dev = lambda mode, pd, a, K, lkp, w, qo_, qdo_, qddo_: L.tds_b200_step_wrench_device(h, mode, pd, vp(qs), vp(qds), vp(a), K, lkp, dp(lc),
                                                                                         vp(w), vp(qo_), vp(qdo_), vp(qddo_), st)
    assert dev(MODE_FULL, 1, acts, 2, ip(lk), None, qs, qds, None) == -1
    assert dev(MODE_FULL, 1, None, 2, ip(lk), Wd, qs, qds, None) == -1
    assert dev(MODE_FULL, 1, acts, 2, ip(bad), Wd, qs, qds, None) == -1
    assert dev(MODE_FULL, 1, acts, 2, ip(lk), Wd, None, qds, None) == -1
    assert dev(MODE_WORLD, 1, acts, 2, ip(lk), Wd, qs, qds, None) == -2
    assert dev(MODE_FULL, 1, acts, 2, ip(lk), Wd, qs, qds, None) == 0
    tid, tWd, tod = z(cols, torch.float64), z(12, torch.float64), z(rows, torch.float64)
    jd = lambda m, ti, tw, tp, to: L.tds_b200_step_wrench_jvp_device(h, MODE_FULL, 1, vp(qs), vp(qds), vp(acts), 2, ip(lk), dp(lc), vp(Wd), m,
                                                                     vp(ti), vp(tw), vp(tp), vp(to), st)
    assert jd(0, tid, None, None, tod) == -1
    assert jd(1, None, None, None, tod) == -1
    assert jd(1, None, tWd, tid, tod) == -4
    assert jd(1, tid, tWd, None, tod) == 0
    Gd, gid, gWd = z(rows, torch.float64), z(cols, torch.float64), z(12, torch.float64)
    vd = lambda g, gi, gw, gp: L.tds_b200_step_wrench_vjp_device(h, MODE_FULL, 1, vp(qs), vp(qds), vp(acts), 2, ip(lk), dp(lc), vp(Wd),
                                                                 vp(g), vp(gi), vp(gw), vp(gp), st)
    assert vd(None, gid, gWd, None) == -1
    assert vd(Gd, None, None, None) == -1
    assert vd(Gd, None, gWd, gid) == -4
    assert vd(Gd, gid, gWd, None) == 0
    torch.cuda.synchronize()
