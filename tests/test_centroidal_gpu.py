"""The centroidal query on the H100 (DESIGN.md section 7.16): the CEN instances of the world-frame kernel as nvcc builds them, against the
host build of the same source, on ragged and chunked batches, with installed parameters, around steps, through torch.autograd (backward,
forward_ad, torch.func.jvp), a rollout loss on c and h_G against chained VJPs, a CoM Gauss-Newton at 4096 environments, and every
argument check of the C-ABI.  The CPU twins are in
tests/test_centroidal_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from tds_b200.model import param_names, set_param_values
from test_mass_matrix_on_host import f32, fixture, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "pendulum5spherical",
            "humanoid_spherical"]


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return q


def _qd(model, n, seed=3):
    return f32(np.random.default_rng(seed).normal(size=(n, int(model[4]))) * 0.7)


def _mass_ids(model):
    """The installable ids that enter the query: masses, centres of mass and inertias."""
    names = param_names(model)
    return [i for i in all_ids(model) if names[i].split(".")[-1] not in ("friction", "restitution", "stiffness", "damping")]


def _concat(out):
    m, c, I, A, b = out
    n = m.shape[0]
    return np.concatenate([m[:, None], c, I.reshape(n, 9)[:, [0, 1, 2, 4, 5, 8]], A.reshape(n, -1), b], axis=1)


@pytest.mark.parametrize("name", FIXTURES)
def test_device_against_the_host_build(name):
    import emu_centroidal as ec
    model, q = fixture(name)
    qd = _qd(model, q.shape[0])
    sim = _sim(model, q.shape[0])
    assert rel(_concat(sim.centroidal_host(q, qd)), ec.centroidal(model, q, qd, concat=True)) <= 1e-12
    assert rel(_concat(sim.centroidal_host(q)), ec.centroidal(model, q, concat=True)) <= 1e-12


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 4096, 3)
    qd = _qd(model, 4096, 4)
    full = _concat(_sim(model, 4096).centroidal_host(q, qd))
    for n in (1, 31, 33, 100):
        assert np.array_equal(_concat(_sim(model, n).centroidal_host(q[-n:], qd[-n:])), full[-n:]), n


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_centroidal as ec
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd = _qd(model, n)
    sim = _sim(model, n)
    ids = _mass_ids(model)
    vals = perturbed(model, ids, n, 12, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(13)
    vin, vp = rng.normal(size=(n, n_q + nd, 2)), rng.normal(size=(n, len(ids), 2))
    dcom, dA, db = sim.centroidal_jvp_host(q, qd, vin[:, :n_q], vin[:, n_q:], vp)
    got = np.concatenate([dcom, dA.reshape(n, 6 * nd, 2), db], axis=1)
    assert rel(got, ec.centroidal_jvp(model, q, qd, vin, vp, ids=ids, values=vals)) <= 1e-12
    G = rng.normal(size=(n, ec.rows(model)))
    g_q, g_qd, g_par = sim.centroidal_vjp_host(q, qd, G[:, :10], G[:, 10:10 + 6 * nd].reshape(n, 6, nd), G[:, 10 + 6 * nd:])
    h_in, h_par = ec.centroidal_vjp(model, q, qd, G, ids=ids, values=vals)
    assert rel(np.concatenate([g_q, g_qd], axis=1), h_in) <= 1e-12 and rel(g_par, h_par) <= 1e-12
    fwd = np.einsum("er,er->e", G, got[..., 0])
    rev = np.einsum("ec,ec->e", h_in, vin[..., 0]) + np.einsum("ek,ek->e", h_par, vp[..., 0])
    assert rel(fwd, rev) <= 1e-10


def test_humanoid_jvp_in_several_chunks_equals_one_chunk():
    """A humanoid batch sized so that m = n_q + n_qd tangents run in at least three launches of the chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_in = probe.n_q + probe.n_qd
    n = 32 * (probe.jacobian_chunk() * 3 // n_in + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    assert n_in >= 3 * chunk - 2, (chunk, n_in)
    q, qd = _q(model, n, 5), _qd(model, n, 6)
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    whole = sim.centroidal_jvp_host(q, qd, V[:, :sim.n_q], V[:, sim.n_q:])
    for j0 in range(0, n_in, chunk):
        part = sim.centroidal_jvp_host(q, qd, V[:, :sim.n_q, j0:j0 + chunk], V[:, sim.n_q:, j0:j0 + chunk])
        for a, b in zip(part, whole):
            assert np.array_equal(a, b[..., j0:j0 + chunk]), j0


def test_steps_unchanged_around_centroidal_calls_and_irrelevant_parameters():
    model, q = fixture("laikago")
    n = q.shape[0]
    qd = _qd(model, n)
    sim = _sim(model, n)
    before = sim.step_host(2, q, qd)
    c0 = _concat(sim.centroidal_host(q, qd))
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm in ("friction", "restitution") or nm.endswith((".stiffness", ".damping"))]
    sim.set_physical_params(ids, perturbed(model, ids, n, 14, 0.5, 0.0))
    assert np.array_equal(_concat(sim.centroidal_host(q, qd)), c0)
    ids = _mass_ids(model)
    vals = perturbed(model, ids, n, 15, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    c1 = _concat(sim.centroidal_host(q, qd))
    for e in range(n):
        ref = _concat(_sim(set_param_values(model, ids, vals[e]), 1).centroidal_host(q[e:e + 1], qd[e:e + 1]))
        assert rel(c1[e:e + 1], ref) <= 1e-12
    sim.set_physical_params(None)
    assert np.array_equal(_concat(sim.centroidal_host(q, qd)), c0)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_and_forward_mode(with_params):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture("humanoid")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    q = f32(q)
    qd = _qd(model, n)
    sim = _sim(model, n)
    ids = _mass_ids(model)[:20] if with_params else []
    vals = perturbed(model, ids, n, 15, 0.5, 0.0) if with_params else None
    if with_params:
        sim.set_physical_params(ids, vals)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    xs = [cu(q), cu(qd)]
    pt = cu(vals, torch.float64) if with_params else None
    rng = np.random.default_rng(16)
    Gm, Gc, GI, GA, Gb = (rng.normal(size=s) for s in ((n,), (n, 3), (n, 3, 3), (n, 6, nd), (n, 6)))
    xr = [x.clone().requires_grad_(True) for x in xs]
    pr = pt.clone().requires_grad_(True) if with_params else None
    outs = tds_b200.autograd.centroidal(sim, *xr, params=pr)
    assert all(o.dtype == torch.float64 for o in outs)
    host = sim.centroidal_host(q, qd)
    for o, h in zip(outs, host):
        assert np.array_equal(o.detach().cpu().numpy(), h)
    sum(((o * cu(g, torch.float64)).sum() for o, g in zip(outs, (Gm, Gc, GI, GA, Gb)))).backward()
    Gcom = np.concatenate([Gm[:, None], Gc, (GI + GI.transpose(0, 2, 1)).reshape(n, 9)[:, [0, 1, 2, 4, 5, 8]]], axis=1)
    Gcom[:, [4, 7, 9]] *= 0.5   # the diagonal is read once
    ref = sim.centroidal_vjp_host(q, qd, Gcom, GA, Gb)
    for x, g in zip(xr, ref[:2]):
        assert x.grad.dtype == torch.float32 and rel(x.grad.cpu().numpy().astype(np.float64), f32(g)) <= 1e-12
    if with_params:
        assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), ref[2]) <= 1e-12
    v = [f32(rng.normal(size=x.shape)) for x in (q, qd)]
    vp = rng.normal(size=(n, len(ids))) if with_params else None
    dcom, dA, db = sim.centroidal_jvp_host(q, qd, *v, vp)
    want = [dcom[:, 0], dcom[:, 1:4], dcom[:, 4:10][:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(n, 3, 3), dA, db]
    ts = [cu(x) for x in v]
    tp = cu(vp, torch.float64) if with_params else None
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x, t) for x, t in zip(xs, ts)]
        dp = fwAD.make_dual(pt, tp) if with_params else None
        tans = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in tds_b200.autograd.centroidal(sim, *duals, params=dp)]
    for a, b in zip(tans, want):
        assert rel(a, b) <= 1e-12
    if with_params:
        _, ft = torch.func.jvp(lambda a, b, c: tds_b200.autograd.centroidal(sim, a, b, c), (*xs, pt), (*ts, tp))
    else:
        _, ft = torch.func.jvp(lambda a, b: tds_b200.autograd.centroidal(sim, a, b), tuple(xs), tuple(ts))
    for a, b in zip(ft, want):
        assert rel(a.cpu().numpy(), b) <= 1e-12


def test_gauss_newton_moves_laikago_com_at_4096_environments():
    """4096 Laikago poses (the fixture's, leg joints perturbed by up to 0.1 rad) each move their CoM 2 cm along x with damped Gauss-Newton
    on the leg joints, A[3:6] / m as the CoM Jacobian and the six base coordinates held, within 5 iterations to 1e-6 m."""
    model, q0 = fixture("laikago")
    n, nd = 4096, int(model[4])
    sim = _sim(model, n)
    rng = np.random.default_rng(17)
    x = f32(q0[rng.integers(0, q0.shape[0], n)] + rng.uniform(-0.1, 0.1, size=(n, int(model[3]))))
    x[:, :6] = f32(q0[0, :6])
    target = sim.centroidal_host(x)[1] + np.array([0.02, 0.0, 0.0])
    legs = np.arange(6, nd)
    for _ in range(5):
        m, c, _, A, _ = sim.centroidal_host(x)
        r = target - c
        J = A[:, 3:][:, :, legs] / m[:, None, None]
        dx = np.einsum("erc,er->ec", J, np.linalg.solve(J @ J.transpose(0, 2, 1) + 1e-12 * np.eye(3), r[..., None])[..., 0])
        x[:, legs] = f32(x[:, legs] + dx)
    err = np.linalg.norm(target - sim.centroidal_host(x)[1], axis=1)
    assert err.max() < 1e-6, err.max()


def test_com_and_momentum_loss_through_a_rollout_against_chained_vjps():
    """loss = <Wc, c> + <Wh, h_G> with h_G = A qd at the end of a 5-step Laikago rollout with PD (autograd.step, then
    autograd.centroidal); the same gradient by chaining the C-ABI's VJPs backwards at the float32 cotangents autograd hands over."""
    import torch
    import tds_b200.workloads as wl
    n, T = 256, 5
    sim = tds_b200.laikago_sim(n, precision=1)
    w = wl.laikago_perturbed(n, seed=31)
    rng = np.random.default_rng(32)
    cu = lambda x: torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    q0, qd0 = cu(w["q"]), cu(w["qd"])
    acts = [cu(rng.uniform(-0.3, 0.3, size=(n, 12))) for _ in range(T)]
    Wc, Wh = rng.normal(size=(n, 3)), rng.normal(size=(n, 6))
    q, qd, states = q0, qd0, []
    for t in range(T):
        states.append((q.detach().cpu().numpy(), qd.detach().cpu().numpy()))
        q, qd = tds_b200.autograd.step(sim, q, qd, acts[t], use_pd=True)
    _, c, _, A, _ = tds_b200.autograd.centroidal(sim, q, qd)
    Wct, Wht = (torch.tensor(x, device="cuda") for x in (Wc, Wh))
    ((c * Wct).sum() + (torch.einsum("erc,ec->er", A, qd.double()) * Wht).sum()).backward()
    # by hand: the centroidal VJP at the final state (G_c = Wc, G_A = Wh qd^T) plus h_G's own qd term A^T Wh, then the step VJPs
    qT, qdT = q.detach().cpu().numpy().astype(np.float64), qd.detach().cpu().numpy().astype(np.float64)
    AT = sim.centroidal_host(qT, qdT)[3]
    G_com = np.zeros((n, 10))
    G_com[:, 1:4] = Wc
    g_q, g_qd, _ = sim.centroidal_vjp_host(qT, qdT, G_com, Wh[:, :, None] * qdT[:, None, :], None)
    gq = g_q.astype(np.float32)
    gqd = g_qd.astype(np.float32) + np.einsum("erc,er->ec", AT, Wh).astype(np.float32)
    nq, nd = sim.n_q, sim.n_qd
    g_act = [None] * T
    for t in reversed(range(T)):
        qs, qds = states[t]
        G = np.concatenate([gq, gqd], axis=1).astype(np.float64)
        g_in = sim.step_vjp_host(tds_b200.MODE_FULL, qs, qds, acts[t].detach().cpu().numpy(), G, use_pd=True)
        gq, gqd = g_in[:, :nq].astype(np.float32), g_in[:, nq:nq + nd].astype(np.float32)
        g_act[t] = g_in[:, nq + nd:nq + nd + 12].astype(np.float32)
    assert rel(q0.grad.cpu().numpy().astype(np.float64), gq.astype(np.float64)) <= 1e-6
    assert rel(qd0.grad.cpu().numpy().astype(np.float64), gqd.astype(np.float64)) <= 1e-6
    for t in range(T):
        assert rel(acts[t].grad.cpu().numpy().astype(np.float64), g_act[t].astype(np.float64)) <= 1e-6, t


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n, nd = q.shape[0], int(model[4])
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    qh, com, t, to, G, g = np.ascontiguousarray(q), np.zeros((n, 10)), np.zeros((n, 2, 1)), np.zeros((n, 10, 1)), np.zeros((n, 10)), np.zeros((n, 2))
    assert L.tds_b200_centroidal_host(None, dp(qh), None, dp(com), None, None) == -1
    assert L.tds_b200_centroidal_host(h, None, None, dp(com), None, None) == -1
    assert L.tds_b200_centroidal_host(h, dp(qh), None, None, None, None) == -1
    assert L.tds_b200_centroidal_device(h, None, None, None, None, None, None) == -1
    assert L.tds_b200_centroidal_jvp_host(h, dp(qh), None, 0, dp(t), None, None, dp(to), None, None) == -1
    assert L.tds_b200_centroidal_jvp_host(h, dp(qh), None, 1, None, None, None, dp(to), None, None) == -1
    assert L.tds_b200_centroidal_jvp_host(h, dp(qh), None, 1, dp(t), None, None, None, None, None) == -1
    assert L.tds_b200_centroidal_jvp_host(h, dp(qh), None, 1, None, None, dp(t), dp(to), None, None) == -4
    assert L.tds_b200_centroidal_jvp_device(h, None, None, 1, None, None, None, None, None, None, None) == -1
    assert L.tds_b200_centroidal_vjp_host(h, dp(qh), None, dp(G), None, None, None, None, None) == -1
    assert L.tds_b200_centroidal_vjp_host(h, dp(qh), None, None, None, None, dp(g), None, None) == -1
    assert L.tds_b200_centroidal_vjp_host(h, None, None, dp(G), None, None, dp(g), None, None) == -1
    assert L.tds_b200_centroidal_vjp_host(h, dp(qh), None, dp(G), None, None, None, None, dp(g)) == -4
    assert L.tds_b200_centroidal_vjp_device(h, None, None, None, None, None, None, None, None, None) == -1
    # refused models: several multibodies, no mass
    mb, qm = fixture("mb_three_bodies")
    s2 = _sim(mb, qm.shape[0])
    assert L.tds_b200_centroidal_host(s2._h, dp(np.ascontiguousarray(qm)), None, dp(np.zeros((qm.shape[0], 10))), None, None) == -2
    assert L.tds_b200_centroidal_jvp_host(s2._h, dp(np.ascontiguousarray(qm)), None, 1, dp(np.zeros((qm.shape[0], int(mb[3]), 1))), None,
                                          None, dp(np.zeros((qm.shape[0], 10, 1))), None, None) == -2
    names = param_names(model)
    massless = set_param_values(model, [names.index(f"link{i}.mass") for i in range(int(model[1]))], [0.0] * int(model[1]))
    s3 = _sim(massless, n)
    assert L.tds_b200_centroidal_host(s3._h, dp(qh), None, dp(com), None, None) == -2
    assert L.tds_b200_centroidal_vjp_host(s3._h, dp(qh), None, dp(G), None, None, dp(g), None, None) == -2
    # a NULL qd is zero
    assert np.array_equal(_concat(sim.centroidal_host(q)), _concat(sim.centroidal_host(q, np.zeros((n, nd)))))
    # the Python layer
    z32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        tds_b200.autograd.centroidal(sim, torch.zeros((n, 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        tds_b200.autograd.centroidal(sim, z32(n, 2), z32(n, 3))
    with pytest.raises(ValueError):
        tds_b200.autograd.centroidal(sim, z32(n, 2), None, torch.zeros((n, 1), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        sim.centroidal_jvp_host(q)
    with pytest.raises(ValueError):
        sim.centroidal_vjp_host(q)
