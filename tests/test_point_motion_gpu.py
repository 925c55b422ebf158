"""Spatial point Jacobians, point velocities and accelerations on the H100 (DESIGN.md section 7.17): the MOT instances of the world-frame
kernel as nvcc builds them, against the host build of the same source, on ragged and chunked batches, around steps and installed
parameters, through torch.autograd (backward, forward_ad, torch.func.jvp), a rollout loss on Laikago's toes against chained VJPs,
contact-consistent dynamics at 4096 environments from M, h and this query, and every argument check of the C-ABI.  The CPU twins are in
tests/test_point_motion_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from test_mass_matrix_on_host import f32, fixture, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "pendulum5spherical",
            "humanoid_spherical", "mb_three_bodies"]
LAIKAGO_TOES = [9, 13, 17, 21]


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return q


def _state(model, n, seed=3):
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return f32(rng.normal(size=(n, nd)) * 0.7), f32(rng.normal(size=(n, nd)))


def _table(model, seed=0):
    """Two base points, and every link's origin and one offset point, at most 64 points."""
    rng = np.random.default_rng(seed)
    lk, lc = [-1, -1], [np.zeros(3), np.array([0.1, -0.05, 0.2])]
    for i in range(int(model[1])):
        lk += [i, i]
        lc += [np.zeros(3), rng.uniform(-0.2, 0.2, 3)]
    return np.array(lk[:64]), np.array(lc[:64])


def _concat(out):
    n = out[0].shape[0]
    return np.concatenate([o.reshape(n, -1) for o in out], axis=1)


@pytest.mark.parametrize("name", FIXTURES)
def test_device_against_the_host_build(name):
    import emu_point_motion as ep
    model, q = fixture(name)
    qd, qdd = _state(model, q.shape[0])
    lk, lc = _table(model)
    sim = _sim(model, q.shape[0])
    assert rel(_concat(sim.point_motion_host(q, qd, lk, lc, qdd)), ep.point_motion(model, q, lk, lc, qd, qdd, concat=True)) <= 1e-12
    assert rel(_concat(sim.point_motion_host(q, None, lk, lc)), ep.point_motion(model, q, lk, lc, concat=True)) <= 1e-12


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 4096, 3)
    qd, qdd = _state(model, 4096, 4)
    lk, lc = _table(model)
    full = _concat(_sim(model, 4096).point_motion_host(q, qd, lk, lc, qdd))
    for n in (1, 31, 33, 100):
        assert np.array_equal(_concat(_sim(model, n).point_motion_host(q[-n:], qd[-n:], lk, lc, qdd[-n:])), full[-n:]), n


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_point_motion as ep
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = _state(model, n)
    lk, lc = _table(model)
    sim = _sim(model, n)
    rng = np.random.default_rng(13)
    vin = rng.normal(size=(n, n_q + 2 * nd, 2))
    got = _concat([x.reshape(n, -1, 2) for x in sim.point_motion_jvp_host(q, qd, lk, lc, qdd, vin[:, :n_q], vin[:, n_q:n_q + nd],
                                                                            vin[:, n_q + nd:])])
    got = got.reshape(n, -1, 2)
    assert rel(got, ep.point_motion_jvp(model, q, lk, lc, vin, qd, qdd)) <= 1e-12
    r_J, r_v, _ = ep.rows(model, len(lk))
    G = rng.normal(size=(n, r_J + 2 * r_v))
    g = sim.point_motion_vjp_host(q, qd, lk, lc, qdd, G[:, :r_J], G[:, r_J:r_J + r_v], G[:, r_J + r_v:])
    h = ep.point_motion_vjp(model, q, lk, lc, G, qd, qdd)
    assert rel(np.concatenate(g, axis=1), h) <= 1e-12
    fwd, rev = np.einsum("er,er->e", G, got[..., 0]), np.einsum("ec,ec->e", h, vin[..., 0])
    assert rel(fwd, rev) <= 1e-10


def test_humanoid_jvp_in_several_chunks_equals_one_chunk():
    """A humanoid batch sized so that m = n_q + 2 n_qd tangents run in at least three launches of the chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_in = probe.n_q + 2 * probe.n_qd
    n = 32 * (probe.jacobian_chunk() * 3 // n_in + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    assert n_in >= 3 * chunk - 2, (chunk, n_in)
    q = _q(model, n, 5)
    qd, qdd = _state(model, n, 6)
    lk, lc = _table(model)
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    nq, nd = sim.n_q, sim.n_qd
    split = lambda W: (W[:, :nq], W[:, nq:nq + nd], W[:, nq + nd:])
    whole = sim.point_motion_jvp_host(q, qd, lk, lc, qdd, *split(V))
    for j0 in range(0, n_in, chunk):
        part = sim.point_motion_jvp_host(q, qd, lk, lc, qdd, *split(V[..., j0:j0 + chunk]))
        for a, b in zip(part, whole):
            assert np.array_equal(a, b[..., j0:j0 + chunk]), j0


def test_steps_unchanged_around_point_motion_calls_and_parameters_do_not_enter():
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, qdd = _state(model, n)
    lk, lc = _table(model)
    sim = _sim(model, n)
    before = sim.step_host(2, q, qd)
    ref = _concat(sim.point_motion_host(q, qd, lk, lc, qdd))
    ids = all_ids(model)
    sim.set_physical_params(ids, perturbed(model, ids, n, 14, 0.5, 0.0))
    assert np.array_equal(_concat(sim.point_motion_host(q, qd, lk, lc, qdd)), ref)
    sim.set_physical_params(None)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("name", ["humanoid", "laikago"])
def test_autograd_backward_and_forward_mode(name):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    q = f32(q)
    qd, qdd = _state(model, n)
    lk, lc = _table(model)
    sim = _sim(model, n)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    xs = [cu(q), cu(qd), cu(qdd)]
    K = len(lk)
    rng = np.random.default_rng(16)
    GJ, Gv, Ga = (rng.normal(size=s) for s in ((n, K, 6, nd), (n, K, 6), (n, K, 6)))
    xr = [x.clone().requires_grad_(True) for x in xs]
    outs = tds_b200.autograd.point_motion(sim, xr[0], xr[1], lk, lc, qdd=xr[2])
    assert all(o.dtype == torch.float64 for o in outs)
    for o, h in zip(outs, sim.point_motion_host(q, qd, lk, lc, qdd)):
        assert np.array_equal(o.detach().cpu().numpy(), h)
    sum(((o * cu(g, torch.float64)).sum() for o, g in zip(outs, (GJ, Gv, Ga)))).backward()
    ref = sim.point_motion_vjp_host(q, qd, lk, lc, qdd, GJ, Gv, Ga)
    for x, g in zip(xr, ref):
        assert x.grad.dtype == torch.float32 and rel(x.grad.cpu().numpy().astype(np.float64), f32(g)) <= 1e-12
    v = [f32(rng.normal(size=x.shape)) for x in (q, qd, qdd)]
    want = sim.point_motion_jvp_host(q, qd, lk, lc, qdd, *v)
    ts = [cu(x) for x in v]
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x, t) for x, t in zip(xs, ts)]
        tans = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in tds_b200.autograd.point_motion(sim, duals[0], duals[1], lk, lc,
                                                                                                   qdd=duals[2])]
    for a, b in zip(tans, want):
        assert rel(a, b) <= 1e-12
    _, ft = torch.func.jvp(lambda a, b, c: tds_b200.autograd.point_motion(sim, a, b, lk, lc, qdd=c), tuple(xs), tuple(ts))
    for a, b in zip(ft, want):
        assert rel(a.cpu().numpy(), b) <= 1e-12
    # qd and qdd None are zero, and get no gradient
    q1 = xs[0].clone().requires_grad_(True)
    J0, v0, a0 = tds_b200.autograd.point_motion(sim, q1, None, lk, lc)
    assert np.array_equal(a0.detach().cpu().numpy(), sim.point_motion_host(q, np.zeros_like(qd), lk, lc)[2])
    (J0.sum() + a0.sum()).backward()
    assert q1.grad is not None


def test_toe_loss_through_a_rollout_against_chained_vjps():
    """loss = <Wv, vel> + <Wa, acc> of Laikago's four toes (acc at qdd = 0: the drift J' qd) at the end of a 5-step rollout with PD
    (autograd.step, then autograd.point_motion); the same gradient by chaining the C-ABI's VJPs backwards at the float32 cotangents
    autograd hands over."""
    import torch
    import tds_b200.workloads as wl
    n, T = 256, 5
    sim = tds_b200.laikago_sim(n, precision=1)
    w = wl.laikago_perturbed(n, seed=31)
    rng = np.random.default_rng(32)
    cu = lambda x: torch.tensor(x, dtype=torch.float32, device="cuda", requires_grad=True)
    q0, qd0 = cu(w["q"]), cu(w["qd"])
    acts = [cu(rng.uniform(-0.3, 0.3, size=(n, 12))) for _ in range(T)]
    lc = np.zeros((4, 3))
    Wv, Wa = rng.normal(size=(n, 4, 6)), rng.normal(size=(n, 4, 6))
    q, qd, states = q0, qd0, []
    for t in range(T):
        states.append((q.detach().cpu().numpy(), qd.detach().cpu().numpy()))
        q, qd = tds_b200.autograd.step(sim, q, qd, acts[t], use_pd=True)
    _, vel, acc = tds_b200.autograd.point_motion(sim, q, qd, LAIKAGO_TOES, lc)
    ((vel * torch.tensor(Wv, device="cuda")).sum() + (acc * torch.tensor(Wa, device="cuda")).sum()).backward()
    qT, qdT = q.detach().cpu().numpy().astype(np.float64), qd.detach().cpu().numpy().astype(np.float64)
    g_q, g_qd, _ = sim.point_motion_vjp_host(qT, qdT, LAIKAGO_TOES, lc, None, None, Wv, Wa)
    gq, gqd = g_q.astype(np.float32), g_qd.astype(np.float32)
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


def test_contact_consistent_dynamics_of_laikago_at_4096_environments():
    """M (section 7.12), h = ID(q, qd, 0) (section 7.14) and the toes' J_c and J_c' qd from this query compose: the solution of
    [M -J_c^T; J_c 0] [qdd; f] = [tau - h; -J_c' qd] gives toe accelerations below 1e-8 m/s^2 at that qdd.  The value path rounds qdd to
    fp32, so the fp64 qdd enters as its fp32 rounding plus the remainder along the exact JVP (acc is linear in qdd)."""
    import torch
    model, q0 = fixture("laikago")
    n, nd = 4096, int(model[4])
    sim = _sim(model, n)
    rng = np.random.default_rng(41)
    q = f32(q0[rng.integers(0, q0.shape[0], n)] + rng.uniform(-0.1, 0.1, size=(n, int(model[3]))))
    qd = f32(rng.normal(size=(n, nd)) * 0.5)
    tau = rng.normal(size=(n, nd)) * 5.0
    lc = np.zeros((4, 3))
    M = sim.mass_matrix_host(q)
    h = sim.inverse_dynamics_host(q, qd)
    J, _, drift = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc)
    Jc, dc = J[:, :, 3:].reshape(n, 12, nd), drift[:, :, 3:].reshape(n, 12)
    KKT = np.zeros((n, nd + 12, nd + 12))
    KKT[:, :nd, :nd], KKT[:, :nd, nd:], KKT[:, nd:, :nd] = M, -Jc.transpose(0, 2, 1), Jc
    rhs = np.concatenate([tau - h, -dc], axis=1)
    sol = torch.linalg.solve(torch.tensor(KKT, device="cuda"), torch.tensor(rhs, device="cuda")[..., None])[..., 0].cpu().numpy()
    qdd = sol[:, :nd]
    hi = f32(qdd)
    _, _, acc = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc, hi)
    _, _, dacc = sim.point_motion_jvp_host(q, qd, LAIKAGO_TOES, lc, hi, None, None, qdd - hi)
    toe = (acc + dacc)[:, :, 3:]
    print(f"largest toe acceleration {np.abs(toe).max():.2e} m/s^2 (fp32 qdd alone: {np.abs(acc[:, :, 3:]).max():.2e})")
    assert np.abs(toe).max() < 1e-8


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    qh = np.ascontiguousarray(q)
    lk, lc = np.array([0, 1], dtype=np.int32), np.zeros((2, 3))
    bad = np.array([0, 2], dtype=np.int32)
    neg = np.array([-2, 0], dtype=np.int32)
    vel, t, to, G, g = np.zeros((n, 12)), np.zeros((n, n_q, 1)), np.zeros((n, 12, 1)), np.zeros((n, 12)), np.zeros((n, n_q))
    host = L.tds_b200_point_motion_host
    assert host(None, dp(qh), None, None, 2, vp(lk), dp(lc), None, dp(vel), None) == -1
    assert host(h, None, None, None, 2, vp(lk), dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, vp(lk), dp(lc), None, None, None) == -1
    assert host(h, dp(qh), None, None, -1, vp(lk), dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 65, vp(lk), dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, vp(bad), dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, vp(neg), dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, None, dp(lc), None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, vp(lk), None, None, dp(vel), None) == -1
    assert host(h, dp(qh), None, None, 2, vp(lk), dp(lc), None, dp(vel), None) == 0
    assert L.tds_b200_point_motion_device(h, None, None, None, 2, vp(lk), dp(lc), None, None, None, None) == -1
    jvp = L.tds_b200_point_motion_jvp_host
    assert jvp(h, dp(qh), None, None, 2, vp(lk), dp(lc), 0, dp(t), None, None, None, dp(to), None) == -1
    assert jvp(h, dp(qh), None, None, 2, vp(lk), dp(lc), 1, None, None, None, None, dp(to), None) == -1
    assert jvp(h, dp(qh), None, None, 2, vp(lk), dp(lc), 1, dp(t), None, None, None, None, None) == -1
    assert jvp(h, dp(qh), None, None, 2, vp(bad), dp(lc), 1, dp(t), None, None, None, dp(to), None) == -1
    assert jvp(h, None, None, None, 2, vp(lk), dp(lc), 1, dp(t), None, None, None, dp(to), None) == -1
    assert L.tds_b200_point_motion_jvp_device(h, None, None, None, 2, vp(lk), dp(lc), 1, None, None, None, None, None, None, None) == -1
    vjp = L.tds_b200_point_motion_vjp_host
    assert vjp(h, dp(qh), None, None, 2, vp(lk), dp(lc), None, dp(G), None, None, None, None) == -1
    assert vjp(h, dp(qh), None, None, 2, vp(lk), dp(lc), None, None, None, dp(g), None, None) == -1
    assert vjp(h, None, None, None, 2, vp(lk), dp(lc), None, dp(G), None, dp(g), None, None) == -1
    assert vjp(h, dp(qh), None, None, 66, vp(lk), dp(lc), None, dp(G), None, dp(g), None, None) == -1
    assert L.tds_b200_point_motion_vjp_device(h, None, None, None, 2, vp(lk), dp(lc), None, None, None, None, None, None, None) == -1
    # NULL qd and qdd are zero
    qd, qdd = _state(model, n)
    a = _concat(sim.point_motion_host(q, None, lk, lc))
    assert np.array_equal(a, _concat(sim.point_motion_host(q, np.zeros((n, nd)), lk, lc, np.zeros((n, nd)))))
    # the Python layer
    z32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        tds_b200.autograd.point_motion(sim, torch.zeros((n, 2), dtype=torch.float64, device="cuda"), None, lk, lc)
    with pytest.raises(ValueError):
        tds_b200.autograd.point_motion(sim, z32(n, 2), z32(n, 3), lk, lc)
    with pytest.raises(ValueError):
        tds_b200.autograd.point_motion(sim, z32(n, 2), None, lk, lc, qdd=z32(n, 3))
    with pytest.raises(ValueError):
        sim.point_motion_host(q, qd, [0, 1], np.zeros((3, 3)))
    with pytest.raises(ValueError):
        sim.point_motion_jvp_host(q, qd, lk, lc)
    with pytest.raises(ValueError):
        sim.point_motion_vjp_host(q, qd, lk, lc)
