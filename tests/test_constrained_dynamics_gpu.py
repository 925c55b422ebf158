"""The point-constrained forward dynamics on the H100 (DESIGN.md section 7.21): the C-ABI's composition of the INV, MINV and MOT launches
with the rows and solve kernels as nvcc builds them, against the host build of the same source within B = 1e-13 kappa_2(M) kappa_2(J_c M^-1
J_c^T) max|ref|, on ragged and chunked batches, around steps and installed parameters, through torch.autograd (backward, forward_ad,
torch.func.jvp), every argument check of the C-ABI, and contact-consistent Laikago dynamics at 4096 environments against the by-hand
path through Lambda^-1.  The CPU twins are in tests/test_constrained_dynamics_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from test_constrained_dynamics_on_host import ALL, full_rank_table, host_pieces, kkt, state, within
from test_mass_inverse_on_host import kappa
from test_mass_matrix_on_host import f32, fixture, rel
from test_params_on_host import all_ids, perturbed
from test_point_motion_gpu import LAIKAGO_TOES

pytestmark = pytest.mark.gpu


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return f32(q)


@pytest.mark.parametrize("name", ALL)
def test_device_against_the_host_build(name):
    """Values (K = 0 and a full-rank table) and JVPs along q, qd, tau and parameter tangents of the nvcc build against the host build
    within B."""
    import emu_constrained_dynamics as ecd
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, tau = state(model, n, 21)
    lk, lc = full_rank_table(model, q, 3)
    K = len(lk)
    M, h, J, d = host_pieces(model, q, qd, lk, lc)
    kM, kA = kappa(M), float(kkt(M, h, J, d, tau, K, 3)[2].max())
    sim = _sim(model, n)
    qdd0, f0 = sim.constrained_dynamics_host(q, qd, tau)
    assert f0 is None and within(qdd0, ecd.constrained_dynamics(model, q, qd, tau)[0], kM, 1.0), name
    qdd, f = sim.constrained_dynamics_host(q, qd, tau, lk, lc, 3)
    hq, hf = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3)
    assert within(qdd, hq, kM, kA) and (K == 0 or within(f, hf, kM, kA)), name
    ids = all_ids(model)[:10]
    vals = perturbed(model, ids, n, 22, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(23)
    V = [rng.normal(size=(n, dim, 2)) for dim in (n_q, nd, nd, len(ids))]
    qdd2, f2, dq, df = sim.constrained_dynamics_jvp_host(q, qd, tau, lk, lc, 3, 0.0, *V)
    hq2, hf2 = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3, ids=ids, values=vals)
    hdq, hdf = ecd.constrained_dynamics_jvp(model, q, qd, tau, lk, lc, 3, 0.0, *V, ids=ids, values=vals)
    assert within(qdd2, hq2, kM, kA) and within(dq, hdq, kM, kA), name
    if K:
        assert within(f2, hf2, kM, kA) and within(df, hdf, kM, kA), name


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, q0 = fixture(name)
    lk, lc = full_rank_table(model, q0, 3)
    q = _q(model, 4096, 3)
    qd, tau = state(model, 4096, 4)
    qdd, f = _sim(model, 4096).constrained_dynamics_host(q, qd, tau, lk, lc, 3, 1e-9)
    for n in (1, 31, 33, 100):
        a, b = _sim(model, n).constrained_dynamics_host(q[-n:], qd[-n:], tau[-n:], lk, lc, 3, 1e-9)
        assert np.array_equal(a, qdd[-n:]) and np.array_equal(b, f[-n:]), n


def test_humanoid_jvp_in_several_chunks_equals_one_call_and_vjp_is_its_adjoint():
    """A humanoid batch sized so that m = n_q + 2 n_qd tangents run in at least three launches of the chunk loop; <G, dOut[v]> =
    <VJP(G), v>."""
    model, q0 = fixture("humanoid")
    probe = _sim(model, 32)
    n_q, nd = probe.n_q, probe.n_qd
    n_in = n_q + 2 * nd
    n = 32 * (probe.jacobian_chunk() * 3 // n_in + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    assert n_in >= 3 * chunk - 2, (chunk, n_in)
    q = _q(model, n, 5)
    qd, tau = state(model, n, 6)
    lk, lc = full_rank_table(model, q0, 3)
    V = np.random.default_rng(7).normal(size=(n, n_in, n_in))
    split = lambda X: (X[:, :n_q], X[:, n_q:n_q + nd], X[:, n_q + nd:])
    _, _, dq, df = sim.constrained_dynamics_jvp_host(q, qd, tau, lk, lc, 3, 0.0, *split(V))
    for j0 in range(0, n_in, chunk):
        _, _, a, b = sim.constrained_dynamics_jvp_host(q, qd, tau, lk, lc, 3, 0.0, *split(V[..., j0:j0 + chunk]))
        assert np.array_equal(a, dq[..., j0:j0 + chunk]) and np.array_equal(b, df[..., j0:j0 + chunk]), j0
    rng = np.random.default_rng(8)
    Gq, Gf = rng.normal(size=dq.shape[:2]), rng.normal(size=df.shape[:3])
    g_q, g_qd, g_tau, _ = sim.constrained_dynamics_vjp_host(q, qd, tau, lk, lc, 3, 0.0, Gq, Gf)
    fwd = np.einsum("ei,eim->em", Gq, dq) + np.einsum("ekd,ekdm->em", Gf, df)
    back = np.einsum("ec,ecm->em", np.concatenate([g_q, g_qd, g_tau], axis=1), V)
    M, h, J, d = host_pieces(model, q[:64], qd[:64], lk, lc)
    bound = 1e-13 * kappa(M) * float(kkt(M, h, J, d, tau[:64], len(lk), 3)[2].max())
    assert rel(fwd, back) <= max(1e-10, bound), (rel(fwd, back), bound)


def test_parameters_and_steps_around_calls():
    """Installed, changed and cleared parameter sets give the edited models' outputs bit for bit; the step is bit-identical around calls."""
    model, q = fixture("laikago")
    n = q.shape[0]
    lk, lc = LAIKAGO_TOES, np.zeros((4, 3))
    sim = _sim(model, n)
    qd, tau = state(model, n, 9)
    before = sim.step_host(2, q, qd)
    ref = sim.constrained_dynamics_host(q, qd, tau, lk, lc, 3)
    ids = all_ids(model)
    for seed in (14, 15):
        vals = perturbed(model, ids, n, seed, 0.5, 0.0)
        sim.set_physical_params(ids, vals)
        qdd, f = sim.constrained_dynamics_host(q, qd, tau, lk, lc, 3)
        g = sim.constrained_dynamics_vjp_host(q, qd, tau, lk, lc, 3, 0.0, G_qdd=np.ones_like(qdd))
        assert g[3].shape == (n, len(ids)) and np.all(g[3][:, :2] == 0.0)   # friction and restitution do not enter
        for e in range(2):
            one = _sim(model, 1)
            one.set_physical_params(ids, vals[e:e + 1])
            a, b = one.constrained_dynamics_host(q[e:e + 1], qd[e:e + 1], tau[e:e + 1], lk, lc, 3)
            assert np.array_equal(a, qdd[e:e + 1]) and np.array_equal(b, f[e:e + 1])
    sim.set_physical_params(None)
    again = sim.constrained_dynamics_host(q, qd, tau, lk, lc, 3)
    assert np.array_equal(again[0], ref[0]) and np.array_equal(again[1], ref[1])
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("name", ["humanoid", "laikago"])
def test_autograd_backward_and_forward_mode(name):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    q = f32(q)
    lk, lc = full_rank_table(model, q, 3)
    K = len(lk)
    qd, tau = state(model, n, 16)
    sim = _sim(model, n)
    ids = all_ids(model)[:8]
    vals = perturbed(model, ids, n, 8, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    rng = np.random.default_rng(17)
    Gq, Gf = rng.normal(size=(n, nd)), rng.normal(size=(n, K, 3))
    qr, qdr, tr, pr = (cu(q).requires_grad_(True), cu(qd).requires_grad_(True), cu(tau).requires_grad_(True),
                       cu(vals, torch.float64).requires_grad_(True))
    qdd, f = tds_b200.autograd.constrained_dynamics(sim, qr, qdr, tr, lk, lc, 3, 0.0, params=pr)
    hq, hf = sim.constrained_dynamics_host(q, qd, tau, lk, lc, 3)
    assert np.array_equal(qdd.detach().cpu().numpy(), hq) and np.array_equal(f.detach().cpu().numpy(), hf)
    ((qdd * cu(Gq, torch.float64)).sum() + (f * cu(Gf, torch.float64)).sum()).backward()
    g_q, g_qd, g_tau, g_par = sim.constrained_dynamics_vjp_host(q, qd, tau, lk, lc, 3, 0.0, Gq, Gf)
    for t, ref in ((qr, g_q), (qdr, g_qd), (tr, g_tau)):
        assert t.grad.dtype == torch.float32 and rel(t.grad.cpu().numpy().astype(np.float64), f32(ref)) <= 1e-12
    assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), g_par) <= 1e-12
    vq, vqd, vt, vp = f32(rng.normal(size=q.shape)), f32(rng.normal(size=qd.shape)), f32(rng.normal(size=tau.shape)), rng.normal(size=vals.shape)
    _, _, wq, wf = sim.constrained_dynamics_jvp_host(q, qd, tau, lk, lc, 3, 0.0, vq, vqd, vt, vp)
    with fwAD.dual_level():
        outs = tds_b200.autograd.constrained_dynamics(sim, fwAD.make_dual(cu(q), cu(vq)), fwAD.make_dual(cu(qd), cu(vqd)),
                                                      fwAD.make_dual(cu(tau), cu(vt)), lk, lc, 3, 0.0,
                                                      params=fwAD.make_dual(cu(vals, torch.float64), cu(vp, torch.float64)))
        tans = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in outs]
    assert rel(tans[0], wq) <= 1e-12 and rel(tans[1], wf) <= 1e-12
    _, ft = torch.func.jvp(lambda a, b, c, p: tds_b200.autograd.constrained_dynamics(sim, a, b, c, lk, lc, 3, 0.0, params=p),
                           (cu(q), cu(qd), cu(tau), cu(vals, torch.float64)), (cu(vq), cu(vqd), cu(vt), cu(vp, torch.float64)))
    assert rel(ft[0].cpu().numpy(), wq) <= 1e-12 and rel(ft[1].cpu().numpy(), wf) <= 1e-12
    # without points: f None, the unconstrained forward dynamics
    sim.set_physical_params(None)
    q1 = cu(q).requires_grad_(True)
    qdd0, f0 = tds_b200.autograd.constrained_dynamics(sim, q1, None, cu(tau))
    assert f0 is None
    qdd0.sum().backward()
    assert q1.grad is not None


def test_argument_checks():
    L = tds_b200.lib()
    model, q = fixture("laikago")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    qh = np.ascontiguousarray(q)
    lk, lc = np.array(LAIKAGO_TOES, dtype=np.int32), np.zeros((4, 3))
    bad = np.array([9, 13, 17, 99], dtype=np.int32)
    qdd, f = np.zeros((n, nd)), np.zeros((n, 12))
    tq, tp, tqdd, tf = np.zeros((n, n_q, 1)), np.zeros((n, 1, 1)), np.zeros((n, nd, 1)), np.zeros((n, 12, 1))
    Gq, gq, gp = np.zeros((n, nd)), np.zeros((n, n_q)), np.zeros((n, 1))
    N = None
    T = (vp(lk), dp(lc))
    assert L.tds_b200_constrained_dynamics_host(h, dp(qh), N, N, 4, *T, 3, 0.0, dp(qdd), dp(f)) == 0
    assert L.tds_b200_constrained_dynamics_host(h, dp(qh), N, N, 0, N, N, 3, 0.0, dp(qdd), N) == 0
    for args in [(N, 4, *T, 3, 0.0, dp(qdd), N), (dp(qh), 4, *T, 3, 0.0, N, N), (dp(qh), -1, *T, 3, 0.0, dp(qdd), N),
                 (dp(qh), 17, *T, 3, 0.0, dp(qdd), N), (dp(qh), 4, *T, 4, 0.0, dp(qdd), N), (dp(qh), 4, *T, 3, -1.0, dp(qdd), N),
                 (dp(qh), 4, *T, 3, float("inf"), dp(qdd), N), (dp(qh), 4, *T, 3, float("nan"), dp(qdd), N),
                 (dp(qh), 0, N, N, 3, 0.0, dp(qdd), dp(f)), (dp(qh), 4, vp(bad), dp(lc), 3, 0.0, dp(qdd), N),
                 (dp(qh), 4, N, dp(lc), 3, 0.0, dp(qdd), N)]:
        assert L.tds_b200_constrained_dynamics_host(h, args[0], N, N, *args[1:]) == -1, args
    J = lambda *a: L.tds_b200_constrained_dynamics_jvp_host(h, dp(qh), N, N, *a)
    assert J(4, *T, 3, 0.0, 1, dp(tq), N, N, N, N, N, dp(tqdd), dp(tf)) == 0
    assert J(4, *T, 3, 0.0, 0, dp(tq), N, N, N, N, N, dp(tqdd), N) == -1
    assert J(4, *T, 3, 0.0, 1, N, N, N, N, N, N, dp(tqdd), N) == -1
    assert J(4, *T, 3, 0.0, 1, dp(tq), N, N, N, N, N, N, N) == -1
    assert J(4, *T, 3, 0.0, 1, dp(tq), N, N, dp(tp), N, N, dp(tqdd), N) == -4
    assert J(0, N, N, 3, 0.0, 1, dp(tq), N, N, N, N, N, dp(tqdd), dp(tf)) == -1   # t_f with K = 0
    assert J(0, N, N, 3, 0.0, 1, dp(tq), N, N, N, N, dp(f), dp(tqdd), N) == -1    # f with K = 0
    V = lambda *a: L.tds_b200_constrained_dynamics_vjp_host(h, dp(qh), N, N, *a)
    assert V(4, *T, 3, 0.0, dp(Gq), N, dp(gq), N, N, N) == 0
    assert V(4, *T, 3, 0.0, N, N, dp(gq), N, N, N) == -1
    assert V(4, *T, 3, 0.0, dp(Gq), N, N, N, N, N) == -1
    assert V(4, *T, 3, 0.0, dp(Gq), N, dp(gq), N, N, dp(gp)) == -4
    assert V(0, N, N, 3, 0.0, dp(Gq), dp(f), dp(gq), N, N, N) == -1
    # the device entries run the same checks
    assert L.tds_b200_constrained_dynamics_device(h, N, N, N, 4, *T, 3, 0.0, N, N, N) == -1
    assert L.tds_b200_constrained_dynamics_jvp_device(h, N, N, N, 4, *T, 3, 0.0, 1, N, N, N, N, N, N, N, N, N) == -1
    assert L.tds_b200_constrained_dynamics_vjp_device(h, N, N, N, 4, *T, 3, 0.0, N, N, N, N, N, N, N) == -1


def test_contact_consistent_dynamics_of_laikago_at_4096_environments():
    """4096 Laikago environments, toes at dims 3: qdd and f match the by-hand path through Lambda^-1 (inverse_dynamics, mass_inverse,
    point_motion and a batched solve) within 1e-9 relative, and the toe accelerations J_c qdd + d_c stay below 1e-8 m/s^2."""
    model, q0 = fixture("laikago")
    n, nd = 4096, int(model[4])
    sim = _sim(model, n)
    rng = np.random.default_rng(41)
    q = f32(q0[rng.integers(0, q0.shape[0], n)] + rng.uniform(-0.1, 0.1, size=(n, int(model[3]))))
    qd = f32(rng.normal(size=(n, nd)) * 0.5)
    tau = f32(rng.normal(size=(n, nd)) * 5.0)
    lc = np.zeros((4, 3))
    qdd, f = sim.constrained_dynamics_host(q, qd, tau, LAIKAGO_TOES, lc, 3)
    Mi, Lam = sim.mass_inverse_host(q, LAIKAGO_TOES, lc)
    h = sim.inverse_dynamics_host(q, qd)
    J, _, drift = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc)
    lin = np.concatenate([np.arange(6 * k + 3, 6 * k + 6) for k in range(4)])
    Jc, dc, Lc = J[:, :, 3:].reshape(n, 12, nd), drift[:, :, 3:].reshape(n, 12), Lam[:, lin][:, :, lin]
    r = tau - h
    fh = -np.linalg.solve(Lc, (np.einsum("eij,ej->ei", Jc, np.einsum("eij,ej->ei", Mi, r)) + dc)[..., None])[..., 0]
    qh = np.einsum("eij,ej->ei", Mi, r + np.einsum("eji,ej->ei", Jc, fh))
    assert np.abs(qdd - qh).max() <= 1e-9 * np.abs(qh).max() and np.abs(f.reshape(n, 12) - fh).max() <= 1e-9 * np.abs(fh).max()
    hi = f32(qdd)
    _, _, acc = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc, hi)
    _, _, dacc = sim.point_motion_jvp_host(q, qd, LAIKAGO_TOES, lc, hi, None, None, qdd - hi)
    assert np.abs((acc + dacc)[:, :, 3:]).max() < 1e-8
