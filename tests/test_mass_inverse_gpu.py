"""The inverse mass matrix and the operational-space inverse inertia on the H100 (DESIGN.md section 7.20): the MINV instances and the
contraction kernel as nvcc builds them, against the host build of the same source within B = 1e-13 kappa_2(M) max|ref|, on ragged and
chunked batches, around steps and installed parameters, through torch.autograd (backward, forward_ad, torch.func.jvp), every argument
check of the C-ABI, and contact-consistent dynamics of Laikago through Lambda^-1.  The CPU twins are in tests/test_mass_inverse_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from test_mass_inverse_on_host import ALL, kappa, points, within_b
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
    return q


@pytest.mark.parametrize("name", ALL)
def test_device_against_the_host_build(name):
    """Values and JVPs (q and parameter tangents) of the nvcc build against the host build within B."""
    import emu_mass
    import emu_mass_inverse as emi
    import emu_point_motion
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    lk, lc = points(model)
    kap = kappa(emu_mass.mass(model, q))
    sim = _sim(model, n)
    Mi, L = sim.mass_inverse_host(q, lk, lc)
    hMi = emi.mass_inverse(model, q)
    J = emu_point_motion.point_motion(model, q, lk, lc)[0].reshape(n, -1, nd)
    assert within_b(Mi, hMi, kap) and within_b(L, emi.osim(J, hMi), kap), name
    assert np.array_equal(Mi, Mi.transpose(0, 2, 1)) and np.array_equal(L, L.transpose(0, 2, 1))
    ids = all_ids(model)[:10]
    vals = perturbed(model, ids, n, 21, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(22)
    vq, vp = rng.normal(size=(n, n_q, 2)), rng.normal(size=(n, len(ids), 2))
    Mi2, L2, dMi, dL = sim.mass_inverse_jvp_host(q, lk, lc, vq, vp)
    hMi2 = emi.mass_inverse(model, q, ids=ids, values=vals)
    hdMi = emi.mass_inverse_jvp(model, q, vq, vp, ids=ids, values=vals)
    tin = np.concatenate([vq, np.zeros((n, 2 * nd, 2))], axis=1)
    dJ = emu_point_motion.point_motion_jvp(model, q, lk, lc, tin)[:, :J.shape[1] * nd].reshape(n, -1, nd, 2)
    assert within_b(Mi2, hMi2, kap) and within_b(dMi, hdMi, kap), name
    assert within_b(L2, emi.osim(J, hMi2), kap) and within_b(dL, emi.osim(J, hMi2, dJ, hdMi), kap), name


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    lk, lc = points(model)
    q = _q(model, 4096, 3)
    Mi, L = _sim(model, 4096).mass_inverse_host(q, lk, lc)
    for n in (1, 31, 33, 100):
        a, b = _sim(model, n).mass_inverse_host(q[-n:], lk, lc)
        assert np.array_equal(a, Mi[-n:]) and np.array_equal(b, L[-n:]), n


def test_humanoid_jvp_in_several_chunks_equals_one_chunk_and_vjp_is_its_adjoint():
    """A humanoid batch sized so that m = n_q tangents run in at least three launches of the chunk loop; <G, dOut[v]> = <VJP(G), v>."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    n_q = probe.n_q
    n = 32 * (probe.jacobian_chunk() * 3 // n_q + 1)
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    assert n_q >= 3 * chunk - 2, (chunk, n_q)
    q = _q(model, n, 5)
    lk, lc = points(model)
    V = np.random.default_rng(6).normal(size=(n, n_q, n_q))
    _, _, dMi, dL = sim.mass_inverse_jvp_host(q, lk, lc, V)
    for j0 in range(0, n_q, chunk):
        _, _, a, b = sim.mass_inverse_jvp_host(q, lk, lc, V[..., j0:j0 + chunk])
        assert np.array_equal(a, dMi[..., j0:j0 + chunk]) and np.array_equal(b, dL[..., j0:j0 + chunk]), j0
    rng = np.random.default_rng(7)
    GM, GL = rng.normal(size=dMi.shape[:3]), rng.normal(size=dL.shape[:3])
    g_q, _ = sim.mass_inverse_vjp_host(q, lk, lc, GM, GL)
    fwd = np.einsum("eij,eijm->em", GM, dMi) + np.einsum("eij,eijm->em", GL, dL)
    # (a JVP along v and the sum of identity-direction JVPs weighted by v differ by rounding amplified by kappa_2(M), as B allows)
    assert rel(fwd, np.einsum("ec,ecm->em", g_q, V)) <= max(1e-10, 1e-13 * kappa(sim.mass_matrix_host(q)))


def test_parameters_and_steps_around_calls():
    """Installed, changed and cleared parameter sets give the edited models' M^-1 bit for bit; the step is bit-identical around calls."""
    model, q = fixture("laikago")
    n = q.shape[0]
    lk, lc = points(model)
    sim = _sim(model, n)
    qd = f32(np.random.default_rng(2).normal(size=(n, int(model[4]))))
    before = sim.step_host(2, q, qd)
    ref = sim.mass_inverse_host(q, lk, lc)[0]
    ids = all_ids(model)
    for seed in (14, 15):
        vals = perturbed(model, ids, n, seed, 0.5, 0.0)
        sim.set_physical_params(ids, vals)
        Mi = sim.mass_inverse_host(q, lk, lc)[0]
        g_q, g_par = sim.mass_inverse_vjp_host(q, lk, lc, G_Minv=np.ones_like(Mi))
        assert g_par.shape == (n, len(ids)) and np.all(g_par[:, :2] == 0.0)   # friction and restitution do not enter
        for e in range(2):
            one = _sim(model, 1)
            one.set_physical_params(ids, vals[e:e + 1])
            assert np.array_equal(one.mass_inverse_host(q[e:e + 1])[0], Mi[e:e + 1])
    sim.set_physical_params(None)
    assert np.array_equal(sim.mass_inverse_host(q, lk, lc)[0], ref)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("name", ["humanoid", "laikago"])
def test_autograd_backward_and_forward_mode(name):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    q = f32(q)
    lk, lc = points(model)
    K = len(lk)
    sim = _sim(model, n)
    ids = all_ids(model)[:8]
    vals = perturbed(model, ids, n, 8, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    rng = np.random.default_rng(16)
    GM, GL = rng.normal(size=(n, nd, nd)), rng.normal(size=(n, 6 * K, 6 * K))
    qr, pr = cu(q).requires_grad_(True), cu(vals, torch.float64).requires_grad_(True)
    Mi, L = tds_b200.autograd.mass_inverse(sim, qr, lk, lc, params=pr)
    hM, hL = sim.mass_inverse_host(q, lk, lc)
    assert np.array_equal(Mi.detach().cpu().numpy(), hM) and np.array_equal(L.detach().cpu().numpy(), hL)
    ((Mi * cu(GM, torch.float64)).sum() + (L * cu(GL, torch.float64)).sum()).backward()
    g_q, g_par = sim.mass_inverse_vjp_host(q, lk, lc, GM, GL)
    assert qr.grad.dtype == torch.float32 and rel(qr.grad.cpu().numpy().astype(np.float64), f32(g_q)) <= 1e-12
    assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), g_par) <= 1e-12
    vq, vp = f32(rng.normal(size=q.shape)), rng.normal(size=vals.shape)
    _, _, wM, wL = sim.mass_inverse_jvp_host(q, lk, lc, vq, vp)
    with fwAD.dual_level():
        outs = tds_b200.autograd.mass_inverse(sim, fwAD.make_dual(cu(q), cu(vq)), lk, lc,
                                              params=fwAD.make_dual(cu(vals, torch.float64), cu(vp, torch.float64)))
        tans = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in outs]
    assert rel(tans[0], wM) <= 1e-12 and rel(tans[1], wL) <= 1e-12
    _, ft = torch.func.jvp(lambda a, p: tds_b200.autograd.mass_inverse(sim, a, lk, lc, params=p), (cu(q), cu(vals, torch.float64)),
                           (cu(vq), cu(vp, torch.float64)))
    assert rel(ft[0].cpu().numpy(), wM) <= 1e-12 and rel(ft[1].cpu().numpy(), wL) <= 1e-12
    # without points: Linv None, and a solve with M differentiates through b
    sim.set_physical_params(None)
    q1, b = cu(q).requires_grad_(True), torch.ones((n, nd, 1), dtype=torch.float64, device="cuda", requires_grad=True)
    Mi0, L0 = tds_b200.autograd.mass_inverse(sim, q1)
    assert L0 is None
    (Mi0 @ b).sum().backward()
    assert q1.grad is not None and b.grad is not None


def test_argument_checks():
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    qh = np.ascontiguousarray(q)
    lk, lc = np.array([0, 1], dtype=np.int32), np.zeros((2, 3))
    bad = np.array([0, 7], dtype=np.int32)
    Mi, Li = np.zeros((n, nd, nd)), np.zeros((n, 12, 12))
    tq, tp = np.zeros((n, n_q, 1)), np.zeros((n, 1, 1))
    GM, gq, gp = np.zeros((n, nd, nd)), np.zeros((n, n_q)), np.zeros((n, 1))
    N = None
    assert L.tds_b200_mass_inverse_host(h, dp(qh), 2, vp(lk), dp(lc), dp(Mi), dp(Li)) == 0
    assert L.tds_b200_mass_inverse_host(h, dp(qh), 0, N, N, dp(Mi), N) == 0
    for args in [(N, 2, vp(lk), dp(lc), dp(Mi), dp(Li)), (dp(qh), 2, vp(lk), dp(lc), N, N), (dp(qh), -1, vp(lk), dp(lc), dp(Mi), N),
                 (dp(qh), 17, vp(lk), dp(lc), dp(Mi), N), (dp(qh), 0, N, N, dp(Mi), dp(Li)), (dp(qh), 2, vp(bad), dp(lc), dp(Mi), N),
                 (dp(qh), 2, N, dp(lc), dp(Mi), N)]:
        assert L.tds_b200_mass_inverse_host(h, *args) == -1, args
    T = (dp(tq), N)
    assert L.tds_b200_mass_inverse_jvp_host(h, dp(qh), 2, vp(lk), dp(lc), 1, *T, N, N, dp(Mi), dp(Li)) == 0
    for args in [(0, *T, N, N, dp(Mi), N), (1, N, N, N, N, dp(Mi), N), (1, *T, N, N, N, N), (1, dp(tq), dp(tp), N, N, dp(Mi), N)]:
        assert L.tds_b200_mass_inverse_jvp_host(h, dp(qh), 2, vp(lk), dp(lc), *args) == (-4 if args[2] is not None else -1), args
    assert L.tds_b200_mass_inverse_jvp_host(h, dp(qh), 0, N, N, 1, *T, N, dp(Li), dp(Mi), N) == -1   # Linv with K = 0
    assert L.tds_b200_mass_inverse_vjp_host(h, dp(qh), 2, vp(lk), dp(lc), dp(GM), N, dp(gq), N) == 0
    assert L.tds_b200_mass_inverse_vjp_host(h, dp(qh), 2, vp(lk), dp(lc), N, N, dp(gq), N) == -1
    assert L.tds_b200_mass_inverse_vjp_host(h, dp(qh), 2, vp(lk), dp(lc), dp(GM), N, N, N) == -1
    assert L.tds_b200_mass_inverse_vjp_host(h, dp(qh), 2, vp(lk), dp(lc), dp(GM), N, dp(gq), dp(gp)) == -4
    assert L.tds_b200_mass_inverse_vjp_host(h, dp(qh), 0, N, N, dp(GM), dp(Li), dp(gq), N) == -1
    # the device entries run the same checks
    assert L.tds_b200_mass_inverse_device(h, N, 2, vp(lk), dp(lc), N, N, N) == -1
    assert L.tds_b200_mass_inverse_jvp_device(h, N, 2, vp(lk), dp(lc), 1, N, N, N, N, N, N, N) == -1
    assert L.tds_b200_mass_inverse_vjp_device(h, N, 2, vp(lk), dp(lc), N, N, N, N, N) == -1


def test_contact_consistent_dynamics_of_laikago_through_lambda():
    """4096 Laikago environments, the toes' linear rows of Lambda^-1_c: f = -(Lambda^-1_c)^-1 (J_c M^-1 (tau - h) + J_c' qd) and
    qdd = M^-1 (tau - h + J_c^T f) give toe accelerations below 1e-8 m/s^2 and agree with the KKT solution within 1e-9 relative."""
    import torch
    model, q0 = fixture("laikago")
    n, nd = 4096, int(model[4])
    sim = _sim(model, n)
    rng = np.random.default_rng(41)
    q = f32(q0[rng.integers(0, q0.shape[0], n)] + rng.uniform(-0.1, 0.1, size=(n, int(model[3]))))
    qd = f32(rng.normal(size=(n, nd)) * 0.5)
    tau = rng.normal(size=(n, nd)) * 5.0
    lc = np.zeros((4, 3))
    Mi, Lam = sim.mass_inverse_host(q, LAIKAGO_TOES, lc)
    M = sim.mass_matrix_host(q)
    h = sim.inverse_dynamics_host(q, qd)
    J, _, drift = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc)
    lin = np.concatenate([np.arange(6 * k + 3, 6 * k + 6) for k in range(4)])
    Jc, dc, Lc = J[:, :, 3:].reshape(n, 12, nd), drift[:, :, 3:].reshape(n, 12), Lam[:, lin][:, :, lin]
    r = tau - h
    f = -np.linalg.solve(Lc, (np.einsum("eij,ej->ei", Jc, np.einsum("eij,ej->ei", Mi, r)) + dc)[..., None])[..., 0]
    qdd = np.einsum("eij,ej->ei", Mi, r + np.einsum("eji,ej->ei", Jc, f))
    KKT = np.zeros((n, nd + 12, nd + 12))
    KKT[:, :nd, :nd], KKT[:, :nd, nd:], KKT[:, nd:, :nd] = M, -Jc.transpose(0, 2, 1), Jc
    rhs = np.concatenate([r, -dc], axis=1)
    kkt = torch.linalg.solve(torch.tensor(KKT, device="cuda"), torch.tensor(rhs, device="cuda")[..., None])[..., 0].cpu().numpy()[:, :nd]
    assert np.abs(qdd - kkt).max() <= 1e-9 * np.abs(kkt).max()
    hi = f32(qdd)
    _, _, acc = sim.point_motion_host(q, qd, LAIKAGO_TOES, lc, hi)
    _, _, dacc = sim.point_motion_jvp_host(q, qd, LAIKAGO_TOES, lc, hi, None, None, qdd - hi)
    toe = (acc + dacc)[:, :, 3:]
    assert np.abs(toe).max() < 1e-8
