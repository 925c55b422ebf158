"""Joint-torque and energy regressors on the H100 (DESIGN.md section 7.19): the REG instances of the world-frame kernel as nvcc builds them,
against the host build of the same source, on ragged and chunked batches, around steps and installed parameters, through torch.autograd
(backward, forward_ad, torch.func.jvp), every argument check of the C-ABI, and identification end to end: Laikago's parameters recovered
by one batched least-squares solve.  The CPU twins are in tests/test_regressor_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from tds_b200.model import inertial_parameters, param_names
from test_mass_matrix_on_host import f32, fixture, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "humanoid_fixed",
            "pendulum5spherical", "humanoid_spherical", "mb_three_bodies", "mb_racket"]


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


def _concat(out):
    n = out[0].shape[0]
    return np.concatenate([o.reshape(n, -1) for o in out], axis=1)


@pytest.mark.parametrize("name", FIXTURES)
def test_device_against_the_host_build(name):
    import emu_regressor as er
    model, q = fixture(name)
    qd, qdd = _state(model, q.shape[0])
    sim = _sim(model, q.shape[0])
    assert rel(_concat(sim.regressor_host(q, qd, qdd)), er.regressor(model, q, qd, qdd, concat=True)) <= 1e-12
    assert rel(_concat(sim.regressor_host(q)), er.regressor(model, q, concat=True)) <= 1e-12
    Y, _, _ = sim.regressor_host(q, qd, qdd)
    tau = sim.inverse_dynamics_host(q, qd, qdd)
    assert rel(Y @ inertial_parameters(model), tau) <= 1e-10


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 4096, 3)
    qd, qdd = _state(model, 4096, 4)
    full = _concat(_sim(model, 4096).regressor_host(q, qd, qdd))
    for n in (1, 31, 33, 100):
        assert np.array_equal(_concat(_sim(model, n).regressor_host(q[-n:], qd[-n:], qdd[-n:])), full[-n:]), n


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_regressor as er
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = _state(model, n)
    sim = _sim(model, n)
    rng = np.random.default_rng(13)
    vin = rng.normal(size=(n, n_q + 2 * nd, 2))
    got = _concat([x.reshape(n, -1, 2) for x in sim.regressor_jvp_host(q, qd, qdd, vin[:, :n_q], vin[:, n_q:n_q + nd], vin[:, n_q + nd:])])
    got = got.reshape(n, -1, 2)
    assert rel(got, er.regressor_jvp(model, q, vin, qd, qdd)) <= 1e-12
    r_Y, r_pi, _ = er.rows(model)
    G = rng.normal(size=(n, r_Y + 2 * r_pi))
    g = sim.regressor_vjp_host(q, qd, qdd, G[:, :r_Y], G[:, r_Y:r_Y + r_pi], G[:, r_Y + r_pi:])
    h = er.regressor_vjp(model, q, G, qd, qdd)
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
    V = np.random.default_rng(6).normal(size=(n, n_in, n_in))
    nq, nd = sim.n_q, sim.n_qd
    split = lambda W: (W[:, :nq], W[:, nq:nq + nd], W[:, nq + nd:])
    whole = sim.regressor_jvp_host(q, qd, qdd, *split(V))
    for j0 in range(0, n_in, chunk):
        part = sim.regressor_jvp_host(q, qd, qdd, *split(V[..., j0:j0 + chunk]))
        for a, b in zip(part, whole):
            assert np.array_equal(a, b[..., j0:j0 + chunk]), j0


def test_steps_unchanged_around_regressor_calls_and_parameters_do_not_enter():
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, qdd = _state(model, n)
    sim = _sim(model, n)
    before = sim.step_host(2, q, qd)
    ref = _concat(sim.regressor_host(q, qd, qdd))
    ids = all_ids(model)
    sim.set_physical_params(ids, perturbed(model, ids, n, 14, 0.5, 0.0))
    assert np.array_equal(_concat(sim.regressor_host(q, qd, qdd)), ref)
    sim.set_physical_params(None)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("name", ["humanoid", "laikago"])
def test_autograd_backward_and_forward_mode(name):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, _ = fixture(name)
    n = 64
    q = f32(_q(model, n, 7))
    qd, qdd = _state(model, n, 8)
    sim = _sim(model, n)
    dev = "cuda"
    qt, qdt, qddt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, qdd))
    Y, yT, yV = tds_b200.autograd.regressor(sim, qt, qdt, qddt)
    ref = sim.regressor_host(q, qd, qdd)
    for a, b in zip((Y, yT, yV), ref):
        assert a.dtype == torch.float64 and np.array_equal(a.cpu().numpy(), b)
    rng = np.random.default_rng(9)
    G = [rng.normal(size=x.shape) for x in ref]
    a, b, c = (x.clone().requires_grad_(True) for x in (qt, qdt, qddt))
    out = tds_b200.autograd.regressor(sim, a, b, c)
    sum((o * torch.tensor(g, device=dev)).sum() for o, g in zip(out, G)).backward()
    g = sim.regressor_vjp_host(q, qd, qdd, *G)
    for t, h in zip((a, b, c), g):
        assert t.grad.dtype == torch.float32
        assert rel(t.grad.cpu().double().numpy(), f32(h)) <= 1e-6
    # forward mode: forward_ad and torch.func.jvp against the C-ABI's JVP
    tv = [rng.normal(size=x.shape) for x in (q, qd, qdd)]
    ref_t = sim.regressor_jvp_host(q, qd, qdd, *tv)
    tt = [torch.tensor(x, dtype=torch.float32, device=dev) for x in tv]
    ref_t32 = sim.regressor_jvp_host(q, qd, qdd, *(f32(x) for x in tv))
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x, t) for x, t in zip((qt, qdt, qddt), tt)]
        outs = tds_b200.autograd.regressor(sim, *duals)
        for o, r in zip(outs, ref_t32):
            assert rel(fwAD.unpack_dual(o).tangent.cpu().numpy(), r) <= 1e-12
    _, jt = torch.func.jvp(lambda x, y, z: tds_b200.autograd.regressor(sim, x, y, z), (qt, qdt, qddt), tuple(tt))
    for o, r in zip(jt, ref_t32):
        assert rel(o.cpu().numpy(), r) <= 1e-12
    assert rel(_concat(ref_t32), _concat(ref_t)) <= 1e-5


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    sim = _sim(model, n)
    npi = sim.n_pi
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    qh = np.ascontiguousarray(q)
    yT, t, to, G, g = np.zeros((n, npi)), np.zeros((n, n_q, 1)), np.zeros((n, npi, 1)), np.zeros((n, npi)), np.zeros((n, n_q))
    host = L.tds_b200_regressor_host
    assert host(None, dp(qh), None, None, None, dp(yT), None) == -1
    assert host(h, None, None, None, None, dp(yT), None) == -1
    assert host(h, dp(qh), None, None, None, None, None) == -1
    assert host(h, dp(qh), None, None, None, dp(yT), None) == 0
    assert L.tds_b200_regressor_device(h, None, None, None, None, None, None, None) == -1
    jvp = L.tds_b200_regressor_jvp_host
    assert jvp(h, dp(qh), None, None, 0, dp(t), None, None, None, dp(to), None) == -1
    assert jvp(h, dp(qh), None, None, 1, None, None, None, None, dp(to), None) == -1
    assert jvp(h, dp(qh), None, None, 1, dp(t), None, None, None, None, None) == -1
    assert jvp(h, None, None, None, 1, dp(t), None, None, None, dp(to), None) == -1
    assert jvp(h, dp(qh), None, None, 1, dp(t), None, None, None, dp(to), None) == 0
    assert L.tds_b200_regressor_jvp_device(h, None, None, None, 1, None, None, None, None, None, None, None) == -1
    vjp = L.tds_b200_regressor_vjp_host
    assert vjp(h, dp(qh), None, None, None, dp(G), None, None, None, None) == -1
    assert vjp(h, dp(qh), None, None, None, None, None, dp(g), None, None) == -1
    assert vjp(h, None, None, None, None, dp(G), None, dp(g), None, None) == -1
    assert vjp(h, dp(qh), None, None, None, dp(G), None, dp(g), None, None) == 0
    assert L.tds_b200_regressor_vjp_device(h, None, None, None, None, None, None, None, None, None, None) == -1
    # NULL qd and qdd are zero
    a = _concat(sim.regressor_host(q))
    assert np.array_equal(a, _concat(sim.regressor_host(q, np.zeros((n, nd)), np.zeros((n, nd)))))
    # the Python layer
    z32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        tds_b200.autograd.regressor(sim, torch.zeros((n, n_q), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        tds_b200.autograd.regressor(sim, z32(n, n_q), z32(n, nd + 1))
    with pytest.raises(ValueError):
        sim.regressor_jvp_host(q)
    with pytest.raises(ValueError):
        sim.regressor_vjp_host(q)


def test_identification_of_laikago_end_to_end():
    """256 Laikago environments, each with its own installed +-20 % masses, +-1 cm centres of mass and +-20 % inertias; 32 random samples
    per environment with tau from inverse_dynamics_device; pi_hat = the minimum-norm least-squares solution of the stacked Y through a
    batched SVD with a relative cut-off (the stacked Y is rank-deficient).  Held-out tau is reproduced and the total mass recovered: with
    every other joint at rest, the vertical prismatic joint's row is (qdd_z + g) times the mass of every body after it, which is all of
    Laikago's mass (the root chain's links are massless)."""
    import torch
    model, _ = fixture("laikago")
    n, S, H = 256, 32, 8
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm.startswith("link") and ".stiffness" not in nm and ".damping" not in nm]
    rng = np.random.default_rng(21)
    pv = tds_b200.model.param_values(model)
    vals = np.repeat(pv[ids][None, :], n, axis=0)
    for j, i in enumerate(ids):
        nm = names[i]
        if ".com." in nm:
            vals[:, j] += rng.uniform(-0.01, 0.01, n)
        else:
            vals[:, j] *= rng.uniform(0.8, 1.2, n)
    sim = _sim(model, n)
    sim.set_physical_params(ids, vals)
    # the vertical prismatic joint: the root chain's dof whose axis is z
    L = model[16 + 13:16 + 13 + int(model[1]) * 34].reshape(-1, 34)
    masses = vals[:, [k for k, i in enumerate(ids) if names[i].endswith(".mass")]]
    total = masses.sum(axis=1)
    Ys, taus = [], []
    for s in range(S + H):
        q = f32(_q(model, n, 100 + s))
        qd, qdd = _state(model, n, 200 + s)
        Y, _, _ = sim.regressor_host(q, qd, qdd)
        qs = torch.tensor(q.T, dtype=torch.float32, device="cuda")
        qds = torch.tensor(qd.T, dtype=torch.float32, device="cuda")
        qdds = torch.tensor(qdd.T, dtype=torch.float32, device="cuda")
        pad = lambda t: torch.nn.functional.pad(t, (0, sim.n_stride - n))
        tau = torch.zeros((sim.n_qd, sim.n_stride), dtype=torch.float64, device="cuda")
        sim.inverse_dynamics_device(pad(qs).contiguous(), pad(qds).contiguous(), pad(qdds).contiguous(), tau)
        torch.cuda.synchronize()
        Ys.append(Y)
        taus.append(tau[:, :n].t().cpu().numpy())
    A = torch.tensor(np.concatenate(Ys[:S], axis=1), device="cuda")          # [n, S n_qd, n_pi]
    b = torch.tensor(np.concatenate(taus[:S], axis=1), device="cuda")        # [n, S n_qd]
    U, sv, Vh = torch.linalg.svd(A, full_matrices=False)
    keep = sv > sv[:, :1] * 1e-10
    inv = torch.where(keep, 1.0 / torch.where(keep, sv, torch.ones_like(sv)), torch.zeros_like(sv))
    pi_hat = (Vh.transpose(1, 2) @ (inv[:, :, None] * (U.transpose(1, 2) @ b[:, :, None])))[..., 0].cpu().numpy()
    print(f"numerical rank of one environment's stacked Y (Laikago's base parameters): {int(keep[0].sum())} of {A.shape[2]}")
    for s in range(S, S + H):
        got = np.einsum("erc,ec->er", Ys[s], pi_hat)
        assert np.all(np.abs(got - taus[s]) <= 1e-6 * np.maximum(1.0, np.abs(taus[s]))), np.abs(got - taus[s]).max()
    # the total mass: the projection of pi_hat on the identifiable direction of the vertical prismatic joint's gravity row
    zj = [i for i in range(L.shape[0]) if int(L[i, 1]) == 2]   # TDSJ_PRISMATIC_Z
    assert zj, "no vertical prismatic joint in Laikago's root chain"
    d = int(L[zj[0], 3])
    q0 = f32(_q(model, n, 999))
    Y0, _, _ = sim.regressor_host(q0)
    m_hat = np.abs(np.einsum("ec,ec->e", Y0[:, d], pi_hat)) / 9.81
    assert np.all(np.abs(m_hat - total) <= 1e-6 * total), np.abs(m_hat / total - 1).max()
