"""The joint-space mass matrix M(q) on the H100 (DESIGN.md section 7.12): the MASS instances of the world-frame kernel as nvcc builds
them, against the host build of the same source and the C oracle, on ragged and chunked batches, with installed parameters, through
torch.autograd (backward, forward_ad, torch.func.jvp), through pytinydiffsim.mass_matrix, and every argument check of the C-ABI.  The
CPU twins are in tests/test_mass_matrix_on_host.py."""
import ctypes
import os

import numpy as np
import pytest

import tds_b200
from tds_b200.model import fixture_path, load_model, param_values
from oracle import port
from test_mass_matrix_on_host import GOLDEN, ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, oracle, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu

ALL = ORACLE_FIXTURES + OTHER_FIXTURES


def _sim(model, n):
    return tds_b200.BatchSim(model, n, precision=1)


def _q(model, n, seed):
    """n random configurations (a floating base's quaternion normalised; spherical joints take any 4-vector as the kernel does)."""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, int(model[3]))) * 0.4
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    return q


@pytest.mark.parametrize("name", ALL)
def test_device_against_the_host_build_and_the_oracle(name):
    import emu_mass
    model, q = fixture(name)
    sim = _sim(model, q.shape[0])
    M = sim.mass_matrix_host(q)
    Mh = emu_mass.mass(model, q)
    assert rel(M, Mh) <= 1e-12
    assert np.array_equal(M, M.transpose(0, 2, 1))
    if name in ORACLE_FIXTURES:
        Mo = oracle(model, q)
        assert np.abs(M - Mo).max() <= 1e-10 * max(1.0, np.abs(Mo).max())


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q = _q(model, 100, 3)
    full = _sim(model, 100).mass_matrix_host(q)
    for n in (1, 31, 33, 100):
        assert np.array_equal(_sim(model, n).mass_matrix_host(q[-n:]), full[-n:]), n


def test_device_layout_and_host_layout_agree():
    import torch
    model, q = fixture("laikago")
    n = q.shape[0]
    sim = _sim(model, n)
    qs = torch.zeros((sim.n_q, sim.n_stride), dtype=torch.float32, device="cuda")
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    M = torch.zeros((sim.n_qd ** 2, sim.n_stride), dtype=torch.float64, device="cuda")
    sim.mass_matrix_device(qs, M)
    torch.cuda.synchronize()
    got = M[:, :n].t().reshape(n, sim.n_qd, sim.n_qd).cpu().numpy()
    assert np.array_equal(got, sim.mass_matrix_host(q))


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_and_vjp_against_the_host_build(name):
    import emu_mass
    model, q = fixture(name)
    n = q.shape[0]
    sim = _sim(model, n)
    ids = all_ids(model)
    vals = perturbed(model, ids, n, 12, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(13)
    vq, vp = rng.normal(size=(n, sim.n_q, 2)), rng.normal(size=(n, len(ids), 2))
    M, dM = sim.mass_matrix_jvp_host(q, vq, vp)
    assert rel(M, emu_mass.mass(model, q, ids=ids, values=vals)) <= 1e-12
    assert rel(dM, emu_mass.mass_jvp(model, q, vq, vp, ids=ids, values=vals)) <= 1e-12
    G = rng.normal(size=(n, sim.n_qd, sim.n_qd))
    g_q, g_par = sim.mass_matrix_vjp_host(q, G)
    hq, hp = emu_mass.mass_vjp(model, q, G, ids=ids, values=vals)
    assert rel(g_q, hq) <= 1e-12 and rel(g_par, hp) <= 1e-12
    fwd = np.einsum("eij,eij->e", G, dM[..., 0])
    assert rel(fwd, np.einsum("ec,ec->e", g_q, vq[:, :, 0]) + np.einsum("ek,ek->e", g_par, vp[:, :, 0])) <= 1e-10


def test_humanoid_jvp_in_several_chunks_equals_one_chunk():
    """A humanoid batch sized so that the tangents run in at least three launches of the chunk loop."""
    model, _ = fixture("humanoid")
    probe = _sim(model, 32)
    warps = probe.jacobian_chunk() // 3 + 1
    n = 32 * warps
    sim = _sim(model, n)
    chunk = sim.jacobian_chunk()
    m = 2 * chunk + 1
    assert 1 <= chunk < m
    q = _q(model, n, 5)
    V = np.random.default_rng(6).normal(size=(n, sim.n_q, m))
    _, dM = sim.mass_matrix_jvp_host(q, V)
    for j0 in range(0, m, chunk):
        _, part = sim.mass_matrix_jvp_host(q, V[:, :, j0:j0 + chunk])
        assert np.array_equal(part, dM[..., j0:j0 + chunk]), j0


def test_parameter_sets_installed_changed_and_cleared():
    """The model's values give M without a set, bit for bit; changed values change M as the edited model; clearing restores it; the
    step's outputs are bit-identical before and after the mass-matrix calls."""
    from tds_b200.model import set_param_values
    model, q = fixture("laikago")
    n = q.shape[0]
    sim = _sim(model, n)
    g = np.load(os.path.join(GOLDEN, "laikago.npz"))
    qd = g["qd_in"][:n]
    before = sim.step_host(2, q, qd)
    M0 = sim.mass_matrix_host(q)
    ids = all_ids(model)
    sim.set_physical_params(ids, param_values(model)[ids])
    assert np.array_equal(sim.mass_matrix_host(q), M0)
    vals = perturbed(model, ids, n, 14, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    M1 = sim.mass_matrix_host(q)
    for e in range(n):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert rel(M1[e:e + 1], _sim(edited, 1).mass_matrix_host(q[e:e + 1])) <= 1e-12
    sim.set_physical_params(None)
    assert np.array_equal(sim.mass_matrix_host(q), M0)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_and_forward_mode(with_params):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture("humanoid")
    n = q.shape[0]
    sim = _sim(model, n)
    ids = all_ids(model)[:20] if with_params else []
    vals = perturbed(model, ids, n, 15, 0.5, 0.0) if with_params else None
    if with_params:
        sim.set_physical_params(ids, vals)
    qt = torch.tensor(q, dtype=torch.float32, device="cuda")
    pt = torch.tensor(vals, dtype=torch.float64, device="cuda") if with_params else None
    rng = np.random.default_rng(16)
    G = rng.normal(size=(n, sim.n_qd, sim.n_qd))
    # backward against the VJP entry
    qr = qt.clone().requires_grad_(True)
    pr = pt.clone().requires_grad_(True) if with_params else None
    M = tds_b200.autograd.mass_matrix(sim, qr, pr)
    assert M.dtype == torch.float64 and tuple(M.shape) == (n, sim.n_qd, sim.n_qd)
    assert np.array_equal(M.detach().cpu().numpy(), sim.mass_matrix_host(f32(q)))
    (M * torch.tensor(G, device="cuda")).sum().backward()
    g_q, g_par = sim.mass_matrix_vjp_host(f32(q), G)
    assert qr.grad.dtype == torch.float32
    assert rel(qr.grad.cpu().numpy().astype(np.float64), g_q.astype(np.float32).astype(np.float64)) <= 1e-12
    if with_params:
        assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), g_par) <= 1e-12
    # forward mode against the JVP entry
    vq = rng.normal(size=(n, sim.n_q))
    vp = rng.normal(size=(n, len(ids))) if with_params else None
    _, ref = sim.mass_matrix_jvp_host(f32(q), vq.astype(np.float32), vp)
    tq = torch.tensor(vq, dtype=torch.float32, device="cuda")
    tp = torch.tensor(vp, dtype=torch.float64, device="cuda") if with_params else None
    with fwAD.dual_level():
        dq = fwAD.make_dual(qt, tq)
        dp = fwAD.make_dual(pt, tp) if with_params else None
        tan = fwAD.unpack_dual(tds_b200.autograd.mass_matrix(sim, dq, dp)).tangent.cpu().numpy()
    assert rel(tan, ref) <= 1e-12
    if with_params:
        _, (ft,) = torch.func.jvp(lambda a, b: (tds_b200.autograd.mass_matrix(sim, a, b),), (qt, pt), (tq, tp))
    else:
        _, (ft,) = torch.func.jvp(lambda a: (tds_b200.autograd.mass_matrix(sim, a),), (qt,), (tq,))
    assert rel(ft.cpu().numpy(), ref) <= 1e-12


def test_pytinydiffsim_mass_matrix_on_the_laikago_urdf():
    """pytinydiffsim.mass_matrix(mb) at mb.q and mass_matrix(mb, q) against the oracle on the Laikago model."""
    import pytinydiffsim as pd
    model = load_model(fixture_path("laikago"))
    mb = pd.TinyMultiBody(False)
    mb._model = model
    mb._bind(tds_b200.BatchSim(model, 1, precision=1))
    q = f32(fixture("laikago")[1][0])
    mb.q[:] = q
    M = pd.mass_matrix(mb)
    assert M.shape == (18, 18)
    Mo = port.mass_matrix(model, q)
    assert np.abs(M - Mo).max() <= 1e-10 * max(1.0, np.abs(Mo).max())
    q2 = f32(q + 0.1)
    assert np.abs(pd.mass_matrix(mb, q2) - port.mass_matrix(model, q2)).max() <= 1e-10 * max(1.0, np.abs(Mo).max())
    assert np.array_equal(mb.q, q)


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n = q.shape[0]
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    qh, M = np.ascontiguousarray(q), np.zeros((n, 2, 2))
    t, tM, G, g = np.zeros((n, 2, 1)), np.zeros((n, 2, 2, 1)), np.zeros((n, 2, 2)), np.zeros((n, 2))
    assert L.tds_b200_mass_matrix_host(None, dp(qh), dp(M)) == -1
    assert L.tds_b200_mass_matrix_host(h, None, dp(M)) == -1
    assert L.tds_b200_mass_matrix_host(h, dp(qh), None) == -1
    assert L.tds_b200_mass_matrix_device(h, None, None, None) == -1
    assert L.tds_b200_mass_matrix_jvp_host(h, dp(qh), 0, dp(t), None, None, dp(tM)) == -1
    assert L.tds_b200_mass_matrix_jvp_host(h, dp(qh), 1, None, None, None, dp(tM)) == -1
    assert L.tds_b200_mass_matrix_jvp_host(h, dp(qh), 1, dp(t), None, None, None) == -1
    assert L.tds_b200_mass_matrix_jvp_host(h, dp(qh), 1, None, dp(t), None, dp(tM)) == -4
    assert L.tds_b200_mass_matrix_jvp_device(h, None, 1, None, None, None, None, None) == -1
    assert L.tds_b200_mass_matrix_vjp_host(h, dp(qh), dp(G), None, None) == -1
    assert L.tds_b200_mass_matrix_vjp_host(h, dp(qh), None, dp(g), None) == -1
    assert L.tds_b200_mass_matrix_vjp_host(h, dp(qh), dp(G), None, dp(g)) == -4
    assert L.tds_b200_mass_matrix_vjp_device(h, None, None, None, None, None) == -1
    # the Python layer
    with pytest.raises(ValueError):
        tds_b200.autograd.mass_matrix(sim, torch.zeros((n, 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        tds_b200.autograd.mass_matrix(sim, torch.zeros((n, 2), dtype=torch.float32, device="cuda"),
                                      torch.zeros((n, 1), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        sim.mass_matrix_jvp_host(q, np.zeros((n, 3, 1)))
