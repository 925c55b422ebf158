"""The Coriolis matrix on the H100 (DESIGN.md section 7.22): the COR instances of the world-frame kernel as nvcc builds them, against the
host build of the same source, on ragged and chunked batches, with installed parameters, around steps, through torch.autograd (backward,
forward_ad, torch.func.jvp), M' - 2 C skew-symmetric and C qd against the device inverse dynamics at 4096 Laikago environments, and every
argument check of the C-ABI.  The CPU twins are in tests/test_coriolis_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
from tds_b200.model import param_names, set_param_values
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, rel
from test_params_on_host import all_ids, perturbed

pytestmark = pytest.mark.gpu


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


def _inertial_ids(model):
    names = param_names(model)
    return [i for i in all_ids(model) if names[i].split(".")[-1] not in ("friction", "restitution", "stiffness", "damping")]


@pytest.mark.parametrize("name", ORACLE_FIXTURES + OTHER_FIXTURES)
def test_device_against_the_host_build(name):
    import emu_coriolis as ecor
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd = _qd(model, n)
    sim = _sim(model, n)
    assert rel(sim.coriolis_host(q, qd), ecor.coriolis(model, q, qd)) <= 1e-12
    assert np.all(sim.coriolis_host(q) == 0.0)
    rng = np.random.default_rng(12)
    tq, tqd = rng.normal(size=(n, n_q, 2)), rng.normal(size=(n, nd, 2))
    C, dC = sim.coriolis_jvp_host(q, qd, tq, tqd)
    assert rel(C, ecor.coriolis(model, q, qd)) <= 1e-12
    assert rel(dC, ecor.coriolis_jvp(model, q, qd, tq, tqd)) <= 1e-12


@pytest.mark.parametrize("name", ["laikago", "humanoid", "humanoid_spherical"])
def test_ragged_batches_equal_the_full_batch(name):
    model, _ = fixture(name)
    q, qd = _q(model, 4096, 3), _qd(model, 4096, 4)
    full = _sim(model, 4096).coriolis_host(q, qd)
    for n in (1, 31, 33, 100):
        assert np.array_equal(_sim(model, n).coriolis_host(q[-n:], qd[-n:]), full[-n:]), n


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical"])
def test_jvp_and_vjp_with_parameters_against_the_host_build(name):
    import emu_coriolis as ecor
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd = _qd(model, n)
    sim = _sim(model, n)
    ids = _inertial_ids(model)
    vals = perturbed(model, ids, n, 12, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(13)
    tq, tqd, tp = rng.normal(size=(n, n_q, 2)), rng.normal(size=(n, nd, 2)), rng.normal(size=(n, len(ids), 2))
    C, dC = sim.coriolis_jvp_host(q, qd, tq, tqd, tp)
    assert rel(C, ecor.coriolis(model, q, qd, ids=ids, values=vals)) <= 1e-12
    assert rel(dC, ecor.coriolis_jvp(model, q, qd, tq, tqd, tp, ids=ids, values=vals)) <= 1e-12
    G = rng.normal(size=(n, nd, nd))
    g = sim.coriolis_vjp_host(q, qd, G)
    h = ecor.coriolis_vjp(model, q, qd, G, ids=ids, values=vals)
    for a, b in zip(g, h):
        assert rel(a, b) <= 1e-12
    fwd = np.einsum("eij,eij->e", G, dC[..., 0])
    rev = sum(np.einsum("ec,ec->e", a, b) for a, b in zip(g, (tq[..., 0], tqd[..., 0], tp[..., 0])))
    assert rel(fwd, rev) <= 1e-10


def test_humanoid_jvp_in_several_chunks_equals_one_call():
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
    _, whole = sim.coriolis_jvp_host(q, qd, V[:, :sim.n_q], V[:, sim.n_q:])
    for j0 in range(0, n_in, chunk):
        _, part = sim.coriolis_jvp_host(q, qd, V[:, :sim.n_q, j0:j0 + chunk], V[:, sim.n_q:, j0:j0 + chunk])
        assert np.array_equal(part, whole[..., j0:j0 + chunk]), j0


def test_parameters_installed_changed_cleared_and_steps_around_calls():
    model, q = fixture("laikago")
    n = q.shape[0]
    qd = _qd(model, n)
    sim = _sim(model, n)
    before = sim.step_host(2, q, qd)
    C0 = sim.coriolis_host(q, qd)
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm in ("friction", "restitution") or nm.endswith((".stiffness", ".damping"))]
    sim.set_physical_params(ids, perturbed(model, ids, n, 14, 0.5, 0.0))
    assert np.array_equal(sim.coriolis_host(q, qd), C0)
    ids = _inertial_ids(model)
    for seed in (15, 16):
        vals = perturbed(model, ids, n, seed, 0.5, 0.0)
        sim.set_physical_params(ids, vals)
        C1 = sim.coriolis_host(q, qd)
        for e in range(n):
            ref = _sim(set_param_values(model, ids, vals[e]), 1).coriolis_host(q[e:e + 1], qd[e:e + 1])
            assert np.array_equal(C1[e:e + 1], ref), (seed, e)
    sim.set_physical_params(None)
    assert np.array_equal(sim.coriolis_host(q, qd), C0)
    after = sim.step_host(2, q, qd)
    assert np.array_equal(after["q"], before["q"]) and np.array_equal(after["qd"], before["qd"])


@pytest.mark.parametrize("with_params", [False, True])
def test_autograd_backward_and_forward_mode(with_params):
    import torch
    import torch.autograd.forward_ad as fwAD
    model, q = fixture("humanoid")
    n = q.shape[0]
    q = f32(q)
    qd = _qd(model, n)
    sim = _sim(model, n)
    ids = _inertial_ids(model)[:20] if with_params else []
    vals = perturbed(model, ids, n, 15, 0.5, 0.0) if with_params else None
    if with_params:
        sim.set_physical_params(ids, vals)
    cu = lambda x, dt=torch.float32: torch.tensor(x, dtype=dt, device="cuda")
    xs = [cu(q), cu(qd)]
    pt = cu(vals, torch.float64) if with_params else None
    rng = np.random.default_rng(16)
    G = rng.normal(size=(n, sim.n_qd, sim.n_qd))
    xr = [x.clone().requires_grad_(True) for x in xs]
    pr = pt.clone().requires_grad_(True) if with_params else None
    C = tds_b200.autograd.coriolis(sim, *xr, params=pr)
    assert C.dtype == torch.float64 and tuple(C.shape) == (n, sim.n_qd, sim.n_qd)
    assert np.array_equal(C.detach().cpu().numpy(), sim.coriolis_host(q, qd))
    (C * cu(G, torch.float64)).sum().backward()
    ref = sim.coriolis_vjp_host(q, qd, G)
    for x, g in zip(xr, ref[:2]):
        assert x.grad.dtype == torch.float32 and rel(x.grad.cpu().numpy().astype(np.float64), f32(g)) <= 1e-12
    if with_params:
        assert pr.grad.dtype == torch.float64 and rel(pr.grad.cpu().numpy(), ref[2]) <= 1e-12
    v = [f32(rng.normal(size=x.shape)) for x in (q, qd)]
    vp = rng.normal(size=(n, len(ids))) if with_params else None
    _, want = sim.coriolis_jvp_host(q, qd, *v, vp)
    ts = [cu(x) for x in v]
    tp = cu(vp, torch.float64) if with_params else None
    with fwAD.dual_level():
        duals = [fwAD.make_dual(x, t) for x, t in zip(xs, ts)]
        dp = fwAD.make_dual(pt, tp) if with_params else None
        tan = fwAD.unpack_dual(tds_b200.autograd.coriolis(sim, *duals, params=dp)).tangent.cpu().numpy()
    assert rel(tan, want) <= 1e-12
    if with_params:
        _, ft = torch.func.jvp(lambda a, b, c: tds_b200.autograd.coriolis(sim, a, b, c), (*xs, pt), (*ts, tp))
    else:
        _, ft = torch.func.jvp(lambda a, b: tds_b200.autograd.coriolis(sim, a, b), tuple(xs), tuple(ts))
    assert rel(ft.cpu().numpy(), want) <= 1e-12


def test_laikago_4096_skew_symmetry_and_bias_forces_on_the_device():
    """At 4096 Laikago states on the device: M' - 2 C is skew-symmetric (M' the mass matrix's JVP along dq/dt) and C qd = ID(q, qd) -
    ID(q, 0) with the joint damping zeroed."""
    import torch
    from test_inverse_dynamics_on_host import without_springs
    from test_point_motion_on_host import dq_dt
    model, q0 = fixture("laikago")
    model = without_springs(model)
    n, n_q, nd = 4096, int(model[3]), int(model[4])
    sim = _sim(model, n)
    rng = np.random.default_rng(21)
    q = f32(q0[rng.integers(0, q0.shape[0], n)] + rng.uniform(-0.2, 0.2, size=(n, n_q)))
    qd = _qd(model, n, 22)
    ns = sim.n_stride
    soa = lambda x, dt: torch.tensor(np.pad(x.T, ((0, 0), (0, ns - n))), dtype=dt, device="cuda").contiguous()
    qs, qds = soa(q, torch.float32), soa(qd, torch.float32)
    C = torch.zeros((nd * nd, ns), dtype=torch.float64, device="cuda")
    dM = torch.zeros((nd * nd, ns), dtype=torch.float64, device="cuda")
    tau1 = torch.zeros((nd, ns), dtype=torch.float64, device="cuda")
    tau0 = torch.zeros((nd, ns), dtype=torch.float64, device="cuda")
    sim.coriolis_device(qs, qds, C)
    sim.mass_matrix_jvp_device(qs, 1, soa(np.stack([dq_dt(model, a, b) for a, b in zip(q, qd)]), torch.float64), None, dM)
    sim.inverse_dynamics_device(qs, qds, None, tau1)
    sim.inverse_dynamics_device(qs, None, None, tau0)
    torch.cuda.synchronize()
    C = C[:, :n].t().reshape(n, nd, nd).cpu().numpy()
    dM = dM[:, :n].t().reshape(n, nd, nd).cpu().numpy()
    K = dM - 2 * C
    assert np.abs(K + K.transpose(0, 2, 1)).max() <= 1e-12 * max(1.0, np.abs(dM).max())
    h = (tau1 - tau0)[:, :n].t().cpu().numpy()
    Cq = np.einsum("eij,ej->ei", C, qd)
    assert np.all(np.abs(Cq - h) <= 1e-10 * np.maximum(1.0, np.abs(h))), np.abs(Cq - h).max()


def test_argument_checks():
    import torch
    L = tds_b200.lib()
    model, q = fixture("cartpole")
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    sim = _sim(model, n)
    h = sim._h
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    qh, C, t, tC, G, g = (np.ascontiguousarray(q), np.zeros((n, nd * nd)), np.zeros((n, n_q, 1)), np.zeros((n, nd * nd, 1)),
                          np.zeros((n, nd * nd)), np.zeros((n, n_q)))
    assert L.tds_b200_coriolis_host(None, dp(qh), None, dp(C)) == -1
    assert L.tds_b200_coriolis_host(h, None, None, dp(C)) == -1
    assert L.tds_b200_coriolis_host(h, dp(qh), None, None) == -1
    assert L.tds_b200_coriolis_device(h, None, None, None, None) == -1
    assert L.tds_b200_coriolis_jvp_host(h, dp(qh), None, 0, dp(t), None, None, None, dp(tC)) == -1
    assert L.tds_b200_coriolis_jvp_host(h, dp(qh), None, 1, None, None, None, None, dp(tC)) == -1
    assert L.tds_b200_coriolis_jvp_host(h, dp(qh), None, 1, dp(t), None, None, dp(C), None) == -1
    assert L.tds_b200_coriolis_jvp_host(h, None, None, 1, dp(t), None, None, None, dp(tC)) == -1
    assert L.tds_b200_coriolis_jvp_host(h, dp(qh), None, 1, None, None, dp(t), None, dp(tC)) == -4
    assert L.tds_b200_coriolis_jvp_device(h, None, None, 1, None, None, None, None, None, None) == -1
    assert L.tds_b200_coriolis_vjp_host(h, dp(qh), None, None, dp(g), None, None) == -1
    assert L.tds_b200_coriolis_vjp_host(h, dp(qh), None, dp(G), None, None, None) == -1
    assert L.tds_b200_coriolis_vjp_host(h, None, None, dp(G), dp(g), None, None) == -1
    assert L.tds_b200_coriolis_vjp_host(h, dp(qh), None, dp(G), None, None, dp(g)) == -4
    assert L.tds_b200_coriolis_vjp_device(h, None, None, None, None, None, None, None) == -1
    # the Python layer
    z32 = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        tds_b200.autograd.coriolis(sim, torch.zeros((n, n_q), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        tds_b200.autograd.coriolis(sim, z32(n, n_q), z32(n, nd + 1))
    with pytest.raises(ValueError):
        tds_b200.autograd.coriolis(sim, z32(n, n_q), None, torch.zeros((n, 1), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        sim.coriolis_jvp_host(q)
