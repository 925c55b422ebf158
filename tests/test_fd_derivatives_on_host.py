"""The derivatives of the forward dynamics d qdd / dq, d qdd / dqd, d qdd / dtau (DESIGN.md section 7.24) on the CPU, from the kernel
SOURCE: the product kernel of csrc/tds_fd_derivatives.cu and the DER instances of csrc/tds_stepw.cu reading qdd in fp64, compiled for the
host (tests/cpp/fd_derivatives_host.cpp) and composed with the host builds of INV, MINV and the constrained dynamics' solve as the C-ABI
composes them (tests/emu_fd_derivatives.py), on the thirteen mass-matrix fixtures: against the host constrained-dynamics JVP along dq_dt
tangents and unit tangents, the host constrained dynamics and mass inverse bit for bit, the equation of motion with the host MASS build,
central differences of the C oracle, damping, worlds of several multibodies, installed parameters, and the JVP against central differences
of the fp64 value.  Tolerances scale with the conditioning of M: B = tol kappa_2(M) max|ref|, as in section 7.21.
tests/test_fd_derivatives_gpu.py checks the same kernels as nvcc builds them, through the C-ABI."""
import numpy as np
import pytest

from oracle import port
import emu_constrained_dynamics as ecd
import emu_dynamics_derivatives as ed
import emu_fd_derivatives as ef
import emu_invdyn
import emu_mass
import emu_mass_inverse as emi
from test_dynamics_derivatives_on_host import tangent_basis
from test_mass_inverse_on_host import kappa
from test_mass_matrix_on_host import BASE, HEADER, LINK, ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture
from test_params_on_host import all_ids, perturbed
from test_point_motion_on_host import grid_state
from tds_b200.model import param_names, param_values, set_param_values

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
# fixed bases whose C oracle runs the MODE_FD step (stiffness and damping included)
FD_STEP = ["pendulum5", "cartpole", "humanoid_fixed"]
N = 3


def state(model, q, seed=1):
    """The fixture's first N configurations, random velocities and joint forces [N, n_qd], all fp32."""
    q = f32(q[:N])
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return q, f32(rng.normal(size=(q.shape[0], nd)) * 0.5), f32(rng.normal(size=(q.shape[0], nd)) * 3.0)


def within(X, ref, kM, tol=1e-13):
    """|X - ref| <= tol kappa_2(M) max|ref| elementwise."""
    return bool(np.all(np.abs(X - ref) <= tol * kM * max(np.abs(ref).max(), 1e-300)))


@pytest.mark.parametrize("name", ALL)
def test_columns_equal_the_constrained_dynamics_jvp(name):
    """Column k of d qdd / dq is the host constrained-dynamics JVP (K = 0) along dq_dt(q, e_k), of d qdd / dqd along e_k in qd and of
    d qdd / dtau along e_k in tau, within 1e-13 kappa_2(M) max|ref|."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    n, nd = q.shape[0], int(model[4])
    _, dq, dqd, dtau = ef.forward_dynamics_derivatives(model, q, qd, tau)
    eye = np.broadcast_to(np.eye(nd), (n, nd, nd)).copy()
    kM = kappa(emu_mass.mass(model, q))
    for X, t in ((dq, dict(t_q=tangent_basis(model, q))), (dqd, dict(t_qd=eye)), (dtau, dict(t_tau=eye))):
        ref, _ = ecd.constrained_dynamics_jvp(model, q, qd, tau, **t)
        assert within(X, ref, kM), (name, list(t), np.abs(X - ref).max(), np.abs(ref).max())


@pytest.mark.parametrize("name", ALL)
def test_qdd_and_d_qdd_d_tau_are_the_existing_queries_bit_for_bit(name):
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    qdd, _, _, dtau = ef.forward_dynamics_derivatives(model, q, qd, tau)
    assert np.array_equal(qdd, ecd.constrained_dynamics(model, q, qd, tau)[0])
    assert np.array_equal(dtau, emi.mass_inverse(model, q))


@pytest.mark.parametrize("name", ALL)
def test_equation_of_motion_residual(name):
    """M d qdd / dq + d tau / dq (q, qd, qdd) = 0 and M d qdd / dqd + d tau / dqd = 0 with the host MASS build, qdd in fp64."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    qdd, dq, dqd, _ = ef.forward_dynamics_derivatives(model, q, qd, tau)
    M = emu_mass.mass(model, q)
    Aq, Aqd = ef.der_qdd64(model, q, qd, qdd)
    kM = kappa(M)
    for X, A in ((dq, Aq), (dqd, Aqd)):
        r = M @ X + A
        assert np.abs(r).max() <= 1e-13 * kM * max(np.abs(A).max(), 1.0), (name, np.abs(r).max())


@pytest.mark.parametrize("name", ALL)
def test_fp64_qdd_of_the_derivative_instances(name):
    """DER reading qdd in fp64 is bit for bit its fp32 path when qdd is fp32-exact; otherwise d tau / dq moves by the MASS JVP term
    dM[dq_dt(e_k)] (qdd64 - qdd32) (within 1e-12 max|d tau / dq|) and d tau / dqd, which does not depend on qdd, barely at all."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    qdd, _ = ecd.constrained_dynamics(model, q, qd, tau)
    q32 = f32(qdd)
    a32, b32 = ed.inverse_dynamics_derivatives(model, q, qd, q32)
    a, b = ef.der_qdd64(model, q, qd, q32)
    assert np.array_equal(a, a32) and np.array_equal(b, b32)
    a64, b64 = ef.der_qdd64(model, q, qd, qdd)
    dM = emu_mass.mass_jvp(model, q, t_q=tangent_basis(model, q))   # [n, nd, nd, nd]: dM_rc along column k
    pred = np.einsum("erck,ec->erk", dM, qdd - q32)
    scale = max(np.abs(a32).max(), 1.0)
    assert np.abs((a64 - a32) - pred).max() <= 1e-12 * scale, (name, np.abs((a64 - a32) - pred).max())
    assert np.abs(b64 - b32).max() <= 1e-12 * max(np.abs(b32).max(), 1.0)


def _solve_oracle(model, q, qd, tau):
    return np.linalg.solve(port.mass_matrix(model, q), tau - emu_invdyn.oracle(model, q, qd))


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_columns_against_central_differences_of_the_oracle(name):
    """Every column against central differences (h = 1e-6) along q +- h dq_dt(q, e_k), qd +- h e_k and tau +- h e_k: of the C oracle's
    MODE_FD qdd on the fixed bases that step, of numpy's solve of the oracle's M and h on the others (floating bases).  The oracle has no
    spherical joints; test_jvp_against_central_differences covers them."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    q, qd, tau = q[:1], qd[:1], tau[:1]
    nd = int(model[4])
    _, dq, dqd, dtau = ef.forward_dynamics_derivatives(model, q, qd, tau)
    if name in FD_STEP:
        F = lambda a, b, c: port.step(model, port.make_params(), 0, a, b, c)["qdd"]
    else:
        F = lambda a, b, c: _solve_oracle(model, a, b, c)
    T = tangent_basis(model, q)[0]
    h = 1e-6
    E = np.eye(nd)
    cd = lambda f: np.stack([(f(k, h) - f(k, -h)) / (2 * h) for k in range(nd)], axis=1)
    fq = cd(lambda k, s: F(q[0] + s * T[:, k], qd[0], tau[0]))
    fqd = cd(lambda k, s: F(q[0], qd[0] + s * E[k], tau[0]))
    ft = cd(lambda k, s: F(q[0], qd[0], tau[0] + s * E[k]))
    for X, ref in ((dq, fq), (dqd, fqd), (dtau, ft)):
        err = np.abs(X[0] - ref).max() / max(1.0, np.abs(ref).max())
        assert err <= 1e-6, (name, err)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "pendulum5spherical", "humanoid_fixed", "laikago", "humanoid_spherical"])
def test_damping_adds_minus_m_inverse_times_its_diagonal(name):
    """Installing every joint's damping at d changes d qdd / dqd by -M^-1 diag(d) (zero on a floating base's dofs)."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm.endswith(".damping")]
    n, nd = q.shape[0], int(model[4])
    d = 0.375
    _, _, a, Mi = ef.forward_dynamics_derivatives(model, q, qd, tau, ids=ids, values=np.full((n, len(ids)), d))
    _, _, b, _ = ef.forward_dynamics_derivatives(model, q, qd, tau, ids=ids, values=np.zeros((n, len(ids))))
    want = np.full(nd, d)
    want[:6 if int(model[2]) else 0] = 0.0
    ref = -Mi * want[None, None, :]
    assert within(a - b, ref, kappa(emu_mass.mass(model, q)), 1e-12), (name, np.abs(a - b - ref).max())


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_worlds_give_exact_zeros_between_multibodies(name):
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    n_links, nd = int(model[1]), int(model[4])
    links = model[HEADER + BASE:HEADER + BASE + n_links * LINK].reshape(n_links, LINK)
    roots = [i for i in range(n_links) if links[i, 0] < 0] + [n_links]
    assert len(roots) > 2
    body = np.zeros(nd, dtype=int)
    for b in range(len(roots) - 1):
        later = links[roots[b + 1]:]
        later = later[later[:, 1] >= 0]
        body[int(later[:, 3].min()) if later.size else nd:] = b + 1
    between = body[:, None] != body[None, :]
    for X in ef.forward_dynamics_derivatives(model, q, qd, tau)[1:]:
        assert np.all(X[:, between] == 0)
        assert np.any(X[:, ~between] != 0)


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical"])
def test_parameters(name):
    """A set installed at the model's values is bitwise equal to no set; +-20 % values per environment equal the edited flat models."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    ids = [i for i in all_ids(model) if i >= 2]   # (friction and restitution do not enter)
    base = ef.forward_dynamics_derivatives(model, q, qd, tau)
    same = ef.forward_dynamics_derivatives(model, q, qd, tau, ids=ids, values=param_values(model)[ids])
    assert all(np.array_equal(a, b) for a, b in zip(base, same))
    vals = perturbed(model, ids, q.shape[0], 5, 0.2, 0.0)
    got = ef.forward_dynamics_derivatives(model, q, qd, tau, ids=ids, values=vals)
    for e in range(q.shape[0]):
        ref = ef.forward_dynamics_derivatives(set_param_values(model, ids, vals[e]), q[e:e + 1], qd[e:e + 1], tau[e:e + 1])
        for a, b in zip(got, ref):
            assert np.array_equal(a[e], b[0]), e


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "sphere2", "humanoid", "pendulum5spherical", "humanoid_spherical",
                                  "mb_three_bodies"])
def test_jvp_against_central_differences(name):
    """Along q (in n_q coordinates), qd, tau and the parameters separately, the JVP of all four outputs against central differences of
    the fp64 value at h = 2^-10, on grids that keep x +- h v exact in fp32 (the parameters are fp64 inputs: h = 2^-16).  Along q and the
    parameters the truncation error bounds the tolerance; the outputs are at most quadratic in qd and tau, so along those only rounding is
    left."""
    model, q = fixture(name)
    q, qd, tau = grid_state(model, q, 23)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = [i for i in all_ids(model) if i >= 2]
    p0 = np.tile(param_values(model)[ids], (n, 1))
    rng = np.random.default_rng(29)
    for part, dim, tol in ((0, n_q, 1e-4), (1, nd, 1e-8), (2, nd, 1e-8), (3, len(ids), 1e-6)):
        h = 2.0 ** (-16 if part == 3 else -10)
        v = np.round(rng.normal(size=(n, dim)) * 16) / 16
        if part == 3:
            v = v * np.maximum(np.abs(p0), 1e-2)
        x = [q, qd, tau, p0]
        xp, xm = list(x), list(x)
        xp[part], xm[part] = x[part] + h * v, x[part] - h * v
        if part < 3:
            assert np.array_equal(f32(xp[part]), xp[part]) and np.array_equal(f32(xm[part]), xm[part])
        P = ef.forward_dynamics_derivatives(model, *xp[:3], ids=ids, values=xp[3])
        Mn = ef.forward_dynamics_derivatives(model, *xm[:3], ids=ids, values=xm[3])
        t = [None] * 4
        t[part] = v[:, :, None]
        jv = ef.forward_dynamics_derivatives_jvp(model, q, qd, tau, *t, ids=ids, values=p0)
        for o in range(4):
            fd = (P[o] - Mn[o]) / (2 * h)
            err = np.abs(jv[o][..., 0] - fd).max() / max(1.0, np.abs(fd).max())
            assert err <= tol, (name, part, o, err)


@pytest.mark.parametrize("name", ["box", "laikago", "humanoid_spherical"])
def test_tangents_of_one_call_are_independent_and_linear(name):
    """m tangents in one call are bit-identical to single calls; <G, J V> = <J^T G, V> with J^T G from the identity tangents, as the VJP
    contracts them."""
    model, q = fixture(name)
    q, qd, tau = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = all_ids(model)[2:8]
    vals = perturbed(model, ids, n, 15, 0.2, 0.0)
    rng = np.random.default_rng(16)
    V = [rng.normal(size=(n, d, 3)) for d in (n_q, nd, nd, len(ids))]
    run = lambda T: ef.forward_dynamics_derivatives_jvp(model, q, qd, tau, *T, ids=ids, values=vals)
    full = run(V)
    for j in range(3):
        one = run([v[..., j:j + 1] for v in V])
        assert all(np.array_equal(a[..., 0], b[..., j]) for a, b in zip(one, full)), j
    dims = (n_q, nd, nd, len(ids))
    total = sum(dims)
    eye = [np.zeros((n, d, total)) for d in dims]
    c0 = 0
    for E, d in zip(eye, dims):
        E[:, np.arange(d), c0 + np.arange(d)] = 1.0
        c0 += d
    flat = lambda outs, m: np.concatenate([o.reshape(n, -1, m) for o in outs], axis=1)
    Jcols = flat(run(eye), total)
    G = rng.normal(size=(n, Jcols.shape[1]))
    gT = np.einsum("er,erc->ec", G, Jcols)
    fwd = np.einsum("er,erm->em", G, flat(full, 3))
    back = np.einsum("ec,ecm->em", gT, np.concatenate(V, axis=1))
    assert np.abs(fwd - back).max() <= 1e-9 * max(1.0, np.abs(fwd).max())


def test_argument_checks():
    """Every entry point returns -1 without a simulator (before any device work, so on a machine without a GPU too)."""
    import tds_b200
    L = tds_b200.lib()
    z = None
    assert L.tds_b200_forward_dynamics_derivatives_device(z, z, z, z, z, z, z, z, z) == -1
    assert L.tds_b200_forward_dynamics_derivatives_host(z, z, z, z, z, z, z, z) == -1
    assert L.tds_b200_forward_dynamics_derivatives_jvp_device(z, z, z, z, 1, *[z] * 13) == -1
    assert L.tds_b200_forward_dynamics_derivatives_jvp_host(z, z, z, z, 1, *[z] * 12) == -1
    assert L.tds_b200_forward_dynamics_derivatives_vjp_device(z, z, z, z, *[z] * 9) == -1
    assert L.tds_b200_forward_dynamics_derivatives_vjp_host(z, z, z, z, *[z] * 8) == -1
