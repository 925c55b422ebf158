"""Inverse dynamics tau = ID(q, qd, qdd) (DESIGN.md section 7.14) on the CPU, from the kernel SOURCE: the INV instances of csrc/tds_stepw.cu
compiled for the host (tests/cpp/invdyn_host.cpp, bound by tests/emu_invdyn.py) against the C oracle's RNEA restated in link frames
(tests/cpp/oracle_invdyn.c), linearity in qdd against the mass matrix (section 7.12), the round trip through the forward dynamics of the
same kernel source, the Lagrangian identities that never touch the RNEA code (Coriolis from dM/dq, gravity from the point Jacobians of
section 7.13), per-environment parameters, the derivatives, and system identification by one Gauss-Newton step.
tests/test_inverse_dynamics_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_names, param_values, set_param_values
import emu
import emu_invdyn
import emu_kin
import emu_mass
from test_mass_matrix_on_host import HEADER, BASE, LINK, ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture, rel
from test_params_on_host import all_ids, perturbed

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
G = (0.0, 0.0, -9.81)


def state(model, q, seed=1, scale=1.0):
    """Random qd, qdd [n, n_qd] (rounded to fp32) for the configurations q."""
    rng = np.random.default_rng(seed)
    n, nd = q.shape[0], int(model[4])
    return f32(rng.normal(size=(n, nd)) * scale), f32(rng.normal(size=(n, nd)) * scale)


def links_of(model):
    n_links = int(model[1])
    return model[HEADER + BASE:HEADER + BASE + n_links * LINK].reshape(n_links, LINK)


def without_springs(model):
    """The model with every joint's stiffness and damping zeroed."""
    m = np.array(model, dtype=np.float64)
    L = links_of(m)
    L[:, 32] = 0.0
    L[:, 33] = 0.0
    m[HEADER + BASE:HEADER + BASE + L.size] = L.ravel()
    return m


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_against_the_c_oracle(name):
    model, q = fixture(name)
    qd, qdd = state(model, q)
    tau = emu_invdyn.inverse_dynamics(model, q, qd, qdd)
    to = np.array([emu_invdyn.oracle(model, a, b, c) for a, b, c in zip(f32(q), qd, qdd)])
    assert tau.shape == to.shape == (q.shape[0], int(model[4]))
    assert np.all(np.abs(tau - to) <= 1e-10 * np.maximum(1.0, np.abs(to))), rel(tau, to)


@pytest.mark.parametrize("name", ALL)
def test_linear_in_qdd_with_the_mass_matrix(name):
    """ID(q, qd, qdd) - ID(q, qd, 0) = M(q) qdd on every fixture: spherical joints, floating bases and worlds of several multibodies."""
    model, q = fixture(name)
    qd, qdd = state(model, q, 2)
    d = emu_invdyn.inverse_dynamics(model, q, qd, qdd) - emu_invdyn.inverse_dynamics(model, q, qd)
    Mq = np.einsum("eij,ej->ei", emu_mass.mass(model, q), qdd)
    assert np.abs(d - Mq).max() <= 1e-10 * max(1.0, np.abs(Mq).max())


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "ant", "humanoid_fixed", "pendulum5spherical", "humanoid_spherical",
                                  "mb_three_bodies", "mb_racket"])
def test_round_trip_through_the_forward_dynamics(name):
    """ID(q, qd, fl32(FD(q, qd, tau))) = tau on fixed bases (the fp64 world-frame step in MODE_FD, the same kernel source).  The error is
    the fp32 rounding of qdd, about |M| |qdd| 2^-24."""
    model, q = fixture(name)
    if int(model[2]):
        pytest.skip("floating base: ID is not the inverse of the reference's floating-base forward dynamics")
    rng = np.random.default_rng(4)
    n, nd = q.shape[0], int(model[4])
    qd = f32(rng.normal(size=(n, nd)) * 0.5)
    tau = f32(rng.normal(size=(n, nd)) * 2.0)
    qdd = f32(emu.step(model, 0, q, qd, tau, precision=1)["qdd"])
    back = emu_invdyn.inverse_dynamics(model, q, qd, qdd)
    M = emu_mass.mass(model, q)
    bound = 4 * 2.0 ** -24 * np.abs(M).max() * np.abs(qdd).max(axis=1, keepdims=True) * nd
    err = np.abs(back - tau)
    assert np.all(err <= bound), (err.max(), bound.max())
    print(f"{name}: largest round-trip error {err.max():.3e} (bound {bound.max():.3e})")


def _unit_tangents(n, dim):
    t = np.zeros((n, dim, dim))
    t[:, np.arange(dim), np.arange(dim)] = 1.0
    return t


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "cartpole_plane", "laikago"])
def test_coriolis_from_the_mass_matrix(name):
    """h(q, qd) - h(q, 0) = Mdot qd - 1/2 d(qd^T M qd)/dq, with dM/dq from the mass matrix's JVP along unit tangents (fixed bases
    without spherical joints, no springs: q and qd have the same coordinates).  Not Ant or the humanoid: their joint axes have lengths
    1 only to 1e-7 and 5e-6, and S = axis is then not exactly the derivative of the joint's rotation (link.hpp normalises the axis for
    the rotation only), so the identity holds there only to that relative size."""
    model, q = fixture(name)
    model = without_springs(model)
    q = f32(q)
    n, nd = q.shape[0], int(model[4])
    assert int(model[3]) == nd
    qd, _ = state(model, q, 5)
    h = emu_invdyn.inverse_dynamics(model, q, qd) - emu_invdyn.inverse_dynamics(model, q)
    dM = emu_mass.mass_jvp(model, q, _unit_tangents(n, nd))       # [n, i, j, c] = dM_ij / dq_c
    Mdot = np.einsum("eijc,ec->eij", dM, qd)
    ref = np.einsum("eij,ej->ei", Mdot, qd) - 0.5 * np.einsum("eijc,ei,ej->ec", dM, qd, qd)
    assert np.abs(h - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "ant", "humanoid_fixed"])
def test_gravity_from_the_point_jacobians(name):
    """h(q, 0) = -sum_i m_i J_ci^T g, J_ci the point Jacobian (section 7.13) at each link's centre of mass (fixed bases, no springs)."""
    model, q = fixture(name)
    model = without_springs(model)
    q = f32(q)
    L = links_of(model)
    moving_mass = L[:, 19] > 0
    links = np.nonzero(moving_mass)[0]
    _, _, J = emu_kin.kinematics(model, q, links, L[links, 20:23])
    ref = -np.einsum("k,ekrc,r->ec", L[links, 19], J, np.asarray(G))
    h = emu_invdyn.inverse_dynamics(model, q)
    assert np.abs(h - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())


def _par_model(name):
    model, q = fixture(name)
    ids = [i for i in all_ids(model) if param_names(model)[i] not in ("friction", "restitution")]
    return model, q, ids


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "pendulum5spherical", "humanoid_spherical", "mb_three_bodies"])
def test_parameters_at_the_model_values_are_bit_identical(name):
    model, q, ids = _par_model(name)
    qd, qdd = state(model, q)
    vals = param_values(model)[ids]
    assert np.array_equal(emu_invdyn.inverse_dynamics(model, q, qd, qdd, ids=ids, values=vals), emu_invdyn.inverse_dynamics(model, q, qd, qdd))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_per_environment_parameters_equal_edited_models(name):
    """+-20 % per-environment masses, centres of mass, inertias and random stiffness / damping are bit-identical to the instance without
    parameters on the flat model edited with those values."""
    model, q, ids = _par_model(name)
    qd, qdd = state(model, q)
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    tau = emu_invdyn.inverse_dynamics(model, q, qd, qdd, ids=ids, values=vals)
    for e in range(q.shape[0]):
        edited = set_param_values(model, ids, vals[e])
        assert np.array_equal(tau[e:e + 1], emu_invdyn.inverse_dynamics(edited, q[e:e + 1], qd[e:e + 1], qdd[e:e + 1])), (name, e)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_fixed"])
def test_jvp_against_central_differences_of_the_oracle(name):
    """dtau along random q, qd, qdd and parameter tangents against central differences of the C oracle on the edited model, h = 1e-6."""
    model, q, ids = _par_model(name)
    q = f32(q[:3])
    qd, qdd = state(model, q, 3)
    base = param_values(model)[ids]
    n_q, nd = int(model[3]), int(model[4])
    rng = np.random.default_rng(17)
    vin = rng.normal(size=(q.shape[0], n_q + 2 * nd))
    vp = rng.normal(size=(q.shape[0], len(ids))) * np.maximum(np.abs(base), 0.01)
    dtau = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, vin[:, :, None], vp[:, :, None], ids=ids, values=base)[..., 0]
    h = 1e-6
    for e in range(q.shape[0]):
        x = np.concatenate([q[e], qd[e], qdd[e]])

        def at(s):
            y = x + s * h * vin[e]
            return emu_invdyn.oracle(set_param_values(model, ids, base + s * h * vp[e]), y[:n_q], y[n_q:n_q + nd], y[n_q + nd:])
        fd = (at(1) - at(-1)) / (2 * h)
        assert np.all(np.abs(dtau[e] - fd) <= 1e-6 * max(1.0, np.abs(fd).max())), (name, e, np.abs(dtau[e] - fd).max())


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_derivative_in_qdd_is_the_mass_matrix(name):
    model, q = fixture(name)
    qd, qdd = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    t = np.zeros((n, n_q + 2 * nd, nd))
    t[:, n_q + nd:, :] = _unit_tangents(n, nd)
    dtau = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, t)
    M = emu_mass.mass(model, q)
    assert np.abs(dtau - M).max() <= 1e-10 * max(1.0, np.abs(M).max())


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_tangents_of_one_call_are_independent(name):
    """m tangents in one call are bit-identical to m calls with one tangent each."""
    model, q, ids = _par_model(name)
    ids = ids[:12]
    qd, qdd = state(model, q)
    vals = perturbed(model, ids, q.shape[0], 4, 0.5, 0.0)
    n_in = int(model[3]) + 2 * int(model[4])
    rng = np.random.default_rng(5)
    vin, vp = rng.normal(size=(q.shape[0], n_in, 3)), rng.normal(size=(q.shape[0], len(ids), 3))
    dtau = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, vin, vp, ids=ids, values=vals)
    for j in range(3):
        one = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, vin[:, :, j:j + 1], vp[:, :, j:j + 1], ids=ids, values=vals)
        assert np.array_equal(one[..., 0], dtau[..., j])


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    """<G, dtau[v]> = <VJP(G), v> within 1e-10, over q, qd, qdd and the installed parameters together."""
    model, q, ids = _par_model(name)
    qd, qdd = state(model, q)
    vals = perturbed(model, ids, q.shape[0], 8, 0.5, 0.0)
    rng = np.random.default_rng(6)
    n, nd = q.shape[0], int(model[4])
    n_in = int(model[3]) + 2 * nd
    Gc = rng.normal(size=(n, nd))
    vin, vp = rng.normal(size=(n, n_in)), rng.normal(size=(n, len(ids)))
    dtau = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, vin[:, :, None], vp[:, :, None], ids=ids, values=vals)[..., 0]
    g_in, g_par = emu_invdyn.inverse_dynamics_vjp(model, q, qd, qdd, Gc, ids=ids, values=vals)
    fwd = np.einsum("ei,ei->e", Gc, dtau)
    rev = np.einsum("ec,ec->e", g_in, vin) + np.einsum("ek,ek->e", g_par, vp)
    assert rel(fwd, rev) <= 1e-10


def test_system_identification_by_one_gauss_newton_step():
    """Laikago, 8 environments: the masses of its massive links and the damping of its moving joints (true damping drawn in [0.1, 0.5]),
    each environment starting from values off by +-20 %.  tau is linear in them, so one Gauss-Newton step on the torque residual, with
    the parameter JVP as the Jacobian, recovers the true values within 1e-8 relative.  (The massless links of the root chain sit at one
    point and move with it; their masses are not separable from the body's and are left out.)"""
    model, _ = fixture("laikago")
    names, L = param_names(model), links_of(model)
    link = lambda i: int(names[i][4:].split(".")[0])
    ids = [i for i, nm in enumerate(names) if nm.startswith("link") and
           ((nm.endswith(".mass") and L[link(i), 19] > 0) or (nm.endswith(".damping") and L[link(i), 1] >= 0))]
    rng = np.random.default_rng(11)
    truth = param_values(model)[ids]
    damping = np.array([names[i].endswith(".damping") for i in ids])
    truth[damping] = f32(rng.uniform(0.1, 0.5, int(damping.sum())))
    n_env, S = 8, 6
    n_q, nd, k = int(model[3]), int(model[4]), len(ids)
    guess = f32(truth * (1.0 + rng.uniform(-0.2, 0.2, size=(n_env, k))))   # (damping enters the step at fp32, as the model stores it)
    q = f32(rng.uniform(-0.5, 0.5, size=(n_env * S, n_q)))
    qd = f32(rng.normal(size=(n_env * S, nd)))
    qdd = f32(rng.normal(size=(n_env * S, nd)) * 3.0)
    measured = emu_invdyn.inverse_dynamics(model, q, qd, qdd, ids=ids, values=truth)
    g_rows = np.repeat(guess, S, axis=0)
    tau0 = emu_invdyn.inverse_dynamics(model, q, qd, qdd, ids=ids, values=g_rows)
    Jp = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, None, _unit_tangents(n_env * S, k), ids=ids, values=g_rows)
    for e in range(n_env):
        rows = slice(e * S, (e + 1) * S)
        A = Jp[rows].reshape(S * nd, k)
        assert np.linalg.matrix_rank(A) == k
        step = np.linalg.lstsq(A, (measured[rows] - tau0[rows]).ravel(), rcond=None)[0]
        est = guess[e] + step
        assert np.all(np.abs(est - truth) <= 1e-8 * np.abs(truth)), (e, np.abs(est / truth - 1).max())
