"""Joint-torque and energy regressors of the inertial parameters (DESIGN.md section 7.19) on the CPU, from the kernel SOURCE: the REG
instances of csrc/tds_stepw.cu compiled for the host (tests/cpp/regressor_host.cpp, bound by tests/emu_regressor.py) against the
inverse-dynamics instances of section 7.14 (tests/emu_invdyn.py) at the model's values and at installed parameter sets, the C oracle's
link-frame RNEA column by column, the mass matrix of section 7.12 (kinetic energy), the kinematics of section 7.13 (potential energy), and
the derivatives (JVP against central differences, independence of the tangents of one call, JVP / VJP duality).
tests/test_regressor_gpu.py checks the same instances as nvcc builds them, and the C-ABI."""
import numpy as np
import pytest

from tds_b200.model import inertial_parameters, param_names, param_values, regressor_names, set_param_values
import emu_invdyn as ei
import emu_kin
import emu_mass
import emu_regressor as er
from test_mass_matrix_on_host import fixture, f32
from test_params_on_host import all_ids, perturbed
from test_kinematics_on_host import quat_matrix
from test_point_motion_on_host import dq_dt

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "humanoid_fixed",
            "pendulum5spherical", "humanoid_spherical", "mb_three_bodies", "mb_racket"]
ORACLE = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "humanoid_fixed"]
FIXED_1DOF = ["pendulum5", "cartpole", "cartpole_plane", "laikago", "humanoid_fixed"]


def close(a, ref, tol):
    return np.all(np.abs(a - ref) <= tol * np.maximum(1.0, np.abs(ref)))


def state(model, n, seed=3):
    """fp32-exact qd, qdd [n, n_qd]."""
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return f32(rng.normal(size=(n, nd)) * 0.7), f32(rng.normal(size=(n, nd)))


def with_springs(model, seed=11):
    """The model with nonzero stiffness and damping on every joint, so that their columns are exercised at the model's values too."""
    ids = [i for i, nm in enumerate(param_names(model)) if nm.endswith(("stiffness", "damping"))]
    rng = np.random.default_rng(seed)
    return set_param_values(model, ids, rng.uniform(0.1, 2.0, len(ids)))


@pytest.mark.parametrize("name", FIXTURES)
def test_torque_regressor_times_model_parameters_is_inverse_dynamics(name):
    """Y pi = ID at the model's values, with qd and / or qdd NULL too; every entry is written (the buffers start as NaN)."""
    model, q = fixture(name)
    model = with_springs(model)
    q = f32(q)
    qd, qdd = state(model, q.shape[0])
    pi = inertial_parameters(model)
    assert len(regressor_names(model)) == pi.size == er.n_pi(model)
    for a, b in ((qd, qdd), (None, qdd), (qd, None), (None, None)):
        Y, yT, yV = er.regressor(model, q, a, b, fill=np.nan)
        assert np.all(np.isfinite(Y)) and np.all(np.isfinite(yT)) and np.all(np.isfinite(yV)), name
        tau = ei.inverse_dynamics(model, q, a, b)
        assert close(Y @ pi, tau, 1e-10), (name, np.abs(Y @ pi - tau).max())


@pytest.mark.parametrize("name", FIXTURES)
def test_torque_regressor_at_installed_parameter_sets(name):
    """Y pi = ID with a +-20 % per-environment set of every inertial, stiffness and damping id installed for ID, pi from the same set."""
    model, q = fixture(name)
    q = f32(q)
    n = q.shape[0]
    qd, qdd = state(model, n)
    ids = [i for i in all_ids(model) if i >= 2]
    vals = perturbed(model, ids, n, 5, 0.5, 0.0)
    pi = inertial_parameters(model, ids, vals)
    Y, _, _ = er.regressor(model, q, qd, qdd)
    tau = ei.inverse_dynamics(model, q, qd, qdd, ids=ids, values=vals)
    got = np.einsum("erc,ec->er", Y, pi)
    assert close(got, tau, 1e-10), (name, np.abs(got - tau).max())


@pytest.mark.parametrize("name", ORACLE)
def test_columns_against_the_oracle_rnea(name):
    """Each inertial column of Y is the C oracle's link-frame RNEA (tests/cpp/oracle_invdyn.c) of the model with every body and spring
    zero but that one unit barycentric parameter.  The oracle takes (m, com, I about the com): a unit m or unit I about the origin is such
    a body with m = 0 where needed; a unit first moment is, by linearity, a unit mass at com e_k with I_com = -(1 - e_k e_k^T) (so that
    its I about the origin is zero) minus a unit mass at the origin.  Independent of the kernel's common-frame arithmetic.  The stiffness
    and damping columns are checked by the ID comparisons above."""
    model, q = fixture(name)
    q = f32(q)
    qd, qdd = state(model, q.shape[0])
    nl = int(model[1])
    Y, _, _ = er.regressor(model, q[:2], qd[:2], qdd[:2])
    names = param_names(model)
    body_ids = list(range(2, 2 + 10 * (nl + 1)))
    zero = set_param_values(model, body_ids + [i for i, nm in enumerate(names) if nm.endswith(("stiffness", "damping"))],
                            np.zeros(len(body_ids) + 2 * nl))
    for col in range(10 * (nl + 1)):
        b, c = divmod(col, 10)
        if b == 0 and not int(model[2]):
            assert np.all(Y[:, :, col] == 0.0)
            continue
        vals = np.zeros(10)
        if c == 0:
            vals[0] = 1.0
            tau = [ei.oracle(set_param_values(zero, range(2 + 10 * b, 12 + 10 * b), vals), q[e], qd[e], qdd[e]) for e in range(2)]
        elif c < 4:
            com = np.zeros(3)
            com[c - 1] = 1.0
            Io = np.eye(3) - np.outer(com, com)
            v1 = np.concatenate([[1.0], com, [-Io[0, 0], -Io[0, 1], -Io[0, 2], -Io[1, 1], -Io[1, 2], -Io[2, 2]]])
            v0 = np.zeros(10)
            v0[0] = 1.0
            t1 = [ei.oracle(set_param_values(zero, range(2 + 10 * b, 12 + 10 * b), v1), q[e], qd[e], qdd[e]) for e in range(2)]
            t0 = [ei.oracle(set_param_values(zero, range(2 + 10 * b, 12 + 10 * b), v0), q[e], qd[e], qdd[e]) for e in range(2)]
            tau = [x - y for x, y in zip(t1, t0)]
        else:
            vals[c] = 1.0
            tau = [ei.oracle(set_param_values(zero, range(2 + 10 * b, 12 + 10 * b), vals), q[e], qd[e], qdd[e]) for e in range(2)]
        tau = np.array(tau)
        assert close(Y[:, :, col], tau, 1e-12), (name, regressor_names(model)[col], np.abs(Y[:, :, col] - tau).max())


@pytest.mark.parametrize("name", ["pendulum5", "humanoid", "laikago", "humanoid_spherical", "mb_racket"])
def test_outputs_do_not_depend_on_installed_parameters(name):
    """Y, yT and yV do not read the model's inertial, stiffness or damping values: they are bitwise equal at a perturbed model.  (The
    C-ABI's outputs with and without an installed set are compared bitwise on the GPU.)"""
    model, q = fixture(name)
    q = f32(q)
    qd, qdd = state(model, q.shape[0])
    ids = [i for i in all_ids(model) if i >= 2]
    other = set_param_values(model, ids, perturbed(model, ids, 1, 9, 0.5, 0.0)[0])
    a = er.regressor(model, q, qd, qdd, concat=True)
    b = er.regressor(other, q, qd, qdd, concat=True)
    assert np.array_equal(a, b), name


@pytest.mark.parametrize("name", FIXTURES)
def test_kinetic_energy(name):
    """yT pi = 1/2 qd^T M qd with M of the mass-matrix instances (section 7.12), fixed and floating bases."""
    model, q = fixture(name)
    q = f32(q)
    qd, _ = state(model, q.shape[0])
    _, yT, _ = er.regressor(model, q, qd)
    M = emu_mass.mass(model, q)
    T = 0.5 * np.einsum("ei,eij,ej->e", qd, M, qd)
    got = yT @ inertial_parameters(model)
    assert close(got, T, 1e-10), (name, np.abs(got - T).max())


@pytest.mark.parametrize("name", FIXTURES)
def test_potential_energy(name):
    """yV pi = -sum_b m_b g . x_com,b + 1/2 k q^2 (1/2 k |axis-angle|^2), the com positions from the kinematics instances (section 7.13)
    at local = com, the base's from q."""
    model, q = fixture(name)
    model = with_springs(model)
    q = f32(q)
    n, nl = q.shape[0], int(model[1])
    _, _, yV = er.regressor(model, q)
    pv = param_values(model)
    g = np.array(er.GRAVITY)
    lk = list(range(nl))
    local = np.array([pv[2 + 10 * (i + 1) + 1:2 + 10 * (i + 1) + 4] for i in range(nl)])
    _, x, _ = emu_kin.kinematics(model, q, lk, local)
    V = np.zeros(n)
    for i in range(nl):
        V -= pv[2 + 10 * (i + 1)] * (x[:, i] @ g)
    if int(model[2]):
        for e in range(n):
            xb = quat_matrix(*q[e, :4]) @ pv[3:6] + q[e, 4:7]
            V[e] -= pv[2] * (xb @ g)
    # spring terms from the stiffness columns' own definition (q, or the axis-angle vector): 1/2 k |s|^2 with s from Y's stiffness column
    Y, _, _ = er.regressor(model, q)
    pi = inertial_parameters(model)
    j0 = 10 * (nl + 1)
    for i in range(nl):
        s = Y[:, :, j0 + 2 * i]   # q, or the axis-angle vector, in the joint's rows only
        V += 0.5 * pi[j0 + 2 * i] * np.sum(s * s, axis=1)
    got = yV @ pi
    assert close(got, V, 1e-10), (name, np.abs(got - V).max())


@pytest.mark.parametrize("name", FIXED_1DOF)
def test_gravity_is_the_gradient_of_the_potential_energy(name):
    """On 1-dof fixed bases the rate of V = yV . pi along the motion with velocity v is v^T ID(q, 0, 0): generalised gravity (and, with
    the model's springs, the spring term).  The tangent of q is dq/dt, which differs from v on joints about a non-unit axis (the kernel
    turns them by q about the normalised axis while S = R a keeps |a|); those models are checked without springs, whose term k q is not
    scaled by |a|."""
    model, q = fixture(name)
    if name != "humanoid_fixed":
        model = with_springs(model)
    q = f32(q)
    n, nd = q.shape[0], int(model[4])
    v = np.random.default_rng(2).normal(size=(n, nd))
    tq = np.array([dq_dt(model, q[e], v[e]) for e in range(n)])
    t_in = np.concatenate([tq, np.zeros((n, 2 * nd))], axis=1)[:, :, None]
    _, _, dyV = er.split(er.regressor_jvp(model, q, t_in), model)
    got = dyV[..., 0] @ inertial_parameters(model)
    ref = np.einsum("ei,ei->e", v, ei.inverse_dynamics(model, q))
    assert close(got, ref, 1e-10), (name, np.abs(got - ref).max())


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_fixed", "pendulum5spherical",
                                  "humanoid_spherical", "mb_racket"])
def test_jvp_against_central_differences(name):
    """The JVP along q, qd and qdd, each alone, against central differences of the value in fp64 (the fp32 rounding of the inputs is
    avoided by a step that keeps every perturbed input fp32-exact: differences of the emulated value at h = 2^-10 on fp32-exact states)."""
    model, q = fixture(name)
    q = f32(q[:2])
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    rng = np.random.default_rng(4)
    h = 2.0 ** -10
    for part in range(3):
        dims = (n_q, nd, nd)[part]
        d = np.zeros((n, n_q + 2 * nd))
        lo = (0, n_q, n_q + nd)[part]
        # a single coordinate per environment keeps q + h d on the fp32 grid; quaternions are not renormalised by the kernels
        k = rng.integers(0, dims, n)
        d[np.arange(n), lo + k] = 1.0
        jv = er.regressor_jvp(model, q, d[:, :, None], qd, qdd)[..., 0]
        x = np.concatenate([q, qd, qdd], axis=1)
        f = lambda z: er.regressor(model, z[:, :n_q], z[:, n_q:n_q + nd], z[:, n_q + nd:], concat=True)
        fd = (f(x + h * d) - f(x - h * d)) / (2 * h)
        scale = np.maximum(1.0, np.abs(jv))
        assert np.all(np.abs(jv - fd) <= 1e-4 * scale), (name, part, np.abs(jv - fd).max())


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "humanoid_spherical"])
def test_tangents_are_independent(name):
    """m tangents in one call are bitwise the m single-tangent calls."""
    model, q = fixture(name)
    q = f32(q[:3])
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    t = np.random.default_rng(6).normal(size=(n, n_q + 2 * nd, 3))
    all3 = er.regressor_jvp(model, q, t, qd, qdd)
    for j in range(3):
        one = er.regressor_jvp(model, q, t[:, :, j:j + 1], qd, qdd)
        assert np.array_equal(all3[..., j], one[..., 0]), (name, j)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_vjp_duality(name):
    """<G, J v> = <VJP(G), v>."""
    model, q = fixture(name)
    q = f32(q[:2])
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    rng = np.random.default_rng(8)
    v = rng.normal(size=(n, n_q + 2 * nd, 1))
    G = rng.normal(size=(n, sum(er.rows(model))))
    jv = er.regressor_jvp(model, q, v, qd, qdd)[..., 0]
    g = er.regressor_vjp(model, q, G, qd, qdd)
    lhs = np.einsum("er,er->e", G, jv)
    rhs = np.einsum("ei,ei->e", g, v[..., 0])
    assert close(lhs, rhs, 1e-10), (name, lhs, rhs)


def test_helpers():
    """inertial_parameters of a set equals that of the model with the set applied; the names follow the parameter ids."""
    model, _ = fixture("humanoid")
    ids = [i for i in all_ids(model) if i >= 2]
    vals = perturbed(model, ids, 3, 1, 0.5, 0.0)
    pi = inertial_parameters(model, ids, vals)
    for e in range(3):
        ref = inertial_parameters(set_param_values(model, ids, vals[e]))
        assert np.allclose(pi[e], ref, rtol=0, atol=1e-15)
    names = regressor_names(model)
    pn = param_names(model)[2:]
    assert names[0] == "base.m" and names[14] == "link0.Ixx" and names[-1] == pn[-1] and names[-2] == pn[-2]
    with pytest.raises(ValueError):
        inertial_parameters(model, [0], [[0.5]])
