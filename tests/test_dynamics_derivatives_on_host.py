"""The derivatives d tau / dq and d tau / dqd of the inverse dynamics (DESIGN.md section 7.23) on the CPU, from the kernel SOURCE: the DER
instances of csrc/tds_stepw.cu compiled for the host (tests/cpp/dynamics_derivatives_host.cpp, bound by tests/emu_dynamics_derivatives.py)
on the thirteen mass-matrix fixtures, against the host INV build's JVP along dq_dt tangents, the host MASS JVP, C qd of the host COR build
and identities of the equation of motion; worlds of several multibodies, installed parameters, and the JVP against central differences of
the fp64 instance.  tests/test_dynamics_derivatives_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

import emu_coriolis as ecor
import emu_dynamics_derivatives as ed
import emu_invdyn
import emu_mass
from test_coriolis_on_host import christoffel_fixtures
from test_inverse_dynamics_on_host import without_springs
from test_mass_matrix_on_host import BASE, HEADER, LINK, ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture
from test_params_on_host import all_ids, perturbed
from tds_b200.model import param_names, param_values, set_param_values
from test_point_motion_on_host import dq_dt, grid_state

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
N = 3


def state(model, q, seed=1):
    """The fixture's first N configurations and random velocities and accelerations [N, n_qd], all fp32."""
    q = f32(q[:N])
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return q, f32(rng.normal(size=(q.shape[0], nd))), f32(rng.normal(size=(q.shape[0], nd)))


def tangent_basis(model, q):
    """dq_dt(q, e_k) for every k: [n, n_q, n_qd]."""
    nd = int(model[4])
    return np.stack([np.stack([dq_dt(model, a, e) for e in np.eye(nd)], axis=1) for a in q])


def close(a, ref, tol):
    err = np.abs(a - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= tol, err


@pytest.mark.parametrize("name", ALL)
def test_columns_equal_the_inverse_dynamics_jvp(name):
    """Column k of d tau / dq is the INV JVP along dq_dt(q, e_k), column k of d tau / dqd the INV JVP along e_k (the host builds)."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    dq, dqd = ed.inverse_dynamics_derivatives(model, q, qd, qdd)
    t = np.zeros((n, n_q + 2 * nd, 2 * nd))
    t[:, :n_q, :nd] = tangent_basis(model, q)
    t[:, n_q:n_q + nd, nd:] = np.eye(nd)
    J = emu_invdyn.inverse_dynamics_jvp(model, q, qd, qdd, t_in=t)
    close(dq, J[:, :, :nd], 1e-10)
    close(dqd, J[:, :, nd:], 1e-10)


@pytest.mark.parametrize("name", ALL)
def test_the_qdd_part_of_d_tau_dq_is_the_mass_matrix_rate(name):
    """d tau / dq (q, qd, qdd) - d tau / dq (q, qd, 0) = (dM along dq_dt(q, e_k)) qdd: the host MASS JVP."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    a, _ = ed.inverse_dynamics_derivatives(model, q, qd, qdd)
    b, _ = ed.inverse_dynamics_derivatives(model, q, qd)
    dM = emu_mass.mass_jvp(model, q, t_q=tangent_basis(model, q))   # [n, nd, nd, nd]: dM_rc along column k
    close(a - b, np.einsum("erck,ec->erk", dM, qdd), 1e-10)


@pytest.mark.parametrize("name", ALL)
def test_d_tau_dqd_does_not_depend_on_qdd(name):
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    close(ed.inverse_dynamics_derivatives(model, q, qd, qdd)[1], ed.inverse_dynamics_derivatives(model, q, qd)[1], 1e-12)


@pytest.mark.parametrize("name", ALL)
def test_d_tau_dqd_times_qd_is_twice_the_velocity_bias(name):
    """Without damping, d tau / dqd . qd = 2 C qd (the host COR build) = 2 (h(q, qd) - h(q, 0)) (the host INV build): h is quadratic in qd."""
    model, q = fixture(name)
    q, qd, _ = state(model, q)
    m0 = without_springs(model)
    _, dqd = ed.inverse_dynamics_derivatives(m0, q, qd)
    v = np.einsum("erc,ec->er", dqd, qd)
    close(v, 2 * np.einsum("erc,ec->er", ecor.coriolis(m0, q, qd), qd), 1e-10)
    close(v, 2 * (emu_invdyn.inverse_dynamics(m0, q, qd) - emu_invdyn.inverse_dynamics(m0, q)), 1e-10)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "pendulum5spherical", "humanoid_fixed", "laikago", "humanoid_spherical"])
def test_damping_adds_its_diagonal(name):
    """Installing every joint's damping at d adds d (exact in fp32) to the diagonal of d tau / dqd at each joint dof, within one rounding
    of the entry, and nothing else: the floating base's dofs and every off-diagonal entry are bitwise unchanged."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm.endswith(".damping")]
    n, nd = q.shape[0], int(model[4])
    d = 0.375
    _, a = ed.inverse_dynamics_derivatives(model, q, qd, qdd, ids=ids, values=np.full((n, len(ids)), d))
    _, b = ed.inverse_dynamics_derivatives(model, q, qd, qdd, ids=ids, values=np.zeros((n, len(ids))))
    off = ~np.eye(nd, dtype=bool)
    assert np.array_equal(a[:, off], b[:, off])
    want = np.full(nd, d)
    want[:6 if int(model[2]) else 0] = 0.0
    da, db = np.diagonal(a, axis1=1, axis2=2), np.diagonal(b, axis1=1, axis2=2)
    assert np.all(np.abs((da - db) - want) <= np.spacing(np.maximum(np.abs(da), d))), np.abs((da - db) - want).max()


@pytest.mark.parametrize("name", christoffel_fixtures())
def test_d_tau_dq_at_rest_is_the_hessian_of_the_potential(name):
    """At qd = qdd = 0 on fixed bases with one-dof joints, tau = dV/dq and d tau / dq is symmetric."""
    model, q = fixture(name)
    q, _, _ = state(model, q)
    dq, _ = ed.inverse_dynamics_derivatives(model, q)
    close(dq, dq.transpose(0, 2, 1), 1e-12)


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_worlds_give_exact_zeros_between_multibodies(name):
    """Entries coupling two multibodies of a world (one root link each, their dofs in order) are exact zeros."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
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
    for X in ed.inverse_dynamics_derivatives(model, q, qd, qdd):
        assert np.all(X[:, between] == 0)
        assert np.any(X[:, ~between] != 0)


@pytest.mark.parametrize("name", ["pendulum5", "box", "laikago", "humanoid_spherical"])
def test_parameters(name):
    """A set installed at the model's values is bitwise equal to no set; per-environment values equal the edited flat models."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    ids = [i for i in all_ids(model) if i >= 2]   # (friction and restitution do not enter)
    base = ed.inverse_dynamics_derivatives(model, q, qd, qdd)
    same = ed.inverse_dynamics_derivatives(model, q, qd, qdd, ids=ids, values=param_values(model)[ids])
    assert all(np.array_equal(a, b) for a, b in zip(base, same))
    vals = perturbed(model, ids, q.shape[0], 5, 0.2, 0.0)
    got = ed.inverse_dynamics_derivatives(model, q, qd, qdd, ids=ids, values=vals)
    for e in range(q.shape[0]):
        ref = ed.inverse_dynamics_derivatives(set_param_values(model, ids, vals[e]), q[e:e + 1], qd[e:e + 1], qdd[e:e + 1])
        for a, b in zip(got, ref):
            assert np.array_equal(a[e], b[0]), e


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "sphere2", "humanoid", "pendulum5spherical", "humanoid_spherical",
                                  "mb_three_bodies"])
def test_jvp_against_central_differences(name):
    """Along q (in n_q coordinates), qd, qdd and the parameters separately, the JVP of both matrices against central differences of the
    fp64 instance at h = 2^-10.  q, qd and qdd sit on grids that keep x +- h v exact in fp32 (the instance rounds them); the parameters
    are fp64 inputs.  Along q and the parameters the truncation error bounds the tolerance; along qd and qdd (the matrices are at most
    linear in them) only rounding is left."""
    model, q = fixture(name)
    q, qd, qdd = grid_state(model, q, 23)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = [i for i in all_ids(model) if i >= 2]
    p0 = np.tile(param_values(model)[ids], (n, 1))
    h = 2.0 ** -10
    rng = np.random.default_rng(29)
    for part, dim, tol in ((0, n_q, 1e-4), (1, nd, 1e-9), (2, nd, 1e-9), (3, len(ids), 1e-6)):
        v = np.round(rng.normal(size=(n, dim)) * 16) / 16
        if part == 3:
            v = v * np.maximum(np.abs(p0), 1e-2)
        x = [q, qd, qdd, p0]
        xp, xm = list(x), list(x)
        xp[part], xm[part] = x[part] + h * v, x[part] - h * v
        if part < 3:
            assert np.array_equal(f32(xp[part]), xp[part]) and np.array_equal(f32(xm[part]), xm[part])
        P = ed.inverse_dynamics_derivatives(model, *xp[:3], ids=ids, values=xp[3])
        Mi = ed.inverse_dynamics_derivatives(model, *xm[:3], ids=ids, values=xm[3])
        t = [None] * 4
        t[part] = v[:, :, None]
        jv = ed.inverse_dynamics_derivatives_jvp(model, q, qd, qdd, *t, ids=ids, values=p0)
        for o in range(2):
            fd = (P[o] - Mi[o]) / (2 * h)
            err = np.abs(jv[o][..., 0] - fd).max() / max(1.0, np.abs(fd).max())
            assert err <= tol, (name, part, o, err)


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_columns_against_central_differences_of_the_oracle(name):
    """Column k of d tau / dq against central differences of the C oracle's link-frame RNEA along q +- h dq_dt(q, e_k) (a retraction
    with that first derivative), column k of d tau / dqd along qd +- h e_k, h = 1e-6."""
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    q, qd, qdd = q[:2], qd[:2], qdd[:2]
    nd = int(model[4])
    dq, dqd = ed.inverse_dynamics_derivatives(model, q, qd, qdd)
    T = tangent_basis(model, q)
    h = 1e-6
    for e in range(q.shape[0]):
        fq = np.stack([(emu_invdyn.oracle(model, q[e] + h * T[e, :, k], qd[e], qdd[e]) - emu_invdyn.oracle(model, q[e] - h * T[e, :, k], qd[e], qdd[e]))
                       / (2 * h) for k in range(nd)], axis=1)
        fqd = np.stack([(emu_invdyn.oracle(model, q[e], qd[e] + h * u, qdd[e]) - emu_invdyn.oracle(model, q[e], qd[e] - h * u, qdd[e])) / (2 * h)
                        for u in np.eye(nd)], axis=1)
        close(dq[e], fq, 1e-6)
        close(dqd[e], fqd, 1e-6)


@pytest.mark.parametrize("name", ["box", "humanoid_spherical"])
def test_m_tangents_in_one_call_equal_single_calls(name):
    model, q = fixture(name)
    q, qd, qdd = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    rng = np.random.default_rng(9)
    tq, tqd, tqdd = rng.normal(size=(n, n_q, 3)), rng.normal(size=(n, nd, 3)), rng.normal(size=(n, nd, 3))
    a, b = ed.inverse_dynamics_derivatives_jvp(model, q, qd, qdd, tq, tqd, tqdd)
    for j in range(3):
        a1, b1 = ed.inverse_dynamics_derivatives_jvp(model, q, qd, qdd, tq[..., j:j + 1], tqd[..., j:j + 1], tqdd[..., j:j + 1])
        assert np.array_equal(a[..., j], a1[..., 0]) and np.array_equal(b[..., j], b1[..., 0])


def test_argument_checks():
    """Every entry point returns -1 without a simulator (before any device work, so on a machine without a GPU too); the host build
    rejects parameter ids the model does not have."""
    import ctypes
    import tds_b200
    L = tds_b200.lib()
    z = None
    assert L.tds_b200_inverse_dynamics_derivatives_device(z, z, z, z, z, z, z) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_host(z, z, z, z, z, z) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_jvp_device(z, z, z, z, 1, z, z, z, z, z, z, z, z, z) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_jvp_host(z, z, z, z, 1, z, z, z, z, z, z, z, z) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_vjp_device(z, z, z, z, z, z, z, z, z, z, z) == -1
    assert L.tds_b200_inverse_dynamics_derivatives_vjp_host(z, z, z, z, z, z, z, z, z, z) == -1
    model, q = fixture("pendulum5")
    with pytest.raises(ValueError):
        ed.inverse_dynamics_derivatives(model, f32(q[:1]), ids=[0, 0], values=np.zeros((1, 2)))
    with pytest.raises(ValueError):
        ed.inverse_dynamics_derivatives(model, f32(q[:1]), ids=[2], values=np.zeros((1, 1)))   # a base id on a fixed base
