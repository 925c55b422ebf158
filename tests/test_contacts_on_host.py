"""The step that reports its contacts (DESIGN.md section 7.15) on the CPU, from the kernel SOURCE: the CF instances of csrc/tds_stepw.cu
compiled for the host (tests/cpp/contacts_host.cpp, bound by tests/emu_contacts.py).  q' and qd' against the host-built step without CF
(bitwise), the impulses against the mass matrix and the point Jacobians (sections 7.12, 7.13) that share no code with the contact
records, the geometry against the contact distances, complementarity, an analytic case, the derivatives and installed parameters.
tests/test_contacts_gpu.py checks the same instances as nvcc builds them."""
import ctypes

import numpy as np
import pytest

import emu
import emu_contacts
import emu_kin
import emu_mass
from oracle import port
from test_mass_matrix_on_host import BASE, HEADER, LINK, f32, fixture
from tds_b200.model import param_ids, param_names, param_values
from test_params_on_host import all_ids

CONTACT_FIXTURES = ["sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "humanoid_spherical", "mb_three_bodies", "mb_racket"]
ORACLE_CONTACT_FIXTURES = ["sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid"]   # single multibodies the C oracle steps
NBODIES, SPHERICAL = 12, 8   # TDSM_H_NBODIES, TDSJ_SPHERICAL (include/tds_b200_model.h)
LAIKAGO_ENV = (12, 6, 100.0, 2.0, 50.0, 0.4) + (0.0, 0.67, -1.25) * 4


def state(name, n=6):
    """(model, q, qd, tau) of a fixture: its golden inputs, torques zero."""
    model, q = fixture(name)
    g = np.load(emu.os.path.join(emu.HERE, "golden", name + ".npz"))
    qd = g["qd_in"][:q.shape[0]][:n]
    n_tau = int(model[4]) - (6 if int(model[2]) else 0)
    return model, q[:n], qd, np.zeros((q[:n].shape[0], n_tau))


def candidates(model):
    """(body_a, link_a, body_b, link_b) per contact candidate, from the C-ABI's host-only candidate table."""
    from tds_b200 import _lib
    m = np.ascontiguousarray(model, dtype=np.float64)
    t = np.zeros((128, 4), dtype=np.int32)
    k = _lib.lib().tds_b200_model_contact_pairs(m.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), m.size, ctypes.c_void_p(t.ctypes.data), 128)
    assert k >= 0
    return t[:k]


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("name", CONTACT_FIXTURES)
def test_q_and_qd_bitwise_equal_to_the_step(name, precision):
    model, q, qd, tau = state(name)
    for mode in (2, 3):
        qo, qdo, C = emu_contacts.step_contacts(model, mode, q, qd, tau, precision=precision)
        ref = emu.step(model, mode, q, qd, tau, precision=precision)
        assert np.array_equal(qo, ref["q"]) and np.array_equal(qdo, ref["qd"])
        assert C.shape == (q.shape[0], ref["contact_dist"].shape[1], 10)
        # the distance row is the step's contact_dist (+inf where a contact function emitted no point)
        assert np.array_equal(C[:, :, 6], ref["contact_dist"])


def test_laikago_with_pd_bitwise_equal_to_the_step():
    model, q, qd, _ = state("laikago")
    act = np.random.default_rng(3).uniform(-0.3, 0.3, size=(q.shape[0], 12))
    for p in (0, 1, 2):
        qo, qdo, _ = emu_contacts.step_contacts(model, 2, q, qd, act, precision=p, use_pd=True, env=LAIKAGO_ENV)
        ref = emu.step(model, 2, q, qd, act, precision=p, use_pd=True, env=LAIKAGO_ENV)
        assert np.array_equal(qo, ref["q"]) and np.array_equal(qdo, ref["qd"])


def _world_to_local(model, q, link, p):
    """p (world) in the frame of `link` (-1: the base) at q, as the point table of the kinematics takes it."""
    if link >= 0:
        xf, _, _ = emu_kin.kinematics(model, q[None], [0], np.zeros(3))
        R, t = xf[0, link, :9].reshape(3, 3), xf[0, link, 9:]
    elif int(model[2]):
        x, y, z, w = f32(q[:4])
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        t = f32(q[4:7])
    else:
        R, t = np.eye(3), np.zeros(3)
    return R.T @ (p - t)


def _links(model):
    """(parent, joint type, qd index) of every link of a flat model."""
    n_links = int(model[1])
    L = np.asarray(model[HEADER + BASE:HEADER + BASE + n_links * LINK]).reshape(n_links, LINK)
    return L[:, 0].astype(int), L[:, 1].astype(int), L[:, 3].astype(int)


def _world_link(model, body, link):
    """The model's link index of link `link` of multibody `body` (bodies 1, 2, ... of the world; every root link starts one)."""
    if int(model[NBODIES]) <= 1 or link < 0:
        return link
    roots = [i for i, p in enumerate(_links(model)[0]) if p < 0]
    return roots[body - 1] + link


def _generalized_impulse(model, q, C, cand):
    """(sum_c J_b(point on b)^T F_c - J_a(point on a)^T F_c, sum_c |J_b|^T |F_c| + |J_a|^T |F_c|) of every environment, with the point
    Jacobians of the kinematics build (the second term: the magnitude the fp32 rounding of F enters with)."""
    n, nd = q.shape[0], int(model[4])
    out, mag = np.zeros((n, nd)), np.zeros((n, nd))
    for e in range(n):
        for k in range(C.shape[1]):
            F = C[e, k, 7:10]
            if not np.any(F):
                continue
            nb, xb, d = C[e, k, 0:3], C[e, k, 3:6], C[e, k, 6]
            for body, link, p, sgn in ((cand[k, 2], cand[k, 3], xb, 1.0), (cand[k, 0], cand[k, 1], xb + d * nb, -1.0)):
                if body == 0:
                    continue   # the plane (body 0) has no dofs
                gl = _world_link(model, body, link)
                if gl < 0 and not int(model[2]):
                    continue   # a fixed base has no dofs
                _, _, J = emu_kin.kinematics(model, q[e][None], [gl], _world_to_local(model, q[e], gl, p))
                out[e] += sgn * J[0, 0].T @ F
                mag[e] += np.abs(J[0, 0]).T @ np.abs(F)
    return out, mag


def _spherical_dofs(model):
    parent, jtype, qd_idx = _links(model)
    return [int(qd_idx[i]) + a for i in range(len(parent)) if jtype[i] == SPHERICAL for a in range(3)]


def _identity_residual(model, q, qd_full, qd_nc, C, dt=1e-3):
    """(|M (qd'_FULL - qd'_NOCONTACT) - sum_c (J_b - J_a)^T F_c| max, scale): qd' of spherical dofs carries the integrator's damping factor
    0.995^(1000 dt), divided out here.  scale = max(1, max_e sum_j |M_ij| (|qd'_FULL| + |qd'_NOCONTACT|)_j + (|J|^T |F|)_i): the sizes whose
    fp32 roundings (qd' and the records are fp32) enter the two sides."""
    M = emu_mass.mass(model, q)
    dq = qd_full - qd_nc
    sph = _spherical_dofs(model)
    if sph:
        dq[:, sph] /= 0.995 ** (1000.0 * dt)
    lhs = np.einsum("eij,ej->ei", M, dq)
    rhs, mag = _generalized_impulse(model, f32(q), C, candidates(model))
    assert np.any(C[:, :, 7:10]), "the case has active contacts"
    scale = max(1.0, float(np.max(np.einsum("eij,ej->ei", np.abs(M), np.abs(qd_full) + np.abs(qd_nc)) + mag)))
    return float(np.abs(lhs - rhs).max()), scale


IDENTITY_CASES = [(name, 1, False) for name in CONTACT_FIXTURES] + [("laikago", 1, True)] + \
    [(name, p, False) for name in ("sphere2", "laikago") for p in (0, 2)] + [("laikago", 0, True), ("laikago", 2, True)]


@pytest.mark.parametrize("name,precision,pd", IDENTITY_CASES)
def test_impulse_identity_with_the_mass_matrix(name, precision, pd):
    """M (qd'_FULL - qd'_NOCONTACT) = sum_c J_b^T F - J_a^T F: the contact solve's own update qd -= M^-1 (J_b - J_a)^T p, checked with M
    from the MASS build and J from the KIN build at the records' points (candidates between multibodies mapped to the world's links).
    Within 2e-5 scale at every precision checked: fp64 on every fixture; fp32 and mixed, which factor M in fp32 (the update then carries
    M's conditioning times the fp32 epsilon, which exceeds the bound on the humanoid), on Laikago and sphere2 only."""
    model, q, qd, tau = state(name)
    kw = dict(use_pd=True, env=LAIKAGO_ENV) if pd else {}
    if pd:
        tau = np.random.default_rng(3).uniform(-0.3, 0.3, size=(q.shape[0], 12))
    _, qd_full, C = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=precision, **kw)
    qd_nc = emu.step(model, 1, q, qd, tau, precision=precision, **kw)["qd"]
    res, scale = _identity_residual(model, q, qd_full, qd_nc, C)
    assert res <= 2e-5 * scale, (res, scale)


@pytest.mark.parametrize("name", ["sphere2", "laikago"])
def test_impulse_identity_of_the_spring_damper_model(name):
    model, q, qd, tau = state(name)
    kw = dict(contact_model=1)
    _, qd_full, C = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=1, **kw)
    qd_nc = emu.step(model, 1, q, qd, tau, precision=1, **kw)["qd"]
    res, scale = _identity_residual(model, q, qd_full, qd_nc, C)
    assert res <= 2e-5 * scale, (res, scale)


@pytest.mark.parametrize("name", ORACLE_CONTACT_FIXTURES)
def test_impulse_identity_against_the_c_oracle(name):
    """The identity with the C oracle's qd' (tdso_step FULL against NOCONTACT at the same fp32-rounded inputs, fp64 throughout): ties the
    records' impulses to an implementation that shares no code with the kernel."""
    model, q, qd, tau = state(name)
    _, _, C = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=1)
    P = port.make_params()
    full = np.array([port.step(model, P, 2, a, b, t)["qd"] for a, b, t in zip(f32(q), f32(qd), tau)])
    nc = np.array([port.step(model, P, 1, a, b, t)["qd"] for a, b, t in zip(f32(q), f32(qd), tau)])
    res, scale = _identity_residual(model, q, full, nc, C)
    assert res <= 2e-5 * scale, (res, scale)


@pytest.mark.parametrize("name", ORACLE_CONTACT_FIXTURES)
def test_geometry_against_the_c_oracle(name):
    """For every contact the oracle keeps (distance < 0), the normal on b, the point on b, the point on a reconstructed as point_on_b +
    distance * normal_on_b, and the distance equal the oracle's contact_data at the same fp32-rounded inputs within fp32 rounding.  The
    oracle lists every candidate in candidate order; its contact_idx names the same link b as the candidate table."""
    model, q, qd, tau = state(name)
    _, _, C = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=1)
    cand = candidates(model)
    P = port.make_params()
    kept = 0
    for e in range(q.shape[0]):
        o = port.step(model, P, 2, f32(q[e]), f32(qd[e]), tau[e])
        assert o["n_contacts"] == C.shape[1] == cand.shape[0]
        assert np.array_equal(o["contact_idx"][:, 1], cand[:, 3])
        for k in range(C.shape[1]):
            d = o["contact_data"][k]
            if d[9] >= 0:
                continue
            kept += 1
            nb, xb, dist = C[e, k, 0:3], C[e, k, 3:6], C[e, k, 6]
            tol = lambda x: 2e-6 * max(1.0, np.abs(x).max())
            assert np.abs(nb - d[0:3]).max() <= tol(d[0:3])
            assert np.abs(xb - d[6:9]).max() <= tol(d[6:9])
            assert np.abs(xb + dist * nb - d[3:6]).max() <= tol(d[3:6])
            assert abs(dist - d[9]) <= tol(d[9])
    assert kept > 0


def plane_space(n):
    """The friction directions of the solver for normal n (mb_constraint_solver.hpp:506-520, k = sqrt(a) as the reference evaluates it:
    not unit vectors in general)."""
    mz = n[2] * n[2] > 0.5
    a = n[1] * n[1] + (n[2] * n[2] if mz else n[0] * n[0])
    k = np.sqrt(a)
    p = np.array([0.0 if mz else -n[1] * k, -n[2] * k if mz else n[0] * k, n[1] * k])
    q = np.array([a * k if mz else -n[2] * p[1], -n[0] * p[2] if mz else n[2] * p[0], n[0] * p[1] if mz else a * k])
    return p, q


@pytest.mark.parametrize("name", CONTACT_FIXTURES)
def test_complementarity_and_inactive_candidates(name):
    """0 <= p_n <= 1e5, |p_1|, |p_2| <= mu p_n (the reference's box bound) and a zero impulse for every candidate outside the active set.
    p is recovered from F = -(p_n n_b + p_1 t_1 + p_2 t_2) with the solver's friction directions; the records are fp32."""
    model, q, qd, tau = state(name)
    _, _, C = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=1, friction=0.7)
    active = C[:, :, 6] < 0
    assert np.all(C[~active][:, 7:10] == 0.0)
    assert np.any(active)
    for e, k in zip(*np.nonzero(active)):
        nb = C[e, k, 0:3]
        t1, t2 = plane_space(nb)
        p = np.linalg.solve(np.stack([nb, t1, t2], axis=1), -C[e, k, 7:10])
        tol = 1e-5 * max(1.0, np.abs(p).max())
        assert -tol <= p[0] <= 1e5
        assert abs(p[1]) <= 0.7 * p[0] + tol and abs(p[2]) <= 0.7 * p[0] + tol, (e, k, p)


def test_analytic_sphere_pressed_into_the_plane():
    """Sphere2 at rest, pressed delta = 0.01 into the plane, identity orientation, qd = 0: p_n = (g dt + erp delta / dt) / (1/m + cfm)."""
    model, q, _, _ = state("sphere2", 1)
    n_qd = int(model[4])
    # place the sphere so that its single candidate has distance -0.01: shift along z by the distance found
    q1 = np.array(q, dtype=np.float64)
    q1[0, :4] = (0.0, 0.0, 0.0, 1.0)
    _, _, C = emu_contacts.step_contacts(model, 2, q1, np.zeros((1, n_qd)), precision=1)
    q1[0, 6] -= C[0, 0, 6] + 0.01
    _, _, C = emu_contacts.step_contacts(model, 2, q1, np.zeros((1, n_qd)), precision=1)
    delta = -C[0, 0, 6]
    assert abs(delta - 0.01) < 1e-6
    mass = model[HEADER + 0]   # the base's mass, first field of the base block
    dt, erp, cfm, g = 1e-3, 0.2, 1e-5, 9.81
    p_expected = (g * dt + erp * delta / dt) / (1.0 / mass + cfm)
    F = C[0, 0, 7:10]
    assert abs(F[2] - p_expected) <= 1e-5 * p_expected, (F, p_expected)
    assert F[0] == 0.0 and F[1] == 0.0


def _jvp_case(name):
    model, q, qd, tau = state(name, 4)
    n_q, n_qd = int(model[3]), int(model[4])
    cols = n_q + n_qd + tau.shape[1]
    return model, q, qd, tau, cols


@pytest.mark.parametrize("name", ["sphere2", "cartpole_plane", "laikago", "ant", "mb_three_bodies", "mb_racket"])
def test_jvp_against_central_differences_of_the_fp64_build(name):
    """The records' JVP against central differences (h = 1e-6) of the fp64 records of the same dual-number instance (its value parts),
    along a tangent of every input and of two installed parameters (friction and a mass), away from branch changes.  The inputs are
    loaded as fp32, so the differences are taken between the fp32 points x +- h v and compared with the JVP along their difference."""
    model, q, qd, tau, cols = _jvp_case(name)
    n, n_q, n_qd = q.shape[0], int(model[3]), int(model[4])
    ids = [0] + [i for i in all_ids(model) if param_names(model)[i].endswith(".mass")][:1]
    base = param_values(model)[ids]
    rng = np.random.default_rng(7)
    x0 = np.concatenate([f32(q), f32(qd), f32(tau)], axis=1)
    v, vp = rng.normal(size=x0.shape), rng.normal(size=(n, len(ids)))
    h = 1e-6
    xp, xm = f32(x0 + h * v), f32(x0 - h * v)
    split = lambda x: (x[:, :n_q], x[:, n_q:n_q + n_qd], x[:, n_q + n_qd:])
    Cp = emu_contacts.step_contacts_fp64(model, 2, *split(xp), ids=ids, values=base + h * vp)
    Cm = emu_contacts.step_contacts_fp64(model, 2, *split(xm), ids=ids, values=base - h * vp)
    fd = (Cp - Cm).reshape(n, -1) / (2 * h)
    t_in = ((xp - xm) / (2 * h))[:, :, None]
    t = emu_contacts.step_contacts_jvp(model, 2, *split(x0), t_in=t_in, t_par=vp[:, :, None], ids=ids, values=base)[:, n_q + n_qd:, 0]
    ok = np.isfinite(fd) & np.isfinite(t)
    assert np.any(t[ok] != 0.0)
    err = np.abs(fd[ok] - t[ok])
    assert err.max() <= 1e-5 * max(1.0, np.abs(t[ok]).max()), err.max()


@pytest.mark.parametrize("name", ["sphere2", "laikago", "mb_racket"])
def test_tangents_of_one_call_equal_single_calls(name):
    model, q, qd, tau, cols = _jvp_case(name)
    v = np.random.default_rng(2).normal(size=(q.shape[0], cols, 3))
    t = emu_contacts.step_contacts_jvp(model, 2, q, qd, tau, t_in=v)
    for j in range(3):
        assert np.array_equal(t[:, :, j], emu_contacts.step_contacts_jvp(model, 2, q, qd, tau, t_in=v[:, :, j:j + 1])[:, :, 0])


@pytest.mark.parametrize("name", ["sphere2", "laikago"])
def test_jvp_of_q_and_qd_rows_equals_the_step_jacobian(name):
    """The JVP's q' | qd' rows are the step's Jacobian (dual instance without CF) applied to the tangent."""
    model, q, qd, tau, cols = _jvp_case(name)
    v = np.random.default_rng(5).normal(size=(q.shape[0], cols, 1))
    t = emu_contacts.step_contacts_jvp(model, 2, q, qd, tau, t_in=v)[:, :, 0]
    Jm = emu.step(model, 2, q, qd, tau, jacobian=True)["jac"]
    nqq = int(model[3]) + int(model[4])
    assert np.allclose(t[:, :nqq], np.einsum("erc,ec->er", Jm, v[:, :, 0]), rtol=0, atol=1e-10)


def test_friction_derivative_on_a_saturated_sliding_contact():
    """Sliding sphere with saturated friction, one PGS sweep: dp_f / dmu = +-p_n along the friction row (parameter id 0 is friction)."""
    model, q, _, _ = state("sphere2", 1)
    n_q, n_qd = int(model[3]), int(model[4])
    q1 = np.array(q, dtype=np.float64)
    q1[0, :4] = (0.0, 0.0, 0.0, 1.0)
    _, _, C = emu_contacts.step_contacts(model, 2, q1, np.zeros((1, n_qd)), precision=1)
    q1[0, 6] -= C[0, 0, 6] + 0.005
    qd1 = np.zeros((1, n_qd))
    qd1[0, 3] = 2.0   # sliding along x
    ids = [param_ids(model, ["friction"])[0]]
    assert ids == [0]
    mu = param_values(model)[ids]
    _, _, C = emu_contacts.step_contacts(model, 2, q1, qd1, precision=1, ids=ids, values=mu)
    F = C[0, 0, 7:10]
    nb = C[0, 0, 0:3]
    p_n = -F @ nb
    ft = -F - nb * p_n
    assert np.linalg.norm(ft) > 0.99 * mu[0] * p_n   # saturated
    t = emu_contacts.step_contacts_jvp(model, 2, q1, qd1, None, t_par=np.ones((1, 1, 1)), ids=ids, values=mu)[:, :, 0]
    dF = t[0, n_q + n_qd + 7:n_q + n_qd + 10]
    dft = -dF - nb * (-dF @ nb)
    assert abs(np.linalg.norm(dft) - p_n) <= 1e-6 * max(1.0, p_n)


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("name", ["sphere2", "laikago", "humanoid", "mb_three_bodies"])
def test_installed_parameters_at_the_model_values_are_bitwise_equal(name, precision):
    model, q, qd, tau = state(name)
    ids = all_ids(model)
    vals = param_values(model)[ids]
    a = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=precision)
    b = emu_contacts.step_contacts(model, 2, q, qd, tau, precision=precision, ids=ids, values=vals)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
