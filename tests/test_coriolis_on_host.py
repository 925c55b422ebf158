"""The Coriolis matrix C(q, qd) (DESIGN.md section 7.22) on the CPU, from the kernel SOURCE: the COR instances of csrc/tds_stepw.cu compiled
for the host (tests/cpp/coriolis_host.cpp, bound by tests/emu_coriolis.py) on the thirteen mass-matrix fixtures, against the three
properties of the factorisation (C qd = h(q, qd) - h(q, 0) with the host INV build and the C oracle's RNEA, C + C^T = M' from the host
MASS JVP and from central differences of the oracle's M, the Christoffel form on fixed bases with one-dof joints), a NumPy restatement
of the defining sum from the point-motion Jacobians, linearity in qd, worlds of several multibodies, per-environment parameters and the
derivatives.  tests/test_coriolis_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_names, param_values, set_param_values
from oracle import port
import emu_coriolis as ecor
import emu_invdyn
import emu_kin
import emu_mass
import emu_point_motion as ep
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, f32, fixture
from test_inverse_dynamics_on_host import without_springs
from test_kinematics_on_host import links_of, quat_matrix
from test_params_on_host import all_ids, perturbed
from test_point_motion_on_host import SPHERICAL, dq_dt, grid_state

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
N = 4


def state(model, q, seed=1):
    """The fixture's first N configurations (fp32) and random velocities qd [N, n_qd] (fp32)."""
    q = f32(q[:N])
    rng = np.random.default_rng(seed)
    return q, f32(rng.normal(size=(q.shape[0], int(model[4]))))


def christoffel_fixtures():
    """The fixed-base fixtures whose joints all have one dof: there the velocities are the rates of (scaled) coordinates."""
    out = []
    for name in ALL:
        model, _ = fixture(name)
        if not int(model[2]) and not np.any(links_of(model)[:, 1] == SPHERICAL):
            out.append(name)
    return out


def path_rate(model, q, qd):
    """dq/dt [n, n_q, 1] of the motions with velocities qd."""
    return np.stack([dq_dt(model, a, b) for a, b in zip(q, qd)])[:, :, None]


def close(a, ref, tol):
    err = np.abs(a - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= tol, err


# ---- the three properties ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ALL)
def test_c_qd_is_the_velocity_part_of_the_bias_forces(name):
    """C qd = h(q, qd) - h(q, 0), h from the host INV build and (where it restates the model) the C oracle's RNEA, damping zeroed."""
    model, q = fixture(name)
    q, qd = state(model, q)
    C = ecor.coriolis(model, q, qd)
    Cq = np.einsum("eij,ej->ei", C, qd)
    m0 = without_springs(model)
    h = emu_invdyn.inverse_dynamics(m0, q, qd) - emu_invdyn.inverse_dynamics(m0, q)
    assert np.all(np.abs(Cq - h) <= 1e-10 * np.maximum(1.0, np.abs(h))), np.abs(Cq - h).max()
    if name in ORACLE_FIXTURES:
        ho = np.array([emu_invdyn.oracle(m0, a, b) - emu_invdyn.oracle(m0, a) for a, b in zip(q, qd)])
        assert np.all(np.abs(Cq - ho) <= 1e-10 * np.maximum(1.0, np.abs(ho))), np.abs(Cq - ho).max()


@pytest.mark.parametrize("name", ALL)
def test_c_plus_its_transpose_is_the_rate_of_the_mass_matrix(name):
    """C + C^T = M' along the motion with velocity qd: the host MASS JVP along dq/dt, and central differences of the oracle's M."""
    model, q = fixture(name)
    q, qd = state(model, q)
    C = ecor.coriolis(model, q, qd)
    S = C + C.transpose(0, 2, 1)
    t = path_rate(model, q, qd)
    Md = emu_mass.mass_jvp(model, q, t_q=t)[..., 0]
    assert np.abs(S - Md).max() <= 1e-12 * max(1.0, np.abs(Md).max()), np.abs(S - Md).max()
    if name in ORACLE_FIXTURES:
        h = 1e-6
        Mo = np.array([(port.mass_matrix(model, a + h * v[:, 0]) - port.mass_matrix(model, a - h * v[:, 0])) / (2 * h) for a, v in zip(q, t)])
        assert np.abs(S - Mo).max() <= 1e-6 * max(1.0, np.abs(Mo).max()), np.abs(S - Mo).max()


@pytest.mark.parametrize("name", christoffel_fixtures())
def test_christoffel_form_on_one_dof_fixed_bases(name):
    """C_ij = sum_k 1/2 (D_k M_ij + D_j M_ik - D_i M_jk) qd_k, D_k M the rate of M along unit velocity k: from the host MASS JVP and from
    central differences of the oracle's M."""
    model, q = fixture(name)
    q, qd = state(model, q)
    q, qd = q[:2], qd[:2]
    n, nd = q.shape[0], int(model[4])
    C = ecor.coriolis(model, q, qd)
    T = np.concatenate([path_rate(model, q, np.tile(np.eye(nd)[k], (n, 1))) for k in range(nd)], axis=2)
    dM = emu_mass.mass_jvp(model, q, t_q=T)                                          # [n, i, j, k] = D_k M_ij
    ref = 0.5 * (np.einsum("eijk,ek->eij", dM, qd) + np.einsum("eikj,ek->eij", dM, qd) - np.einsum("ejki,ek->eij", dM, qd))
    assert np.abs(C - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), np.abs(C - ref).max()
    if name in ORACLE_FIXTURES:
        h = 1e-6
        dMo = np.stack([np.stack([(port.mass_matrix(model, q[e] + h * T[e, :, k]) - port.mass_matrix(model, q[e] - h * T[e, :, k])) / (2 * h)
                                  for k in range(nd)], axis=2) for e in range(n)])
        refo = 0.5 * (np.einsum("eijk,ek->eij", dMo, qd) + np.einsum("eikj,ek->eij", dMo, qd) - np.einsum("ejki,ek->eij", dMo, qd))
        assert np.abs(C - refo).max() <= 1e-6 * max(1.0, np.abs(refo).max()), np.abs(C - refo).max()


# ---- the defining sum ---------------------------------------------------------------------------------------------------------------

def skew(p):
    return np.array([[0.0, -p[2], p[1]], [p[2], 0.0, -p[0]], [-p[1], p[0], 0.0]])


def crm(v):
    """v x (motion) as a 6 x 6 matrix, [w; u] order."""
    X = np.zeros((6, 6))
    X[:3, :3] = X[3:, 3:] = skew(v[:3])
    X[3:, :3] = skew(v[3:])
    return X


def crf(v):
    return -crm(v).T


def defining_sum(model, q, qd):
    """C = sum_i J_i^T (I_i J_i' + B(I_i, v_i) J_i) in NumPy: J_i the point-motion Jacobian at body i's origin moved to the world origin,
    J_i' its JVP along dq/dt, I_i the body's spatial inertia about the world origin in world axes."""
    nd = int(model[4])
    names = param_names(model)
    pv = param_values(model)
    lk = ([-1] if int(model[2]) else []) + list(range(int(model[1])))
    lc = np.zeros((len(lk), 3))
    J, vel, _ = ep.point_motion(model, q, lk, lc, qd)
    n_q = int(model[3])
    t_in = np.zeros((q.shape[0], n_q + 2 * nd, 1))
    t_in[:, :n_q] = path_rate(model, q, qd)
    dJ = ep.point_motion_jvp(model, q, lk, lc, t_in, qd)[..., 0]
    dJ = dJ[:, :6 * len(lk) * nd].reshape(q.shape[0], len(lk), 6, nd)
    xf, x, _ = emu_kin.kinematics(model, q, lk, lc)
    out = np.zeros((q.shape[0], nd, nd))
    for e in range(q.shape[0]):
        for b, l in enumerate(lk):
            r = pv[2 + 10 * (l + 1):12 + 10 * (l + 1)]
            assert names[2 + 10 * (l + 1)].endswith("mass")
            R = quat_matrix(*q[e, :4]) if l < 0 else xf[e, l, :9].reshape(3, 3)
            p, pd = x[e, b], vel[e, b, 3:]
            X = np.eye(6)
            X[3:, :3] = skew(p)                                # [w; v_p] -> [w; v_O], v_O = v_p + p x w
            Xd = np.zeros((6, 6))
            Xd[3:, :3] = skew(pd)
            Jb = X @ J[e, b]
            Jbd = Xd @ J[e, b] + X @ dJ[e, b]
            m, c = r[0], p + R @ r[1:4]
            Ic = R @ np.array([[r[4], r[5], r[6]], [r[5], r[7], r[8]], [r[6], r[8], r[9]]]) @ R.T
            I = np.zeros((6, 6))
            I[:3, :3] = Ic - m * skew(c) @ skew(c)
            I[:3, 3:] = m * skew(c)
            I[3:, :3] = -m * skew(c)
            I[3:, 3:] = m * np.eye(3)
            v = Jb @ qd[e]
            Iv = I @ v
            bar = np.stack([crf(np.eye(6)[k]) @ Iv for k in range(6)], axis=1)
            B = 0.5 * (crf(v) @ I + bar - I @ crm(v))
            out[e] += Jb.T @ (I @ Jbd + B @ Jb)
    return out


@pytest.mark.parametrize("name", ALL)
def test_the_defining_sum(name):
    """The sum over the bodies in NumPy from the host-built point motions: pins the skew part, which the properties leave free on floating
    bases and spherical joints."""
    model, q = fixture(name)
    q, qd = state(model, q)
    q, qd = q[:2], qd[:2]
    C = ecor.coriolis(model, q, qd)
    ref = defining_sum(model, q, qd)
    assert np.abs(C - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max()), np.abs(C - ref).max()


# ---- structure ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ALL)
def test_linear_in_qd(name):
    """C(q, 2 qd) = 2 C(q, qd) bitwise (every term is linear in qd), a C(q, x) + b C(q, y) = C(q, a x + b y) within round-off, and qd =
    NULL gives exact zeros."""
    model, q = fixture(name)
    q, x = state(model, q, 2)
    x, y = (np.round(np.random.default_rng(s).normal(size=x.shape) * 1024) / 1024 for s in (3, 4))
    Cx = ecor.coriolis(model, q, x)
    assert np.array_equal(ecor.coriolis(model, q, 2.0 * x), 2.0 * Cx)
    a, b = 0.75, -1.5
    z = a * x + b * y
    assert np.array_equal(f32(z), z)
    close(ecor.coriolis(model, q, z), a * Cx + b * ecor.coriolis(model, q, y), 1e-13)
    assert np.all(ecor.coriolis(model, q) == 0.0)


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_world_has_exact_zeros_between_multibodies(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    C = ecor.coriolis(model, q, qd)
    L = links_of(model)
    root = np.zeros(int(model[4]), dtype=int)   # the root link of each dof's multibody
    for i, row in enumerate(L):
        if row[3] < 0:
            continue
        r = i
        while L[r, 0] >= 0:
            r = int(L[r, 0])
        root[int(row[3]):int(row[3]) + (3 if int(row[1]) == SPHERICAL else 1)] = r
    between = root[:, None] != root[None, :]
    assert between.any() and len(set(root)) == int(model[12])
    assert np.all(C[:, between] == 0.0)
    assert np.all(emu_mass.mass(model, q)[:, between] == 0.0)
    assert np.abs(C).max() > 0.0


# ---- parameters -----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_parameters_at_the_model_values_are_bit_identical(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    ids = all_ids(model)
    vals = param_values(model)[ids]
    assert np.array_equal(ecor.coriolis(model, q, qd, ids=ids, values=vals), ecor.coriolis(model, q, qd))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_per_environment_parameters_equal_edited_models(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    C = ecor.coriolis(model, q, qd, ids=ids, values=vals)
    for e in range(q.shape[0]):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert np.array_equal(C[e:e + 1], ecor.coriolis(edited, q[e:e + 1], qd[e:e + 1])), (name, e)


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "humanoid_spherical"])
def test_stiffness_damping_friction_restitution_do_not_enter(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    names = param_names(model)
    ids = [i for i in all_ids(model) if names[i] in ("friction", "restitution") or names[i].endswith(("stiffness", "damping"))]
    vals = perturbed(model, ids, q.shape[0], 11, 0.5, 0.0)
    assert np.array_equal(ecor.coriolis(model, q, qd, ids=ids, values=vals), ecor.coriolis(model, q, qd))


# ---- derivatives ----------------------------------------------------------------------------------------------------------------------

def inertial_ids(model):
    names = param_names(model)
    return [i for i in all_ids(model) if names[i].startswith(("base.", "link")) and not names[i].endswith(("stiffness", "damping"))]


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "sphere2", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_against_central_differences(name):
    """Along q, qd and the parameters separately, central differences of the fp64 instance at h = 2^-10.  q and qd sit on grids that
    keep q +- h v exact in fp32 (the instance rounds them), the parameters are fp64 inputs; along q the truncation error bounds the
    tolerance, along qd (C is linear in it) only rounding is left, along the parameters (C is a polynomial of degree three in them) the
    truncation error again."""
    model, q = fixture(name)
    q, qd, _ = grid_state(model, q, 23)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = inertial_ids(model)
    p0 = np.tile(param_values(model)[ids], (n, 1))
    h = 2.0 ** -10
    rng = np.random.default_rng(29)
    for part, dim, tol in ((0, n_q, 1e-4), (1, nd, 1e-9), (2, len(ids), 1e-6)):
        v = np.round(rng.normal(size=(n, dim)) * 16) / 16
        x = [q, qd, p0]
        xp, xm = list(x), list(x)
        xp[part], xm[part] = x[part] + h * v * (np.abs(p0) if part == 2 else 1), x[part] - h * v * (np.abs(p0) if part == 2 else 1)
        if part < 2:
            assert np.array_equal(f32(xp[part]), xp[part]) and np.array_equal(f32(xm[part]), xm[part])
        fd = (ecor.coriolis(model, xp[0], xp[1], ids=ids, values=xp[2]) - ecor.coriolis(model, xm[0], xm[1], ids=ids, values=xm[2])) / (2 * h)
        t = [None, None, None]
        t[part] = (v * (np.abs(p0) if part == 2 else 1))[:, :, None]
        jv = ecor.coriolis_jvp(model, q, qd, *t, ids=ids, values=p0)[..., 0]
        err = np.abs(jv - fd).max() / max(1.0, np.abs(fd).max())
        assert err <= tol, (name, part, err)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "humanoid"])
def test_q_tangent_against_the_oracle_bias_forces(name):
    """dC[t_q] qd = d/dq (h(q, qd) - h(q, 0)) [t_q], central differences of the C oracle's fp64 RNEA (h = 1e-6)."""
    model, q = fixture(name)
    q, qd = state(model, q)
    q, qd = q[:2], qd[:2]
    m0 = without_springs(model)
    t = np.random.default_rng(7).normal(size=q.shape)
    dC = ecor.coriolis_jvp(model, q, qd, t_q=t[:, :, None])[..., 0]
    h = 1e-6
    hv = lambda a, b: emu_invdyn.oracle(m0, a, b) - emu_invdyn.oracle(m0, a)
    fd = np.array([(hv(a + h * u, b) - hv(a - h * u, b)) / (2 * h) for a, b, u in zip(q, qd, t)])
    close(np.einsum("eij,ej->ei", dC, qd), fd, 1e-6)


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid_spherical", "mb_racket"])
def test_tangents_of_one_call_are_independent(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = inertial_ids(model)
    vals = perturbed(model, ids, n, 3, 0.5, 0.0)
    rng = np.random.default_rng(5)
    tq, tqd, tp = rng.normal(size=(n, n_q, 3)), rng.normal(size=(n, nd, 3)), rng.normal(size=(n, len(ids), 3))
    all_ = ecor.coriolis_jvp(model, q, qd, tq, tqd, tp, ids=ids, values=vals)
    for j in range(3):
        one = ecor.coriolis_jvp(model, q, qd, tq[..., j:j + 1], tqd[..., j:j + 1], tp[..., j:j + 1], ids=ids, values=vals)[..., 0]
        assert np.array_equal(all_[..., j], one)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    model, q = fixture(name)
    q, qd = state(model, q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    ids = inertial_ids(model)
    vals = perturbed(model, ids, n, 4, 0.5, 0.0)
    rng = np.random.default_rng(6)
    G = rng.normal(size=(n, nd, nd))
    v = [rng.normal(size=(n, d)) for d in (n_q, nd, len(ids))]
    jv = ecor.coriolis_jvp(model, q, qd, *(x[:, :, None] for x in v), ids=ids, values=vals)[..., 0]
    g = ecor.coriolis_vjp(model, q, qd, G, ids=ids, values=vals)
    fwd = np.einsum("eij,eij->e", G, jv)
    rev = sum(np.einsum("ec,ec->e", a, b) for a, b in zip(g, v))
    assert np.all(np.abs(fwd - rev) <= 1e-10 * np.maximum(1.0, np.abs(fwd))), (fwd, rev)
