"""Forward kinematics and linear point Jacobians (DESIGN.md section 7.13) on the CPU, from the kernel SOURCE: the KIN instances of
csrc/tds_stepw.cu compiled for the host (tests/cpp/kin_host.cpp, bound by tests/emu_kin.py) against the fp64 C oracle (link transforms of
its kinematics pass, its point_jacobian: tests/cpp/oracle_kin.c), an independent NumPy restatement from the kernel's own transforms and
the model's joint axes, worlds of several multibodies, the derivatives (JVP against J and against central differences, independence of
the tangents of one call, JVP / VJP duality), and a batched inverse kinematics on Laikago.  tests/test_kinematics_gpu.py checks the same
instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_values, set_param_values
from oracle import port
import emu_kin
from test_mass_matrix_on_host import fixture, f32, ORACLE_FIXTURES, OTHER_FIXTURES, HEADER, BASE, LINK
from test_params_on_host import all_ids, perturbed

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
LAIKAGO_TOES = [9, 13, 17, 21]


def links_of(model):
    n = int(model[1])
    return np.asarray(model[HEADER + BASE:HEADER + BASE + n * LINK]).reshape(n, LINK)


def tables(model, seed=0):
    """Point tables of at most 64 points covering every link origin, one offset point per link and two base points."""
    rng = np.random.default_rng(seed)
    lk, lc = [-1, -1], [np.zeros(3), np.array([0.1, -0.05, 0.2])]
    for i in range(int(model[1])):
        lk += [i, i]
        lc += [np.zeros(3), rng.uniform(-0.2, 0.2, 3)]
    lc = np.array(lc)
    return [(np.array(lk[a:a + 64]), lc[a:a + 64]) for a in range(0, len(lk), 64)]


def quat_matrix(x, y, z, w):
    """The rotation of the quaternion (x, y, z, w) as the reference builds it: s = 2 / |q|^2 (tiny_matrix3x3.h setRotation)."""
    s = 2.0 / (x * x + y * y + z * z + w * w)
    return np.array([[1 - s * (y * y + z * z), s * (x * y - z * w), s * (x * z + y * w)],
                     [s * (x * y + z * w), 1 - s * (x * x + z * z), s * (y * z - x * w)],
                     [s * (x * z - y * w), s * (y * z + x * w), 1 - s * (x * x + y * y)]])


def base_xf(model, q):
    if int(model[2]):
        return quat_matrix(*q[:4]), np.asarray(q[4:7], dtype=np.float64)
    return np.eye(3), np.zeros(3)


def oracle_outputs(model, q, lk, lc):
    """(xf [n_links, 12], x [K, 3], J [K, 3, n_qd]) of the C oracle at q (fp64, as given)."""
    xf = port.step(model, port.make_params(), port.MODE_FD, q, np.zeros(int(model[4])))["link_xf"]
    Rb, pb = base_xf(model, q)
    x = np.array([(Rb @ c + pb) if l < 0 else (xf[l, :9].reshape(3, 3) @ c + xf[l, 9:]) for l, c in zip(lk, lc)])
    J = np.array([emu_kin.oracle_point_jacobian(model, q, l, p) for l, p in zip(lk, x)])
    return xf, x, J


def close(a, ref, tol):
    return np.all(np.abs(a - ref) <= tol * np.maximum(1.0, np.abs(ref)))


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_against_the_c_oracle(name):
    model, q = fixture(name)
    q = f32(q[:4])
    for lk, lc in tables(model):
        xf, x, J = emu_kin.kinematics(model, q, lk, lc)
        for e in range(q.shape[0]):
            xo, xo_, Jo = oracle_outputs(model, q[e], lk, lc)
            assert close(xf[e], xo, 1e-10), (name, np.abs(xf[e] - xo).max())
            assert close(x[e], xo_, 1e-10), (name, np.abs(x[e] - xo_).max())
            assert close(J[e], Jo, 1e-10), (name, np.abs(J[e] - Jo).max())


def numpy_jacobian(model, q, xf, lk, x):
    """J [K, 3, n_qd] from the kernel's link transforms xf and the model's joint axes (jacobian.hpp:13-83 restated)."""
    L = links_of(model)
    nd = int(model[4])
    J = np.zeros((len(lk), 3, nd))
    Rb, pb = base_xf(model, q)
    for k, (l, xk) in enumerate(zip(lk, x)):
        if int(model[2]):   # trap 13: [-[x - r0]x^T | I3], the base rotation ignored
            d = xk - pb
            for c in range(3):
                J[k, :, c] = np.cross(np.eye(3)[c], d)
            J[k, :, 3:6] = np.eye(3)
        j = l
        while j >= 0:
            jt, qd0 = int(L[j, 1]), int(L[j, 3])
            R, p = xf[j, :9].reshape(3, 3), xf[j, 9:]
            a = L[j, 4:7]
            if jt == 8:
                for c in range(3):
                    J[k, :, qd0 + c] = np.cross(R[:, c], xk - p)
            elif 0 <= jt <= 3:
                J[k, :, qd0] = R @ a
            elif 4 <= jt <= 7:
                J[k, :, qd0] = np.cross(R @ a, xk - p)
            j = int(L[j, 0])
    return J


@pytest.mark.parametrize("name", ALL)
def test_against_a_numpy_restatement(name):
    model, q = fixture(name)
    q = f32(q)
    for lk, lc in tables(model, 1):
        xf, x, J = emu_kin.kinematics(model, q, lk, lc)
        for e in range(q.shape[0]):
            Rb, pb = base_xf(model, q[e])
            xr = np.array([(Rb @ c + pb) if l < 0 else (xf[e, l, :9].reshape(3, 3) @ c + xf[e, l, 9:]) for l, c in zip(lk, lc)])
            assert close(x[e], xr, 1e-12), name
            Jn = numpy_jacobian(model, q[e], xf[e], lk, x[e])
            assert close(J[e], Jn, 1e-10), (name, np.abs(J[e] - Jn).max())


def body_columns(model):
    """The dof columns of the multibody of every link (a world of several multibodies: every root link starts one)."""
    L = links_of(model)
    body, cols = [], {}
    for i in range(L.shape[0]):
        b = len(cols) if L[i, 0] < 0 else body[int(L[i, 0])]
        body.append(b)
        if int(L[i, 1]) >= 0:
            nc = 3 if int(L[i, 1]) == 8 else 1
            cols.setdefault(b, set()).update(range(int(L[i, 3]), int(L[i, 3]) + nc))
        else:
            cols.setdefault(b, set())
    return body, cols


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_columns_outside_the_points_multibody_are_zero(name):
    model, q = fixture(name)
    body, cols = body_columns(model)
    assert len(cols) >= 2
    nd = int(model[4])
    for lk, lc in tables(model, 2):
        _, _, J = emu_kin.kinematics(model, q, lk, lc)
        for k, l in enumerate(lk):
            if l < 0:
                assert np.all(J[:, k] == 0.0)
                continue
            outside = np.array([c not in cols[body[l]] for c in range(nd)])
            assert np.all(J[:, k][:, :, outside] == 0.0), (name, l)
            assert np.any(J[:, k][:, :, ~outside] != 0.0) or not cols[body[l]]


FIXED_REVOLUTE = ["pendulum5", "cartpole", "laikago", "ant", "humanoid_fixed", "mb_three_bodies", "mb_racket"]


@pytest.mark.parametrize("name", FIXED_REVOLUTE)
def test_jvp_of_x_is_J_v(name):
    """Fixed bases without spherical joints (q-space = qd-space): dx[v] = J v within 1e-10.  A joint about a given axis (REVOLUTE_AXIS)
    turns by q about the normalised axis while its column is the reference's S = R a (link.hpp:229-336), so that column is divided by |a|
    here (the fp32-rounded axes of ant and the humanoid are unit only to ~1e-7)."""
    model, q = fixture(name)
    assert int(model[2]) == 0 and int(model[3]) == int(model[4])
    L = links_of(model)
    scale = np.ones(int(model[4]))
    for i in range(L.shape[0]):
        if int(L[i, 1]) == 7:
            scale[int(L[i, 3])] = 1.0 / np.linalg.norm(L[i, 4:7])
    v = np.random.default_rng(11).normal(size=(q.shape[0], q.shape[1], 1))
    for lk, lc in tables(model):
        _, x, J = emu_kin.kinematics(model, q, lk, lc)
        _, dx, _ = emu_kin.kinematics_jvp(model, q, lk, lc, v)
        assert close(dx[..., 0], np.einsum("ekrc,ec->ekr", J * scale, v[..., 0]), 1e-10), name


def _stack(xf, x, J):
    n = xf.shape[0]
    return np.concatenate([xf.reshape(n, -1), x.reshape(n, -1), J.reshape(n, -1)], axis=1)


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_jvp_against_central_differences_of_the_oracle(name):
    """d(xf | x | J) along random q tangents against central differences of the oracle, h = 1e-6."""
    model, q = fixture(name)
    q = f32(q[:2])
    v = np.random.default_rng(13).normal(size=q.shape)
    h, worst = 1e-6, 0.0
    for lk, lc in tables(model):
        d = emu_kin.kinematics_jvp(model, q, lk, lc, v[:, :, None])
        dk = _stack(*(a[..., 0] for a in d))
        for e in range(q.shape[0]):
            fd = (_stack(*(a[None] for a in oracle_outputs(model, q[e] + h * v[e], lk, lc))) -
                  _stack(*(a[None] for a in oracle_outputs(model, q[e] - h * v[e], lk, lc))))[0] / (2 * h)
            err = np.abs(dk[e] - fd).max() / max(1.0, np.abs(fd).max())
            worst = max(worst, err)
            assert err <= 1e-6, (name, err)
    print(f"{name}: largest relative error {worst:.2e}")


@pytest.mark.parametrize("name", ["pendulum5spherical", "humanoid_spherical"])
def test_jvp_against_central_differences_of_the_host_build(name):
    """Spherical joints (not restated by the oracle): central differences of the host build itself, h = 2^-10, at q and tangents on a
    grid that keeps q +- h v exact in fp32 (the kernel rounds q to fp32)."""
    model, q = fixture(name)
    q = np.round(q[:2] * 4096) / 4096
    v = np.round(np.random.default_rng(17).normal(size=q.shape) * 16) / 16
    h = 2.0 ** -10
    assert np.array_equal(f32(q + h * v), q + h * v)
    for lk, lc in tables(model):
        dk = _stack(*(a[..., 0] for a in emu_kin.kinematics_jvp(model, q, lk, lc, v[:, :, None])))
        fd = (_stack(*emu_kin.kinematics(model, q + h * v, lk, lc)) - _stack(*emu_kin.kinematics(model, q - h * v, lk, lc))) / (2 * h)
        err = np.abs(dk - fd).max() / max(1.0, np.abs(fd).max())
        print(f"{name}: largest relative error {err:.2e}")
        assert err <= 1e-4, (name, err)


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_tangents_of_one_call_are_independent(name):
    model, q = fixture(name)
    v = np.random.default_rng(5).normal(size=(q.shape[0], q.shape[1], 3))
    lk, lc = tables(model)[0]
    d = emu_kin.kinematics_jvp(model, q, lk, lc, v)
    for j in range(3):
        one = emu_kin.kinematics_jvp(model, q, lk, lc, v[:, :, j:j + 1])
        for a, b in zip(one, d):
            assert np.array_equal(a[..., 0], b[..., j])


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    model, q = fixture(name)
    rng = np.random.default_rng(6)
    n = q.shape[0]
    lk, lc = tables(model)[0]
    r_xf, r_x, r_J = emu_kin.rows(model, len(lk))
    G = [rng.normal(size=(n, r)) for r in (r_xf, r_x, r_J)]
    v = rng.normal(size=q.shape)
    d = emu_kin.kinematics_jvp(model, q, lk, lc, v[:, :, None])
    fwd = sum(np.einsum("er,er->e", g, a.reshape(n, -1)) for g, a in zip(G, d))
    g_q = emu_kin.kinematics_vjp(model, q, lk, lc, *G)
    rev = np.einsum("ec,ec->e", g_q, v)
    assert np.all(np.abs(fwd - rev) <= 1e-10 * np.maximum(1.0, np.abs(fwd))), (fwd, rev)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_physical_parameters_do_not_enter(name):
    """Masses, centres of mass, inertias, stiffness and damping (edited per environment, +-20 %) leave every output bit-identical."""
    model, q = fixture(name)
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    lk, lc = tables(model)[0]
    ref = emu_kin.kinematics(model, q, lk, lc)
    for e in range(2):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert not np.array_equal(param_values(edited), param_values(model))
        out = emu_kin.kinematics(edited, q, lk, lc)
        for a, b in zip(out, ref):
            assert np.array_equal(a, b)


def laikago_ik(kin, q_target, rng, iters=15, lam=1e-6):
    """Damped Gauss-Newton on the four toe positions over the 12 leg joints, from 0.1 rad away from q_target.  kin(q) -> (x [n, 4, 3],
    J [n, 4, 3, n_qd]).  Returns (final errors [n], iterations used)."""
    legs = np.arange(6, 18)
    x_t, _ = kin(q_target)
    q = q_target.copy()
    q[:, legs] += 0.1 * rng.choice([-1.0, 1.0], size=(q.shape[0], 12))
    for it in range(1, iters + 1):
        x, J = kin(q)
        r = (x_t - x).reshape(q.shape[0], 12)
        Jl = J.reshape(q.shape[0], 12, -1)[:, :, legs]
        A = Jl @ Jl.transpose(0, 2, 1) + lam * np.eye(12)
        q[:, legs] += np.einsum("eji,ej->ei", Jl, np.linalg.solve(A, r[..., None])[..., 0])
        err = np.linalg.norm((x_t - kin(q)[0]).reshape(q.shape[0], 4, 3), axis=2).max(axis=1)
        if err.max() <= 1e-4:
            return err, it
    return err, iters


def laikago_targets(n, seed):
    model, q = fixture("laikago")
    rng = np.random.default_rng(seed)
    qt = np.repeat(q[:1], n, axis=0)
    qt[:, 6:] += rng.uniform(-0.3, 0.3, size=(n, 12))
    return model, f32(qt), rng


def test_batched_inverse_kinematics_on_laikago():
    """Damped Gauss-Newton on the four toes with this feature's x and J alone: within 1e-4 m on every environment in <= 15 iterations."""
    model, qt, rng = laikago_targets(8, 21)
    lc = np.zeros((4, 3))

    def kin(q):
        _, x, J = emu_kin.kinematics(model, q, LAIKAGO_TOES, lc)
        return x, J
    err, it = laikago_ik(kin, qt, rng)
    print(f"laikago IK: {it} iterations, largest toe error {err.max():.2e} m")
    assert err.max() <= 1e-4 and it <= 15
