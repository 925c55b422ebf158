"""Centre of mass, centroidal momentum matrix A_G and its bias A_G' qd (DESIGN.md section 7.16) on the CPU, from the kernel SOURCE: the CEN
instances of csrc/tds_stepw.cu compiled for the host (tests/cpp/centroidal_host.cpp, bound by tests/emu_centroidal.py) against a NumPy
restatement over the C oracle's link transforms, the point Jacobians (section 7.13), the mass matrix (section 7.12) and inverse dynamics
(section 7.14) of the same kernel source, central differences, per-environment parameters, and a Gauss-Newton use.
tests/test_centroidal_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_names, param_values, set_param_values
from oracle import port
import emu_centroidal as ec
import emu_invdyn
import emu_kin
import emu_mass
from test_mass_matrix_on_host import fixture, f32, rel
from test_params_on_host import all_ids, perturbed

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "pendulum5spherical",
            "humanoid_spherical"]
FLOATING = ["sphere2", "box", "humanoid"]
HEADER, BASE, LINK = 16, 13, 34
SPHERICAL = 8


def dims(model):
    return int(model[1]), int(model[2]), int(model[3]), int(model[4])


def has_spherical(model):
    n_links = int(model[1])
    return any(int(model[HEADER + BASE + i * LINK + 1]) == SPHERICAL for i in range(n_links))


def velocities(model, n, seed=3, scale=0.7):
    return f32(np.random.default_rng(seed).normal(size=(n, int(model[4]))) * scale)


def quat_matrix(x, y, z, w):
    """The rotation of a quaternion that need not be unit, as the kernel and the reference form it (s = 2 / |q|^2)."""
    s = 2.0 / (x * x + y * y + z * z + w * w)
    return np.array([[1 - s * (y * y + z * z), s * (x * y - z * w), s * (x * z + y * w)],
                     [s * (x * y + z * w), 1 - s * (x * x + z * z), s * (y * z - x * w)],
                     [s * (x * z - y * w), s * (y * z + x * w), 1 - s * (x * x + y * y)]])


def bodies(model, q):
    """[(m, x world com, I about the com in world axes)] of the counted bodies at q, from the C oracle's link transforms (MODE_FD, zero
    qd) and the model's masses, coms and inertias.  The oracle has no spherical joints: there the transforms come from the kinematics
    instance (section 7.13), whose code the centroidal instance does not run."""
    n_links, floating, _, nd = dims(model)
    pv = param_values(model)
    if has_spherical(model):
        xf = emu_kin.kinematics(model, q[None], [], np.zeros((0, 3)))[0][0]
    else:
        xf = port.step(model, port.make_params(), port.MODE_FD, q, np.zeros(nd))["link_xf"]

    def body(b, R, p):
        r = pv[2 + 10 * b:12 + 10 * b]
        I = np.array([[r[4], r[5], r[6]], [r[5], r[7], r[8]], [r[6], r[8], r[9]]])
        return r[0], p + R @ r[1:4], R @ I @ R.T

    out = [body(0, quat_matrix(*q[:4]), np.asarray(q[4:7]))] if floating else []
    return out + [body(i + 1, xf[i, :9].reshape(3, 3), xf[i, 9:]) for i in range(n_links)]


def record(bs):
    m = sum(b[0] for b in bs)
    c = sum(b[0] * b[1] for b in bs) / m
    I = sum(b[2] + b[0] * (np.dot(b[1] - c, b[1] - c) * np.eye(3) - np.outer(b[1] - c, b[1] - c)) for b in bs)
    return np.concatenate([[m], c, I[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]])


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def base_map(model, q, c):
    """T [6, 6] with A = T M[0:6, :] on a floating base: [Rb, -[c - p_b]x Rb; 0, Rb]."""
    Rb = quat_matrix(*q[:4])
    T = np.zeros((6, 6))
    T[:3, :3] = Rb
    T[:3, 3:] = -skew(c - q[4:7]) @ Rb
    T[3:, 3:] = Rb
    return T


def advance(model, q, qd, t):
    """q moved by t qd on a fixed base: 1-dof joints along their dof, spherical joints by the exponential map of their link-frame qd."""
    out = np.array(q, dtype=np.float64)
    for i in range(int(model[1])):
        o = HEADER + BASE + i * LINK
        qi, di = int(model[o + 2]), int(model[o + 3])
        if di < 0:
            continue
        if int(model[o + 1]) != SPHERICAL:
            out[qi] = q[qi] + t * qd[di]
            continue
        w = qd[di:di + 3] * t
        a = np.linalg.norm(w)
        x2, y2, z2, w2 = np.concatenate([np.sin(a / 2) * w / a, [np.cos(a / 2)]]) if a > 0 else (0.0, 0.0, 0.0, 1.0)
        x1, y1, z1, w1 = q[qi:qi + 4]
        out[qi:qi + 4] = [w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                          w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2]
    return out


@pytest.mark.parametrize("name", FIXTURES)
def test_body_record_against_the_oracle_transforms(name):
    model, q = fixture(name)
    com, _, _ = ec.centroidal(model, q)
    ref = np.array([record(bodies(model, x)) for x in f32(q)])
    assert np.all(np.abs(com - ref) <= 1e-10 * np.maximum(1.0, np.abs(ref))), rel(com, ref)


@pytest.mark.parametrize("name", FIXTURES)
def test_linear_rows_are_the_mass_weighted_com_jacobians(name):
    model, q = fixture(name)
    n_links, floating, _, nd = dims(model)
    _, A, _ = ec.centroidal(model, q)
    pv = param_values(model)
    links = list(range(n_links))
    local = np.array([pv[12 + 10 * i + 1:12 + 10 * i + 4] for i in links])
    _, _, J = emu_kin.kinematics(model, q, links, local)
    ref = np.einsum("l,elrc->erc", np.array([pv[12 + 10 * i] for i in links]), J)
    c0 = 6 if floating else 0
    if nd == c0:
        pytest.skip("no joint columns")
    assert np.abs(A[:, 3:, c0:] - ref[:, :, c0:]).max() <= 1e-10 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", [f for f in FIXTURES if f not in FLOATING and "spherical" not in f])
def test_momentum_against_oracle_velocities(name):
    """h_G = A qd against sum R I R^T w_i + m_i (x_i - c) x x_i', with w_i and x_i' by central differences of the oracle's transforms.
    (The oracle has no spherical joints; those fixtures are covered by the body record, the linear rows and the derivative checks.)"""
    model, q = fixture(name)
    n_links, _, _, nd = dims(model)
    qd = velocities(model, q.shape[0])
    com, A, _ = ec.centroidal(model, q, qd)
    h = 1e-6
    pv = param_values(model)
    for e, x in enumerate(f32(q)):
        xp = port.step(model, port.make_params(), port.MODE_FD, advance(model, x, qd[e], h), np.zeros(nd))["link_xf"]
        xm = port.step(model, port.make_params(), port.MODE_FD, advance(model, x, qd[e], -h), np.zeros(nd))["link_xf"]
        bs = bodies(model, x)
        c = com[e, 1:4]
        k, l = np.zeros(3), np.zeros(3)
        for i, (m, xc, I) in enumerate(bs):
            r = pv[12 + 10 * i + 1:12 + 10 * i + 4]
            Rp, Rm = xp[i, :9].reshape(3, 3), xm[i, :9].reshape(3, 3)
            v = ((xp[i, 9:] + Rp @ r) - (xm[i, 9:] + Rm @ r)) / (2 * h)
            W = (Rp - Rm) / (2 * h) @ (0.5 * (Rp + Rm)).T
            w = 0.5 * np.array([W[2, 1] - W[1, 2], W[0, 2] - W[2, 0], W[1, 0] - W[0, 1]])
            k += I @ w + m * np.cross(xc - c, v)
            l += m * v
        hg = A[e] @ qd[e]
        ref = np.concatenate([k, l])
        assert np.abs(hg - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max()), (e, hg, ref)


@pytest.mark.parametrize("name", FLOATING)
def test_floating_base_against_the_mass_matrix(name):
    model, q = fixture(name)
    com, A, _ = ec.centroidal(model, q)
    M = emu_mass.mass(model, q)
    for e, x in enumerate(f32(q)):
        ref = base_map(model, x, com[e, 1:4]) @ M[e, :6, :]
        assert np.abs(A[e] - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", FLOATING)
def test_floating_bias_against_inverse_dynamics(name):
    model, q = fixture(name)
    qd = velocities(model, q.shape[0])
    com, _, bias = ec.centroidal(model, q, qd)
    tau = emu_invdyn.inverse_dynamics(model, q, qd, None, gravity=(0.0, 0.0, 0.0))
    for e, x in enumerate(f32(q)):
        ref = base_map(model, x, com[e, 1:4]) @ tau[e, :6]
        assert np.abs(bias[e] - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())


FIXED_REVOLUTE = [f for f in FIXTURES if f not in FLOATING and "spherical" not in f]


@pytest.mark.parametrize("name", FIXED_REVOLUTE)
def test_fixed_bias_is_the_derivative_of_A(name):
    """bias = d/dt [A(q + t qd)] qd at t = 0, by central differences of the fp64 instance.  The instance rounds q to fp32, so q and the
    steps q +- h qd stay on the fp32 grid: qd is rounded to a multiple of 2^-10 and h = 2^-10."""
    model, q = fixture(name)
    q = f32(q)
    qd = np.round(velocities(model, q.shape[0]) * 1024) / 1024
    h = 2.0 ** -10
    _, _, bias = ec.centroidal(model, q, qd)
    dA = (ec.centroidal(model, q + h * qd)[1] - ec.centroidal(model, q - h * qd)[1]) / (2 * h)
    ref = np.einsum("erc,ec->er", dA, qd)
    assert np.abs(bias - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", FIXED_REVOLUTE)
def test_com_velocity_is_the_linear_rows(name):
    """The JVP of c along qd (through q) equals A[3:6] qd / m.  Equal in exact arithmetic up to the models' joint axes, which the
    reference normalises in the rotation but not in S: they are unit to about 1e-9."""
    model, q = fixture(name)
    n_links, _, n_q, nd = dims(model)
    qd = velocities(model, q.shape[0])
    com, A, _ = ec.centroidal(model, q, qd)
    t_in = np.zeros((q.shape[0], n_q + nd, 1))
    t_in[:, :n_q, 0] = qd
    dc = ec.centroidal_jvp(model, q, qd, t_in)[:, 1:4, 0]
    ref = np.einsum("erc,ec->er", A[:, 3:], qd) / com[:, :1]
    assert np.abs(dc - ref).max() <= 1e-8 * max(1.0, np.abs(ref).max())


def fd(model, q, qd, ids, values, d_q, d_qd, d_par, h=1e-6):
    """Central difference of the concatenated fp64 outputs along (d_q, d_qd, d_par) at fp32-exact base points (the instance rounds its
    inputs to fp32, so the steps go through the parameters' fp64 path and the q / qd tangents through the linear direction only)."""
    def at(t):
        v = None if values is None else values + t * d_par
        return ec.centroidal(model, q + t * d_q, qd + t * d_qd, ids, v, concat=True)
    return (at(h) - at(-h)) / (2 * h)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "humanoid", "box"])
def test_jvp_against_central_differences_of_parameters(name):
    """Along two installed parameters (fp64 inputs: central differences resolve them), and along q, qd by the JVP's linearity checks."""
    model, q = fixture(name)
    n_links, floating, n_q, nd = dims(model)
    names = param_names(model)
    ids = [names.index("link0.mass"), names.index(f"link{n_links - 1}.com.x")] if n_links else [names.index("base.mass"), names.index("base.com.x")]
    values = np.broadcast_to(param_values(model)[ids], (q.shape[0], 2)).copy()
    qd = velocities(model, q.shape[0])
    rng = np.random.default_rng(5)
    d_par = rng.normal(size=values.shape)
    ref = fd(model, f32(q), qd, ids, values, 0.0, 0.0, d_par)
    jv = ec.centroidal_jvp(model, q, qd, None, d_par[:, :, None], ids, values)[..., 0]
    assert np.abs(jv - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "humanoid_spherical"])
def test_jvp_along_q_and_qd_against_central_differences(name):
    """q, qd tangents against central differences of the fp64 instance.  It rounds q, qd to fp32, so the steps stay on the fp32 grid:
    unit directions and h = 2^-10 (the truncation error bounds the tolerance)."""
    model, q = fixture(name)
    n_links, floating, n_q, nd = dims(model)
    q = f32(q)
    qd = velocities(model, q.shape[0])
    d_q, d_qd = np.zeros_like(q), np.ones_like(qd)
    d_q[:, [k for k in range(n_q) if not (floating and k < 7)][:3]] = 1.0
    jv = ec.centroidal_jvp(model, q, qd, np.concatenate([d_q, d_qd], axis=1)[:, :, None])[..., 0]
    ref = fd(model, q, qd, (), None, d_q, d_qd, 0.0, 2.0 ** -10)
    assert np.abs(jv - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid"])
def test_batched_tangents_are_bitwise_single_calls(name):
    model, q = fixture(name)
    n_links, _, n_q, nd = dims(model)
    qd = velocities(model, q.shape[0])
    rng = np.random.default_rng(7)
    T = rng.normal(size=(q.shape[0], n_q + nd, 4))
    all_ = ec.centroidal_jvp(model, q, qd, T)
    for j in range(4):
        assert np.array_equal(all_[..., j], ec.centroidal_jvp(model, q, qd, T[..., j:j + 1])[..., 0])


@pytest.mark.parametrize("name", ["cartpole", "laikago", "humanoid"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    model, q = fixture(name)
    n_links, _, n_q, nd = dims(model)
    names = param_names(model)
    ids = [names.index("link0.mass"), names.index("link0.inertia.xx")]
    values = np.broadcast_to(param_values(model)[ids], (q.shape[0], 2)).copy()
    qd = velocities(model, q.shape[0])
    rng = np.random.default_rng(8)
    G = rng.normal(size=(q.shape[0], ec.rows(model)))
    v_in, v_par = rng.normal(size=(q.shape[0], n_q + nd, 1)), rng.normal(size=(q.shape[0], 2, 1))
    jv = ec.centroidal_jvp(model, q, qd, v_in, v_par, ids, values)[..., 0]
    g_in, g_par = ec.centroidal_vjp(model, q, qd, G, ids, values)
    lhs = np.einsum("er,er->e", G, jv)
    rhs = np.einsum("ec,ec->e", g_in, v_in[..., 0]) + np.einsum("ec,ec->e", g_par, v_par[..., 0])
    assert np.abs(lhs - rhs).max() <= 1e-10 * max(1.0, np.abs(lhs).max())


@pytest.mark.parametrize("name", FIXTURES)
def test_installed_parameters_against_edited_models(name):
    model, q = fixture(name)
    ids = [i for i in all_ids(model) if param_names(model)[i].split(".")[-1] not in ("friction", "restitution", "stiffness", "damping")]
    n = q.shape[0]
    vals = perturbed(model, ids, n, 11, 0.5, 0.0)
    qd = velocities(model, n)
    out = ec.centroidal(model, q, qd, ids, vals, concat=True)
    for e in range(n):
        ref = ec.centroidal(set_param_values(model, ids, vals[e]), q[e:e + 1], qd[e:e + 1], concat=True)[0]
        assert np.all(np.abs(out[e] - ref) <= 1e-12 * np.maximum(1.0, np.abs(ref))), rel(out[e], ref)


@pytest.mark.parametrize("name", ["cartpole", "laikago", "humanoid"])
def test_irrelevant_parameters_are_bitwise_no_parameters(name):
    model, q = fixture(name)
    names = param_names(model)
    ids = [i for i, nm in enumerate(names) if nm in ("friction", "restitution") or nm.endswith((".stiffness", ".damping"))]
    vals = perturbed(model, ids, q.shape[0], 12, 0.5, 0.0)
    qd = velocities(model, q.shape[0])
    assert np.array_equal(ec.centroidal(model, q, qd, ids, vals, concat=True), ec.centroidal(model, q, qd, concat=True))


def test_gauss_newton_moves_laikago_com():
    """Damped Gauss-Newton on the leg joints with A[3:6] / m as the CoM Jacobian moves the CoM 2 cm within 5 iterations (1e-6 m)."""
    model, q = fixture("laikago")
    n_links, _, n_q, nd = dims(model)
    x = f32(q[:1])[0]
    com0 = ec.centroidal(model, x[None])[0][0, 1:4]
    target = com0 + np.array([0.02, 0.0, 0.0])
    legs = np.arange(6, nd)
    err = np.inf
    for _ in range(5):
        com, A, _ = ec.centroidal(model, x[None])
        r = target - com[0, 1:4]
        err = np.linalg.norm(r)
        if err < 1e-6:
            break
        J = A[0, 3:][:, legs] / com[0, 0]
        dx = J.T @ np.linalg.solve(J @ J.T + 1e-12 * np.eye(3), r)
        x = x.copy()
        x[legs] = f32(x[legs] + dx)
    err = np.linalg.norm(target - ec.centroidal(model, x[None])[0][0, 1:4])
    assert err < 1e-6, err
