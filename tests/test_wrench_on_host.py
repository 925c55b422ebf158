"""The step with external wrenches (DESIGN.md section 7.18) on the CPU, from the kernel SOURCE: the EXT instances of csrc/tds_stepw.cu
compiled for the host (tests/cpp/wrench_host.cpp, bound by tests/emu_wrench.py).  Zero wrenches against the host-built step (bitwise), qdd
against the C oracle's forward dynamics with the reference's f_ext term (tests/cpp/oracle_wrench.c), the slope M^-1 J^T against the mass
matrix and point Jacobians (sections 7.12, 7.17) that share no code with the wrench term, rigid-body equivalences, inverse dynamics with
wrenches by composition, the derivatives and multibody isolation.  tests/test_wrench_gpu.py checks the same instances as nvcc builds them.

qdd is affine in the wrenches at fixed q, qd and tau, so the JVP along t_W = W is exactly qdd(W) - qdd(0) in fp64: the checks below that
need fp64 values of the wrench term (the step's value outputs are fp32) take it from the dual-number instance."""
import numpy as np
import pytest

import emu
import emu_invdyn
import emu_kin
import emu_mass
import emu_params
import emu_point_motion
import emu_wrench
from test_mass_matrix_on_host import HEADER, BASE, LINK, f32, fixture, rel

ALL = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "pendulum5spherical", "humanoid_spherical",
       "mb_three_bodies", "mb_racket"]
# the fixtures where M dqdd/dtau = I (test_mass_matrix_on_host.py::test_inverse_of_the_dual_forward_dynamics_jacobian)
FIXED = ["pendulum5", "cartpole", "cartpole_plane", "laikago", "ant", "pendulum5spherical", "humanoid_spherical", "humanoid_fixed",
         "mb_three_bodies"]
FLOATING = ["sphere2", "box", "humanoid"]
LAIKAGO_ENV = (12, 6, 100.0, 2.0, 50.0, 0.4) + (0.0, 0.67, -1.25) * 4
N = 4


def state(name, n=N, seed=1):
    """(model, q, qd, tau) of a fixture: golden configurations, random fp32 velocities and torques."""
    model, q = fixture(name)
    q = q[:n]
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    n_tau = nd - (6 if int(model[2]) else 0)
    return model, q, f32(rng.normal(size=(q.shape[0], nd)) * 0.3), f32(rng.normal(size=(q.shape[0], n_tau)))


def table(model, seed=2):
    """The point table: two base points, every link origin and one offset point per link, as many of the last as
    TDS_B200_MAX_KIN_POINTS (64) leaves room for."""
    nl = int(model[1])
    rng = np.random.default_rng(seed)
    n_off = min(nl, 64 - 2 - nl)
    links = [-1, -1] + list(range(nl)) + list(range(n_off))
    local = np.concatenate([rng.normal(size=(2, 3)) * 0.1, np.zeros((nl, 3)), rng.normal(size=(n_off, 3)) * 0.1])
    return links, local


def wrenches(n, K, seed=3, scale=1.0):
    return f32(np.random.default_rng(seed).normal(size=(n, K, 6)) * scale)


def param_set(model, q):
    """Every installable parameter of the model (test_params_on_host.all_ids) at values near the model's."""
    from test_params_on_host import all_ids
    from tds_b200.model import param_values
    ids = all_ids(model)
    v = np.asarray(param_values(model), dtype=np.float64)[ids]
    return ids, np.broadcast_to(v * 1.05, (q.shape[0], len(ids))).copy()


def link_body(model):
    """The multibody of every link (a root link starts one)."""
    m = np.asarray(model)
    out = []
    for i in range(int(m[1])):
        p = int(m[HEADER + BASE + i * LINK])
        out.append(out[p] if p >= 0 else (max(out) + 1 if out else 0))
    return out


def dof_body(model):
    m = np.asarray(model)
    body = link_body(model)
    d = np.full(int(m[4]), -1)
    for i in range(int(m[1])):
        o = HEADER + BASE + i * LINK
        jt, qd0 = int(m[o + 1]), int(m[o + 3])
        if jt != -1:
            d[qd0:qd0 + (3 if jt == 8 else 1)] = body[i]
    return d


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("name", ALL)
def test_zero_wrenches_change_nothing(name, precision):
    """K = 0 and W = 0: q', qd' and qdd bitwise those of the step's host instance of the same precision."""
    model, q, qd, tau = state(name)
    links, local = table(model)
    for mode in (0, 1, 2):
        ref = emu.step(model, mode, q, qd, tau, precision=precision)
        for lk, lc in (([], np.zeros((0, 3))), (links, local)):
            out = emu_wrench.step_wrench(model, mode, q, qd, tau, lk, lc, np.zeros((q.shape[0], len(lk), 6)), precision=precision)
            if mode == 0:
                assert np.array_equal(out, ref["qdd"])
            else:
                assert np.array_equal(out[0], ref["q"]) and np.array_equal(out[1], ref["qd"])


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_zero_wrenches_with_pd_and_parameters(precision):
    """Laikago with PD, and a fixture with an installed parameter set: W = 0 is bitwise the step."""
    model, q, qd, _ = state("laikago")
    act = f32(np.random.default_rng(4).uniform(-0.3, 0.3, size=(q.shape[0], 12)))
    links, local = table(model)
    W0 = np.zeros((q.shape[0], len(links), 6))
    qo, qdo = emu_wrench.step_wrench(model, 2, q, qd, act, links, local, W0, precision=precision, use_pd=True, env=LAIKAGO_ENV)
    ref = emu.step(model, 2, q, qd, act, precision=precision, use_pd=True, env=LAIKAGO_ENV)
    assert np.array_equal(qo, ref["q"]) and np.array_equal(qdo, ref["qd"])
    for name in ("laikago", "humanoid"):
        model, q, qd, tau = state(name)
        links, local = table(model)
        ids, vals = param_set(model, q)
        W0 = np.zeros((q.shape[0], len(links), 6))
        for mode in (0, 2):
            out = emu_wrench.step_wrench(model, mode, q, qd, tau, links, local, W0, precision=precision, ids=ids, values=vals)
            ref = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, precision=precision)
            if mode == 0:
                assert np.array_equal(out, ref["qdd"])
            else:
                assert np.array_equal(out[0], ref["q"]) and np.array_equal(out[1], ref["qd"])


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid"])
def test_against_the_c_oracle(name):
    """MODE_FD: the wrench term qdd(W) - qdd(0) (the JVP along t_W = W) within 1e-10 of the oracle's, and the fp64 instance's qdd within
    its fp32 output rounding of the oracle's qdd(W)."""
    model, q, qd, tau = state(name)
    links, local = table(model)
    W = wrenches(q.shape[0], len(links))
    qdd = emu_wrench.step_wrench(model, 0, q, qd, tau, links, local, W, precision=1)
    dW = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_W=W[..., None])[:, :, 0]
    for e in range(q.shape[0]):
        o1 = emu_wrench.oracle_fd(model, f32(q[e]), qd[e], tau[e], links, local, W[e])
        o0 = emu_wrench.oracle_fd(model, f32(q[e]), qd[e], tau[e], links, local, np.zeros_like(W[e]))
        assert o1 is not None, "the oracle does not cover the model"
        assert rel(dW[e], o1 - o0) <= 1e-10, rel(dW[e], o1 - o0)
        assert rel(qdd[e], o1) <= 1e-6, rel(qdd[e], o1)


@pytest.mark.parametrize("name", FIXED)
def test_slope_is_m_inverse_jt_on_fixed_bases(name):
    """M dqdd/dW t_W = sum_k J_k^T t_W_k within 1e-10, with M from the mass-matrix and J from the point-motion host builds."""
    model, q, qd, tau = state(name)
    links, local = table(model)
    tW = wrenches(q.shape[0], len(links), seed=5)
    d = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, np.zeros_like(tW), t_W=tW[..., None])[:, :, 0]
    M = emu_mass.mass(model, q)
    J, _, _ = emu_point_motion.point_motion(model, q, links, local)
    rhs = np.einsum("nkrc,nkr->nc", J, tW)
    assert rel(np.einsum("nij,nj->ni", M, d), rhs) <= 1e-10


@pytest.mark.parametrize("name", FLOATING)
def test_slope_residual_on_floating_bases(name):
    """Reported, not asserted: |M dqdd/dW t_W - sum J^T t_W| on a floating base, where the reference's forward dynamics does not invert
    its own M (DESIGN.md sections 7.12, 7.14).  The oracle and the equivalences pin the values there."""
    model, q, qd, tau = state(name)
    links, local = table(model)
    tW = wrenches(q.shape[0], len(links), seed=5)
    d = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, np.zeros_like(tW), t_W=tW[..., None])[:, :, 0]
    M = emu_mass.mass(model, q)
    J, _, _ = emu_point_motion.point_motion(model, q, links, local)
    r = rel(np.einsum("nij,nj->ni", M, d), np.einsum("nkrc,nkr->nc", J, tW))
    print(f"{name}: M dqdd/dW t_W - J^T t_W, largest relative residual {r:.3e}")
    assert np.isfinite(r)


def _term(model, q, qd, tau, links, local, W):
    """The wrench term qdd(W) - qdd(0) in fp64 (the JVP along t_W = W)."""
    return emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_W=np.asarray(W)[..., None])[:, :, 0]


@pytest.mark.parametrize("name", ALL)
def test_rigid_body_equivalences(name):
    """A force sliding along its line of action, a wrench moved to another point of its body with n' = n + (x - x') x f, a wrench moved
    from a fixed-joint link to its parent and a wrench split over two points with the same resultant all give the same qdd."""
    model, q, qd, tau = state(name)
    n, nl = q.shape[0], int(model[1])
    rng = np.random.default_rng(6)
    bodies = [-1] + list(range(nl)) if int(model[2]) else list(range(nl))
    for l in bodies:
        a, b = rng.normal(size=3) * 0.1, rng.normal(size=3) * 0.1
        # the same link-frame direction d in every environment: the line through a along d is a line of the body
        dirn = rng.normal(size=3)
        _, x, _ = emu_kin.kinematics(model, q, [l, l], np.array([a, b]))
        f = _frame(model, q, l) @ dirn
        m = rng.normal(size=(n, 3))
        W1 = np.concatenate([m, f], axis=1)[:, None]
        base = _term(model, q, qd, tau, [l], a[None], W1)
        scale = max(1.0, np.abs(base).max())
        slid = _term(model, q, qd, tau, [l], (a + 0.7 * dirn)[None], W1)
        assert np.abs(slid - base).max() <= 1e-10 * scale, ("slide", l)
        moved = np.concatenate([m + np.cross(x[:, 0] - x[:, 1], f), f], axis=1)[:, None]
        assert np.abs(_term(model, q, qd, tau, [l], b[None], moved) - base).max() <= 1e-10 * scale, ("move", l)
        half = np.concatenate([m / 2, f / 2], axis=1)
        other = np.concatenate([m / 2 + np.cross(x[:, 0] - x[:, 1], f / 2), f / 2], axis=1)
        split = _term(model, q, qd, tau, [l, l], np.array([a, b]), np.stack([half, other], axis=1))
        assert np.abs(split - base).max() <= 1e-10 * scale, ("split", l)
    m_ = np.asarray(model)
    for l in range(nl):   # a fixed-joint link and its parent
        o = HEADER + BASE + l * LINK
        p = int(m_[o])
        if int(m_[o + 1]) != -1 or (p < 0 and not int(model[2])):
            continue
        a = rng.normal(size=3) * 0.1
        _, x, _ = emu_kin.kinematics(model, q, [l, p], np.array([a, np.zeros(3)]))
        ap = _frame(model, q, p)[0].T @ (x[0, 0] - x[0, 1])
        W = wrenches(n, 1, seed=7 + l)
        t1 = _term(model, q, qd, tau, [l], a[None], W)
        t2 = _term(model, q, qd, tau, [p], ap[None], W)
        assert np.abs(t1 - t2).max() <= 1e-9 * max(1.0, np.abs(t1).max()), ("fixed link", l)


def _frame(model, q, l):
    """The world rotation [n, 3, 3] of body l (-1: the base) as the kernels evaluate it: point positions of the unit vectors."""
    _, x, _ = emu_kin.kinematics(model, q, [l] * 4, np.vstack([np.zeros(3), np.eye(3)]))
    return np.stack([x[:, 1] - x[:, 0], x[:, 2] - x[:, 0], x[:, 3] - x[:, 0]], axis=2)


@pytest.mark.parametrize("name", FIXED)
def test_inverse_dynamics_with_wrenches_by_composition(name):
    """ID(q, qd, fl32(FD(q, qd, tau, W))) - sum_k J_k^T W_k = tau within the fp32 rounding of qdd (the bound of
    test_inverse_dynamics_on_host.py::test_round_trip_through_the_forward_dynamics)."""
    model, q, qd, tau = state(name)
    links, local = table(model)
    nd = int(model[4])
    W = wrenches(q.shape[0], len(links), scale=0.5)
    qdd = f32(emu_wrench.step_wrench(model, 0, q, qd, tau, links, local, W, precision=1))
    J, _, _ = emu_point_motion.point_motion(model, q, links, local)
    back = emu_invdyn.inverse_dynamics(model, q, qd, qdd) - np.einsum("nkrc,nkr->nc", J, W)
    M = emu_mass.mass(model, q)
    bound = 4 * 2.0 ** -24 * np.abs(M).max() * np.abs(qdd).max(axis=1, keepdims=True) * nd
    err = np.abs(back - tau)
    assert np.all(err <= bound), (err.max(), bound.max())


def _cols(model, use_pd=False, env=None):
    nq, nd = int(model[3]), int(model[4])
    return nq + nd + ((int(env[0]) + 3) if use_pd else nd - (6 if int(model[2]) else 0))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_against_central_differences(name):
    """MODE_FD JVP along q, qd, tau, W and the installed parameters, each separately, against central differences of the fp64 instance
    (whose qdd is rounded to fp32: a relative tolerance of 1e-3).  qdd is linear in tau and W and quadratic in qd, where central
    differences are exact and take steps of 0.1; q and the parameters take steps of 1e-2."""
    model, q, qd, tau = state(name, n=2)
    links, local = table(model)
    n, nq, nd = q.shape[0], int(model[3]), int(model[4])
    W = wrenches(n, len(links), scale=0.5)
    rng = np.random.default_rng(8)
    cols = _cols(model)
    h = 1e-2

    def fd(**kw):
        a = dict(q=q, qd=qd, tau=tau, W=W)
        a.update(kw)
        return emu_wrench.step_wrench(model, 0, a["q"], a["qd"], a["tau"], links, local, a["W"], precision=1)

    for what in ("qd", "tau", "W"):
        v = {"qd": qd, "tau": tau, "W": W}[what]
        t = rng.normal(size=v.shape)
        cd = (fd(**{what: v + 0.1 * t}) - fd(**{what: v - 0.1 * t})) / 0.2
        if what == "W":
            jv = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_W=t[..., None])[:, :, 0]
        else:
            ti = np.zeros((n, cols, 1))
            r0 = nq if what == "qd" else nq + nd
            ti[:, r0:r0 + v.shape[1], 0] = t
            jv = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_in=ti)[:, :, 0]
        assert np.abs(jv - cd).max() <= 1e-3 * max(1.0, np.abs(jv).max()), what
    if not int(model[2]):   # q: joint coordinates only on fixed bases (a floating base's quaternion is normalised as loaded)
        t = rng.normal(size=q.shape) * 0.1
        cd = (fd(q=f32(q + h * t)) - fd(q=f32(q - h * t))) / (2 * h)
        ti = np.zeros((n, cols, 1))
        ti[:, :nq, 0] = (f32(q + h * t) - f32(q - h * t)) / (2 * h)
        jv = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_in=ti)[:, :, 0]
        assert np.abs(jv - cd).max() <= 2e-3 * max(1.0, np.abs(jv).max()), "q"
    ids, vals = param_set(model, q)
    tp = rng.normal(size=vals.shape) * np.abs(vals) * 0.05
    cdp = (emu_wrench.step_wrench(model, 0, q, qd, tau, links, local, W, precision=1, ids=ids, values=vals + h * tp) -
           emu_wrench.step_wrench(model, 0, q, qd, tau, links, local, W, precision=1, ids=ids, values=vals - h * tp)) / (2 * h)
    jvp = emu_wrench.step_wrench_jvp(model, 0, q, qd, tau, links, local, W, t_par=tp[..., None], ids=ids, values=vals)[:, :, 0]
    assert np.abs(jvp - cdp).max() <= 1e-3 * max(1.0, np.abs(jvp).max()), "params"


@pytest.mark.parametrize("name", ["laikago", "humanoid", "mb_racket"])
def test_batched_tangents_bitwise_equal_to_single_calls(name):
    model, q, qd, tau = state(name, n=2)
    links, local = table(model)
    n, K = q.shape[0], len(links)
    W = wrenches(n, K)
    rng = np.random.default_rng(9)
    m = 3
    ti, tw = rng.normal(size=(n, _cols(model), m)), rng.normal(size=(n, K, 6, m))
    for mode in (0, 2):
        all_ = emu_wrench.step_wrench_jvp(model, mode, q, qd, tau, links, local, W, t_in=ti, t_W=tw)
        for j in range(m):
            one = emu_wrench.step_wrench_jvp(model, mode, q, qd, tau, links, local, W, t_in=ti[:, :, j:j + 1], t_W=tw[..., j:j + 1])
            assert np.array_equal(all_[:, :, j], one[:, :, 0])


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "humanoid", "mb_three_bodies"])
def test_jvp_rows_along_the_step_columns_equal_the_step_jacobian(name):
    """With the wrenches at zero, the JVP along unit tangents of the step's columns is step_jacobian (the dual instance without EXT)."""
    model, q, qd, tau = state(name, n=2)
    links, local = table(model)
    n, cols = q.shape[0], _cols(model)
    eye = np.broadcast_to(np.eye(cols), (n, cols, cols)).copy()
    for mode in (0, 1, 2):
        jv = emu_wrench.step_wrench_jvp(model, mode, q, qd, tau, links, local, np.zeros((n, len(links), 6)), t_in=eye)
        ref = emu.step(model, mode, q, qd, tau, jacobian=True)["jac"]
        assert np.abs(jv - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (mode, np.abs(jv - ref).max())


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_a_wrench_moves_only_its_own_multibody(name):
    model, q, qd, tau = state(name)
    nl = int(model[1])
    body, dofs = link_body(model), dof_body(model)
    ref = emu_wrench.step_wrench(model, 1, q, qd, tau, [], np.zeros((0, 3)), np.zeros((q.shape[0], 0, 6)))[1]
    for l in range(nl):
        W = wrenches(q.shape[0], 1, seed=10 + l)
        out = emu_wrench.step_wrench(model, 1, q, qd, tau, [l], np.array([[0.05, -0.02, 0.03]]), W)[1]
        others = dofs != body[l]
        assert np.array_equal(out[:, others], ref[:, others]), l
        assert not np.array_equal(out[:, ~others], ref[:, ~others]) or not np.any(~others), l
