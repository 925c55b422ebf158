"""Spatial point Jacobians, point velocities and accelerations J qdd + J' qd (DESIGN.md section 7.17) on the CPU, from the kernel SOURCE: the
MOT instances of csrc/tds_stepw.cu compiled for the host (tests/cpp/point_motion_host.cpp, bound by tests/emu_point_motion.py) against the
C oracle's link velocities and accelerations (tests/cpp/oracle_motion.c), exact time derivatives through the feature's own dual instance and
the kinematics instance (section 7.13), the linear point Jacobians of section 7.13, a NumPy restatement of the angular rows, the centroidal
quantities of section 7.16, and the derivatives (JVP against central differences, independence of the tangents of one call, JVP / VJP
duality).  tests/test_point_motion_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_values, set_param_values
import emu_centroidal as ec
import emu_kin
import emu_point_motion as ep
from test_mass_matrix_on_host import fixture, f32
from test_kinematics_on_host import tables, links_of, body_columns, quat_matrix
from test_params_on_host import all_ids, perturbed

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "pendulum5spherical",
            "humanoid_spherical", "mb_three_bodies"]
ORACLE = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid"]
SINGLE = [f for f in FIXTURES if not f.startswith("mb_")]
SPHERICAL, REVOLUTE_AXIS = 8, 7


def close(a, ref, tol):
    return np.all(np.abs(a - ref) <= tol * np.maximum(1.0, np.abs(ref)))


def state(model, n, seed=3):
    """fp32-exact qd, qdd [n, n_qd]."""
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return f32(rng.normal(size=(n, nd)) * 0.7), f32(rng.normal(size=(n, nd)))


def qmul(a, b):
    """The product of xyzw quaternions."""
    x1, y1, z1, w1 = a
    x2, y2, z2, w2 = b
    return np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                     w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])


def dq_dt(model, q, qd):
    """dq/dt of the motion with velocity qd: a floating base's quaternion 1/2 q_b (x) (w_b, 0) and position R_b v_b, a spherical joint's
    1/2 q (x) (w, 0); a joint about a given axis |a| qd (the reference turns it by q about the normalised axis while its S = R a is
    not normalised); other joints qd."""
    out = np.zeros_like(q)
    if int(model[2]):
        out[:4] = 0.5 * qmul(q[:4], np.append(qd[:3], 0.0))
        out[4:7] = quat_matrix(*q[:4]) @ qd[3:6]
    for row in links_of(model):
        jt, qi, di = int(row[1]), int(row[2]), int(row[3])
        if di < 0:
            continue
        if jt == SPHERICAL:
            out[qi:qi + 4] = 0.5 * qmul(q[qi:qi + 4], np.append(qd[di:di + 3], 0.0))
        else:
            out[qi] = qd[di] * (np.linalg.norm(row[4:7]) if jt == REVOLUTE_AXIS else 1.0)
    return out


@pytest.mark.parametrize("name", ORACLE)
def test_velocities_and_accelerations_against_the_oracle(name):
    """vel and acc against the oracle's link-frame v and a (kinematics.hpp:18-148 with qdd), moved to world axes and to the point."""
    model, q = fixture(name)
    q = f32(q)
    qd, qdd = state(model, q.shape[0])
    for lk, lc in tables(model):
        _, vel, acc = ep.point_motion(model, q, lk, lc, qd, qdd)
        for e in range(q.shape[0]):
            R, o, v, a = ep.oracle_motion(model, q[e], qd[e], qdd[e])
            for k, (l, c) in enumerate(zip(lk, lc)):
                Rl, ol = R[l + 1], o[l + 1]
                x = Rl @ c + ol
                w, vo, al, ao = Rl @ v[l + 1, :3], Rl @ v[l + 1, 3:], Rl @ a[l + 1, :3], Rl @ a[l + 1, 3:]
                xd = vo + np.cross(w, x - ol)
                xdd = ao + np.cross(al, x - ol) + np.cross(w, xd)
                assert close(vel[e, k], np.concatenate([w, xd]), 1e-10), (name, e, k, vel[e, k], w, xd)
                assert close(acc[e, k], np.concatenate([al, xdd]), 1e-10), (name, e, k, acc[e, k], al, xdd)


@pytest.mark.parametrize("name", FIXTURES)
def test_exact_time_derivatives(name):
    """x' (vel's linear rows) is the JVP of the kinematics' x along dq/dt, and acc is the JVP of vel along (dq/dt, qdd): the column
    convention of a floating base and the spherical joints' rates are the ones of the motion the inputs describe."""
    model, q = fixture(name)
    q = f32(q)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    tq = np.array([dq_dt(model, q[e], qd[e]) for e in range(n)])
    for lk, lc in tables(model):
        K = len(lk)
        _, vel, acc = ep.point_motion(model, q, lk, lc, qd, qdd)
        _, dx, _ = emu_kin.kinematics_jvp(model, q, lk, lc, tq[:, :, None])
        assert close(vel[..., 3:], dx[..., 0], 1e-10), (name, np.abs(vel[..., 3:] - dx[..., 0]).max())
        t_in = np.concatenate([tq, qdd, np.zeros((n, nd))], axis=1)[:, :, None]
        _, dvel, _ = ep.split(ep.point_motion_jvp(model, q, lk, lc, t_in, qd, qdd), model, K)
        assert close(acc, dvel[..., 0], 1e-10), (name, np.abs(acc - dvel[..., 0]).max())


def angular_rows(model, q, xf, lk):
    """The angular rows [K, 3, n_qd] restated: R_j a_j of each revolute ancestor j (R_j from the kinematics' xf), the columns of R_j of a
    spherical one, R_b of a floating base."""
    L = links_of(model)
    out = np.zeros((len(lk), 3, int(model[4])))
    for k, l in enumerate(lk):
        if int(model[2]):
            out[k, :, :3] = quat_matrix(*q[:4])
        j = l
        while j >= 0:
            jt, d0 = int(L[j, 1]), int(L[j, 3])
            R = xf[j, :9].reshape(3, 3)
            if jt == SPHERICAL:
                out[k, :, d0:d0 + 3] = R
            elif 4 <= jt <= 7:
                out[k, :, d0] = R @ L[j, 4:7]
            j = int(L[j, 0])
    return out


def allowed_columns(model, l):
    """The columns a point on link l may have: a floating base's and its chain's dofs."""
    L = links_of(model)
    cols = set(range(6)) if int(model[2]) else set()
    j = l
    while j >= 0:
        if int(L[j, 1]) >= 0:
            cols.update(range(int(L[j, 3]), int(L[j, 3]) + (3 if int(L[j, 1]) == SPHERICAL else 1)))
        j = int(L[j, 0])
    return cols


@pytest.mark.parametrize("name", FIXTURES + ["mb_racket"])
def test_jacobian_against_vel_and_the_kinematics(name):
    model, q = fixture(name)
    q = f32(q)
    n, nd, floating = q.shape[0], int(model[4]), int(model[2])
    qd, _ = state(model, n)
    for lk, lc in tables(model, 1):
        J, vel, _ = ep.point_motion(model, q, lk, lc, qd)
        assert close(np.einsum("ekrc,ec->ekr", J, qd), vel, 1e-12), name
        xf, _, Jk = emu_kin.kinematics(model, q, lk, lc)
        c0 = 6 if floating else 0
        assert close(J[:, :, 3:, c0:], Jk[:, :, :, c0:], 1e-12), name
        for e in range(n):
            if floating:
                Rb = quat_matrix(*q[e, :4])
                D = np.kron(np.eye(2), Rb)
                assert close(J[e, :, 3:, :6], Jk[e, :, :, :6] @ D, 1e-12), name
            assert close(J[e, :, :3], angular_rows(model, q[e], xf[e], lk), 1e-12), name
        for k, l in enumerate(lk):
            outside = np.array([c not in allowed_columns(model, l) for c in range(nd)])
            assert np.all(J[:, k][:, :, outside] == 0.0), (name, l)
        if name.startswith("mb_"):
            body, cols = body_columns(model)
            for k, l in enumerate(lk):
                if l >= 0:
                    assert np.all(J[:, k][:, :, [c for c in range(nd) if c not in cols[body[l]]]] == 0.0)


@pytest.mark.parametrize("name", FIXTURES)
def test_acceleration_is_linear_in_qdd(name):
    model, q = fixture(name)
    qd, qdd = state(model, q.shape[0])
    for lk, lc in tables(model, 2):
        J, _, acc = ep.point_motion(model, q, lk, lc, qd, qdd)
        _, _, drift = ep.point_motion(model, q, lk, lc, qd)
        d = acc - drift
        ref = np.einsum("ekrc,ec->ekr", J, qdd)
        assert np.abs(d - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (name, np.abs(d - ref).max())


def bodies(model):
    """(links [B], local coms [B, 3], masses [B], link-frame inertias [B, 3, 3]) of the counted bodies: a floating base, then the links."""
    pv = param_values(model)
    lk, lc, ms, Is = [], [], [], []
    for b in range(int(model[1]) + 1):
        if b == 0 and not int(model[2]):
            continue
        r = pv[2 + 10 * b:12 + 10 * b]
        lk.append(b - 1)
        lc.append(r[1:4])
        ms.append(r[0])
        Is.append(np.array([[r[4], r[5], r[6]], [r[5], r[7], r[8]], [r[6], r[8], r[9]]]))
    return np.array(lk), np.array(lc), np.array(ms), np.array(Is)


@pytest.mark.parametrize("name", SINGLE)
def test_consistent_with_the_centroidal_quantities(name):
    """With a point table of every counted body's centre of mass: sum m J_lin = A[3:6], sum I J_w + m (c_i - c) x J_lin = A[0:3], and at
    qdd = 0 sum m c_i'' = bias[3:6], sum I w' + w x I w + m (c_i - c) x c_i'' = bias[0:3] (I in world axes)."""
    model, q = fixture(name)
    q = f32(q)
    n = q.shape[0]
    qd, _ = state(model, n)
    lk, lc, ms, Is = bodies(model)
    assert len(lk) <= 64
    com, A, bias = ec.centroidal(model, q, qd)
    J, vel, acc = ep.point_motion(model, q, lk, lc, qd)
    xf, x, _ = emu_kin.kinematics(model, q, lk, lc)
    for e in range(n):
        c = com[e, 1:4]
        Rs = [quat_matrix(*q[e, :4]) if l < 0 else xf[e, l, :9].reshape(3, 3) for l in lk]
        Iw = np.array([R @ I @ R.T for R, I in zip(Rs, Is)])
        r = x[e] - c
        lin = np.einsum("b,brc->rc", ms, J[e, :, 3:])
        rxJ = np.cross(r[:, :, None], J[e, :, 3:], axisa=1, axisb=1, axisc=1)   # (c_i - c) x J_lin(c_i), column by column
        ang = np.einsum("bij,bjc->ic", Iw, J[e, :, :3]) + np.einsum("b,bic->ic", ms, rxJ)
        tol = 1e-10 * max(1.0, np.abs(A[e]).max())
        assert np.abs(lin - A[e, 3:]).max() <= tol, (name, np.abs(lin - A[e, 3:]).max())
        assert np.abs(ang - A[e, :3]).max() <= tol, (name, np.abs(ang - A[e, :3]).max())
        w, wd, xdd = vel[e, :, :3], acc[e, :, :3], acc[e, :, 3:]
        bl = np.einsum("b,br->r", ms, xdd)
        ba = (np.einsum("bij,bj->i", Iw, wd) + np.cross(w, np.einsum("bij,bj->bi", Iw, w)).sum(axis=0)
              + np.einsum("b,br->r", ms, np.cross(r, xdd)))
        tol = 1e-10 * max(1.0, np.abs(bias[e]).max())
        assert np.abs(bl - bias[e, 3:]).max() <= tol, (name, np.abs(bl - bias[e, 3:]).max())
        assert np.abs(ba - bias[e, :3]).max() <= tol, (name, np.abs(ba - bias[e, :3]).max())


def grid_state(model, q, seed):
    """q, qd, qdd on grids that keep the steps x +- h v (h = 2^-10, v a multiple of 1/16) exact in fp32 (the instance rounds to fp32)."""
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    q = np.round(q[:2] * 4096) / 4096
    qd, qdd = (np.round(rng.normal(size=(2, nd)) * 1024) / 1024 for _ in range(2))
    return q, qd, qdd


@pytest.mark.parametrize("name", ["pendulum5", "laikago", "sphere2", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_jvp_against_central_differences(name):
    """Along q, qd and qdd separately, central differences of the fp64 instance at h = 2^-10; along q the truncation error bounds the
    tolerance, along qd and qdd (the outputs are at most quadratic in them) only rounding is left."""
    model, q = fixture(name)
    q, qd, qdd = grid_state(model, q, 23)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    h = 2.0 ** -10
    rng = np.random.default_rng(29)
    lk, lc = tables(model)[0]
    for part, dim, tol in ((0, n_q, 1e-4), (1, nd, 1e-9), (2, nd, 1e-9)):
        v = np.round(rng.normal(size=(n, dim)) * 16) / 16
        x = [q, qd, qdd]
        xp, xm = list(x), list(x)
        xp[part], xm[part] = x[part] + h * v, x[part] - h * v
        assert np.array_equal(f32(xp[part]), xp[part]) and np.array_equal(f32(xm[part]), xm[part])
        fd = (ep.point_motion(model, xp[0], lk, lc, xp[1], xp[2], concat=True) -
              ep.point_motion(model, xm[0], lk, lc, xm[1], xm[2], concat=True)) / (2 * h)
        t_in = np.zeros((n, n_q + 2 * nd))
        off = (0, n_q, n_q + nd)[part]
        t_in[:, off:off + dim] = v
        jv = ep.point_motion_jvp(model, q, lk, lc, t_in[:, :, None], qd, qdd)[..., 0]
        err = np.abs(jv - fd).max() / max(1.0, np.abs(fd).max())
        assert err <= tol, (name, part, err)


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid_spherical", "mb_racket"])
def test_tangents_of_one_call_are_independent(name):
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    T = np.random.default_rng(5).normal(size=(n, n_q + 2 * nd, 3))
    lk, lc = tables(model)[0]
    all_ = ep.point_motion_jvp(model, q, lk, lc, T, qd, qdd)
    for j in range(3):
        assert np.array_equal(all_[..., j], ep.point_motion_jvp(model, q, lk, lc, T[..., j:j + 1], qd, qdd)[..., 0])


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    qd, qdd = state(model, n)
    lk, lc = tables(model)[0]
    rng = np.random.default_rng(6)
    G = rng.normal(size=(n, sum(ep.rows(model, len(lk)))))
    v = rng.normal(size=(n, n_q + 2 * nd))
    jv = ep.point_motion_jvp(model, q, lk, lc, v[:, :, None], qd, qdd)[..., 0]
    g = ep.point_motion_vjp(model, q, lk, lc, G, qd, qdd)
    fwd, rev = np.einsum("er,er->e", G, jv), np.einsum("ec,ec->e", g, v)
    assert np.all(np.abs(fwd - rev) <= 1e-10 * np.maximum(1.0, np.abs(fwd))), (fwd, rev)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_physical_parameters_do_not_enter(name):
    """Masses, centres of mass, inertias, stiffness and damping (edited per environment) leave every output bit-identical."""
    model, q = fixture(name)
    qd, qdd = state(model, q.shape[0])
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    lk, lc = tables(model)[0]
    ref = ep.point_motion(model, q, lk, lc, qd, qdd, concat=True)
    for e in range(2):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert not np.array_equal(param_values(edited), param_values(model))
        assert np.array_equal(ep.point_motion(edited, q, lk, lc, qd, qdd, concat=True), ref)
