"""The point-constrained forward dynamics qdd, f = FD_c(q, qd, tau) (DESIGN.md section 7.21) on the CPU, from the kernel SOURCE: the rows
and solve kernels of csrc/tds_constrained.cu compiled for the host (tests/cpp/constrained_dynamics_host.cpp, bound by
tests/emu_constrained_dynamics.py) on h, M^-1, J and the drift of the host builds of the INV, MINV and MOT instances, against numpy's KKT
solve of the host-built pieces and of the C oracle's (port.mass_matrix, tests/cpp/oracle_invdyn.c, oracle_motion.c), the MODE_FD step
and the step with wrenches on fixed bases, the damping, worlds of several multibodies, per-environment parameters, and the derivatives
(central differences of the oracle-built KKT solve, independence of the tangents of one call, linearity).  Tolerances scale with the
conditioning of M and of the constraint system: B = tol kappa_2(M) kappa_2(J_c M^-1 J_c^T + eps I) max|ref| elementwise, tol = 1e-13
against the host-built pieces.  tests/test_constrained_dynamics_gpu.py checks the same kernels as nvcc builds them, through the C-ABI."""
import numpy as np
import pytest

from tds_b200.model import param_values, set_param_values
from oracle import port
import emu_constrained_dynamics as ecd
import emu_invdyn
import emu_mass
import emu_mass_inverse as emi
import emu_point_motion as ep
import emu_wrench
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, _mass_ids, f32, fixture
from test_mass_inverse_on_host import body_of, kappa, points
from test_params_on_host import all_ids, perturbed

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
MB_WORLDS = ["mb_three_bodies", "mb_racket"]
FIXED = ["pendulum5", "cartpole", "humanoid_fixed", "pendulum5spherical", "mb_three_bodies", "mb_racket"]
# fixtures whose C oracle restates M, h and the link motion
ORACLE = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid"]


def state(model, n, seed=1):
    """fp32-exact qd and tau [n, n_qd]."""
    rng = np.random.default_rng(seed)
    nd = int(model[4])
    return f32(rng.normal(size=(n, nd)) * 0.5), f32(rng.normal(size=(n, nd)) * 3.0)


def rows_of(K, dims):
    """The rows of the 6K rows of J a table of K points holds: 6k + 3..5 (dims 3) or 6k + 0..5 (dims 6)."""
    return np.concatenate([np.arange(6 * k + 6 - dims, 6 * k + 6) for k in range(K)]).astype(int) if K else np.zeros(0, int)


def host_pieces(model, q, qd, links, local):
    """(M, h, J [n, 6K, n_qd], drift [n, 6K]) of the host builds."""
    n, nd, K = q.shape[0], int(model[4]), len(links)
    M, h = emu_mass.mass(model, q), emu_invdyn.inverse_dynamics(model, q, qd)
    if not K:
        return M, h, np.zeros((n, 0, nd)), np.zeros((n, 0))
    J, _, acc = ep.point_motion(model, q, links, local, qd)
    return M, h, J.reshape(n, 6 * K, nd), acc.reshape(n, 6 * K)


def oracle_pieces(model, q, qd, links, local):
    """(M, h, J, drift) of one configuration from the C oracle: J's columns are the oracle's point velocities at unit qd, the drift its
    point acceleration at qdd = 0."""
    nd, K = int(model[4]), len(links)

    def motion(v):
        R, o, vl, al = ep.oracle_motion(model, q, v, None)
        out_v, out_a = np.zeros(6 * K), np.zeros(6 * K)
        for k, (l, c) in enumerate(zip(links, local)):
            Rl, ol = R[l + 1], o[l + 1]
            x = Rl @ c + ol
            w, vo, a, ao = Rl @ vl[l + 1, :3], Rl @ vl[l + 1, 3:], Rl @ al[l + 1, :3], Rl @ al[l + 1, 3:]
            xd = vo + np.cross(w, x - ol)
            out_v[6 * k:6 * k + 6] = np.concatenate([w, xd])
            out_a[6 * k:6 * k + 6] = np.concatenate([a, ao + np.cross(a, x - ol) + np.cross(w, xd)])
        return out_v, out_a

    J = np.stack([motion(np.eye(nd)[i])[0] for i in range(nd)], axis=1) if K else np.zeros((0, nd))
    drift = motion(qd)[1] if K else np.zeros(0)
    return port.mass_matrix(model, q), emu_invdyn.oracle(model, q, qd), J, drift


def kkt(M, h, J, drift, tau, K, dims, eps=0.0):
    """numpy's solve of the KKT system: (qdd [n, n_qd], f [n, K, dims], kappa_2 of J_c M^-1 J_c^T + eps I per environment)."""
    n, nd = M.shape[0], M.shape[1]
    sel = rows_of(K, dims)
    Jc, dc = J[:, sel], drift[:, sel]
    R = len(sel)
    A = np.zeros((n, nd + R, nd + R))
    A[:, :nd, :nd], A[:, :nd, nd:], A[:, nd:, :nd] = M, -Jc.transpose(0, 2, 1), Jc
    A[:, nd:, nd:] = eps * np.eye(R)
    x = np.linalg.solve(A, np.concatenate([tau - h, -dc], axis=1)[..., None])[..., 0]
    lam = Jc @ np.linalg.solve(M, Jc.transpose(0, 2, 1)) + eps * np.eye(R) if R else np.ones((n, 1, 1))
    return x[:, :nd], x[:, nd:].reshape(n, K, dims), np.linalg.cond(lam)


def within(X, ref, kM, kA, tol=1e-13):
    """|X - ref| <= tol kappa_2(M) kappa_2(A) max|ref| elementwise."""
    return bool(np.all(np.abs(X - ref) <= tol * kM * kA * max(np.abs(ref).max(), 1e-300)))


def full_rank_table(model, q, dims, most=4):
    """A point table (links, local) of up to `most` points from the leaf links and the base whose J_c has full row rank at every
    configuration of q (singular values checked in numpy), greedy in the order of points(model)."""
    lk, lc = points(model)
    n, nd = q.shape[0], int(model[4])
    keep = []
    for i in range(len(lk)):
        trial = keep + [i]
        J = ep.point_motion(model, q, lk[trial], lc[trial])[0].reshape(n, 6 * len(trial), nd)[:, rows_of(len(trial), dims)]
        s = np.linalg.svd(J, compute_uv=False)
        if J.shape[1] <= nd and np.all(s[:, -1] > 1e-3 * s[:, 0]):
            keep = trial
        if len(keep) == most:
            break
    return lk[keep], lc[keep]


@pytest.mark.parametrize("name", ALL)
def test_unconstrained_is_the_solve_with_the_mass_matrix(name):
    """K = 0: qdd = M^-1 (tau - h) of numpy from the host-built M and h, and from the C oracle's; ID(q, qd, qdd) = tau."""
    model, q = fixture(name)
    n = q.shape[0]
    qd, tau = state(model, n)
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau)
    assert f.shape == (n, 0, 3)
    M, h = emu_mass.mass(model, q), emu_invdyn.inverse_dynamics(model, q, qd)
    kM = kappa(M)
    assert within(qdd, np.linalg.solve(M, (tau - h)[..., None])[..., 0], kM, 1.0), name
    back = emu_invdyn.inverse_dynamics(model, q, qd, qdd)   # (qdd rounded to fp32 on the way in)
    assert np.abs(back - tau).max() <= 4 * 2.0 ** -24 * np.abs(M).max() * np.abs(qdd).max() * M.shape[1] + 1e-12 * np.abs(tau).max()
    if name in ORACLE_FIXTURES:
        for e in range(min(n, 3)):
            Mo, ho = port.mass_matrix(model, f32(q[e])), emu_invdyn.oracle(model, f32(q[e]), qd[e])
            assert within(qdd[e], np.linalg.solve(Mo, tau[e] - ho), kM, 1.0, 1e-10), (name, e)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "humanoid_fixed"])
def test_unconstrained_is_the_forward_dynamics_step_on_fixed_bases(name):
    """K = 0 on a fixed base: the MODE_FD qdd of the C oracle's step (oracle.port.step), stiffness and damping included."""
    model, q = fixture(name)
    qd, tau = state(model, q.shape[0], 2)
    qdd, _ = ecd.constrained_dynamics(model, q, qd, tau)
    kM = kappa(emu_mass.mass(model, q))
    for e in range(q.shape[0]):
        ref = port.step(model, port.make_params(), 0, f32(q[e]), qd[e], tau[e])["qdd"]
        assert within(qdd[e], ref, kM, 1.0, 1e-10), (name, e, np.abs(qdd[e] - ref).max())


@pytest.mark.parametrize("name", ALL)
def test_jvp_along_tau_without_points_is_the_inverse_mass_matrix(name):
    """K = 0: the JVP along the identity tangents of tau is mass_inverse's M^-1, bit for bit (one term of each sum is non-zero)."""
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    qd, tau = state(model, n, 3)
    dqdd, _ = ecd.constrained_dynamics_jvp(model, q, qd, tau, t_tau=np.broadcast_to(np.eye(nd), (n, nd, nd)).copy())
    assert np.array_equal(dqdd, emi.mass_inverse(model, q)), name


@pytest.mark.parametrize("dims", [3, 6])
@pytest.mark.parametrize("name", ALL)
def test_against_the_kkt_solve(name, dims):
    """K > 0: qdd and f against numpy's KKT solve of the host-built M, h, J and drift within B, and of the C oracle's within 1e-10
    kappa kappa max; the residuals of both KKT rows."""
    model, q = fixture(name)
    n = q.shape[0]
    lk, lc = full_rank_table(model, q, dims, 4 if dims == 3 else 1)
    K = len(lk)
    if K == 0:
        pytest.skip("no point of the table has full row rank with these rows (a planar chain)")
    qd, tau = state(model, n, 4)
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, dims)
    M, h, J, d = host_pieces(model, q, qd, lk, lc)
    rq, rf, kA = kkt(M, h, J, d, tau, K, dims)
    kM, kA = kappa(M), float(kA.max())
    assert within(qdd, rq, kM, kA) and within(f, rf, kM, kA), (name, np.abs(qdd - rq).max(), np.abs(f - rf).max())
    sel = rows_of(K, dims)
    Jc = J[:, sel]
    r1 = np.einsum("eij,ej->ei", M, qdd) + h - tau - np.einsum("eji,ej->ei", Jc, f.reshape(n, -1))
    r2 = np.einsum("eij,ej->ei", Jc, qdd) + d[:, sel]
    assert np.abs(r1).max() <= 1e-13 * kM * kA * max(np.abs(tau - h).max(), np.abs(f).max() * np.abs(Jc).max())
    assert np.abs(r2).max() <= 1e-13 * kM * kA * max(1.0, np.abs(Jc).max() * np.abs(qdd).max())
    if name in ORACLE:
        for e in range(min(n, 3)):
            Mo, ho, Jo, do = oracle_pieces(model, f32(q[e]), qd[e], lk, lc)
            oq, of, _ = kkt(Mo[None], ho[None], Jo[None], do[None], tau[e:e + 1], K, dims)
            assert within(qdd[e], oq[0], kM, kA, 1e-10) and within(f[e], of[0], kM, kA, 1e-10), (name, e)


@pytest.mark.parametrize("dims", [3, 6])
@pytest.mark.parametrize("name", ["pendulum5spherical", "humanoid_fixed", "mb_three_bodies"])
def test_sign_of_f_through_the_step_with_wrenches(name, dims):
    """Fixed bases: the MODE_FD step with the wrenches W = f (dims 6) or [0; f] (dims 3) at the points, in fp64, reproduces qdd within the
    fp32 rounding of W: f is the force the constraint applies to the robot, in step_wrench's convention."""
    model, q = fixture(name)
    n, nd = q.shape[0], int(model[4])
    lk, lc = full_rank_table(model, q, dims, 4 if dims == 3 else 1)
    K = len(lk)
    assert K > 0
    qd, tau = state(model, n, 5)
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, dims)
    W = np.zeros((n, K, 6))
    W[:, :, 6 - dims:] = f
    ref = emu_wrench.step_wrench(model, 0, q, qd, tau, lk, lc, W, precision=1)
    M, _, J, _ = host_pieces(model, q, qd, lk, lc)
    MiJ = np.linalg.solve(M, J.transpose(0, 2, 1))
    bound = 4 * 2.0 ** -24 * np.abs(MiJ).max() * np.abs(f).max() * 6 * K + 1e-10 * np.abs(qdd).max()
    assert np.abs(ref - qdd).max() <= bound, (name, np.abs(ref - qdd).max(), bound)


@pytest.mark.parametrize("name", ["laikago", "humanoid", "ant"])
def test_damping(name):
    """eps > 0 against numpy's damped solve (J_c qdd = -d_c - eps f)."""
    model, q = fixture(name)
    lk, lc = full_rank_table(model, q, 3)
    K, n = len(lk), q.shape[0]
    qd, tau = state(model, n, 6)
    M, h, J, d = host_pieces(model, q, qd, lk, lc)
    for eps in (1e-6, 1e-2):
        qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3, eps)
        rq, rf, kA = kkt(M, h, J, d, tau, K, 3, eps)
        assert within(qdd, rq, kappa(M), float(kA.max())) and within(f, rf, kappa(M), float(kA.max())), (name, eps)


def test_rank_deficient_tables_give_nan_in_the_affected_environments_only():
    """A 3-row point on a planar chain at eps = 0 is structurally rank-deficient: NaN outputs; at eps > 0 finite.  In the kernels alone,
    an environment whose J_c is zero gets NaN while the others keep their values bit for bit."""
    model, q = fixture("pendulum5")
    n = q.shape[0]
    qd, tau = state(model, n, 7)
    lk, lc = np.array([int(model[1]) - 1]), np.array([[0.1, 0.0, 0.05]])
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3)
    assert np.all(np.isnan(qdd)) and np.all(np.isnan(f))
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3, 1e-3)
    assert np.all(np.isfinite(qdd)) and np.all(np.isfinite(f))
    model, q = fixture("laikago")
    n = q.shape[0]
    qd, tau = state(model, n, 8)
    lk, lc = full_rank_table(model, q, 3)
    K = len(lk)
    M, h, J, d = host_pieces(model, q, qd, lk, lc)
    Mi = emi.mass_inverse(model, q)
    ref = ecd.kernels(K, 3, 0.0, tau, h, Mi, J, d)
    J2 = J.copy()
    J2[1] = 0.0
    qdd, f = ecd.kernels(K, 3, 0.0, tau, h, Mi, J2, d)
    assert np.all(np.isnan(qdd[1])) and np.all(np.isnan(f[1]))
    keep = np.arange(n) != 1
    assert np.array_equal(qdd[keep], ref[0][keep]) and np.array_equal(f[keep], ref[1][keep])


@pytest.mark.parametrize("name", MB_WORLDS)
def test_worlds_of_several_multibodies(name):
    """Points on two multibodies against the KKT solve; a point on one multibody leaves the other's qdd at its K = 0 value within B."""
    model, q = fixture(name)
    n = q.shape[0]
    lk, lc = full_rank_table(model, q, 3)
    bodies = body_of(model, lk)
    assert len(set(bodies)) >= 2, bodies
    qd, tau = state(model, n, 9)
    M, h, J, d = host_pieces(model, q, qd, lk, lc)
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3)
    rq, rf, kA = kkt(M, h, J, d, tau, len(lk), 3)
    kM = kappa(M)
    assert within(qdd, rq, kM, float(kA.max())) and within(f, rf, kM, float(kA.max())), name
    free, _ = ecd.constrained_dynamics(model, q, qd, tau)
    one = [i for i, b in enumerate(bodies) if b == bodies[0]]
    qdd1, _ = ecd.constrained_dynamics(model, q, qd, tau, lk[one], lc[one], 3)
    Jone = J.reshape(n, len(lk), 6, -1)[:, one].reshape(n, -1, J.shape[2])
    other = ~np.any(Jone != 0.0, axis=(0, 1))   # the dofs the point's multibody does not own
    assert other.any()
    assert within(qdd1[:, other], free[:, other], kM, float(kA.max())), name


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_parameters(name):
    """A set at the model's values is bit-identical to no set; random +-20 % values per environment are bit-identical to the edited
    model."""
    model, q = fixture(name)
    n = q.shape[0]
    lk, lc = full_rank_table(model, q, 3)
    qd, tau = state(model, n, 10)
    ids = all_ids(model)
    a = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3, ids=ids, values=param_values(model)[ids])
    b = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    vals = perturbed(model, ids, n, 11, 0.5, 0.0)
    qdd, f = ecd.constrained_dynamics(model, q, qd, tau, lk, lc, 3, ids=ids, values=vals)
    for e in range(n):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        qe, fe = ecd.constrained_dynamics(edited, q[e:e + 1], qd[e:e + 1], tau[e:e + 1], lk, lc, 3)
        assert np.array_equal(qdd[e:e + 1], qe) and np.array_equal(f[e:e + 1], fe), (name, e)


def _kkt_oracle(model, q, qd, tau, lk, lc, dims):
    M, h, J, d = oracle_pieces(model, q, qd, lk, lc)
    qdd, f, _ = kkt(M[None], h[None], J[None], d[None], tau[None], len(lk), dims)
    return np.concatenate([qdd[0], f[0].ravel()])


@pytest.mark.parametrize("dims", [3, 6])
@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago", "humanoid"])
def test_jvp_against_central_differences_of_the_oracle(name, dims):
    """dqdd and df along random q, qd, tau and parameter tangents against central differences (h = 1e-6) of the KKT solve of the C
    oracle's M, h, J and drift on the edited model."""
    model, q = fixture(name)
    q = f32(q[:2])
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    lk, lc = full_rank_table(model, q, dims, 4 if dims == 3 else 1)
    qd, tau = state(model, n, 12)
    ids = _mass_ids(model)
    base = param_values(model)[ids]
    rng = np.random.default_rng(13)
    vq, vqd, vt = rng.normal(size=(n, n_q)), rng.normal(size=(n, nd)), rng.normal(size=(n, nd))
    vp = rng.normal(size=(n, len(ids))) * np.maximum(np.abs(base), 0.01)
    dqdd, df = ecd.constrained_dynamics_jvp(model, q, qd, tau, lk, lc, dims, 0.0, vq[..., None], vqd[..., None], vt[..., None],
                                            vp[..., None], ids=ids, values=base)
    got = np.concatenate([dqdd[..., 0], df[..., 0].reshape(n, -1)], axis=1)
    hs = 1e-6
    for e in range(n):
        F = lambda s: _kkt_oracle(set_param_values(model, ids, base + s * hs * vp[e]), q[e] + s * hs * vq[e], qd[e] + s * hs * vqd[e],
                                  tau[e] + s * hs * vt[e], lk, lc, dims)
        fd = (F(1) - F(-1)) / (2 * hs)
        assert np.all(np.abs(got[e] - fd) <= 1e-5 * max(1.0, np.abs(fd).max())), (name, e, np.abs(got[e] - fd).max(), np.abs(fd).max())


@pytest.mark.parametrize("name", ["laikago", "humanoid", "mb_racket"])
def test_tangents_of_one_call_are_independent_and_linear(name):
    """m tangents in one call are bit-identical to single calls; <G, J V> = <J^T G, V> with J^T G from the identity tangents, as the VJP
    contracts them."""
    model, q = fixture(name)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    lk, lc = full_rank_table(model, q, 3)
    R = 3 * len(lk)
    qd, tau = state(model, n, 14)
    ids = all_ids(model)[:6]
    vals = perturbed(model, ids, n, 15, 0.5, 0.0)
    rng = np.random.default_rng(16)
    V = [rng.normal(size=(n, d, 3)) for d in (n_q, nd, nd, len(ids))]
    run = lambda T: ecd.constrained_dynamics_jvp(model, q, qd, tau, lk, lc, 3, 0.0, *T, ids=ids, values=vals)
    dqdd, df = run(V)
    for j in range(3):
        a, b = run([v[..., j:j + 1] for v in V])
        assert np.array_equal(a[..., 0], dqdd[..., j]) and np.array_equal(b[..., 0], df[..., j]), j
    dims = (n_q, nd, nd, len(ids))
    total = sum(dims)
    eye = [np.zeros((n, d, total)) for d in dims]
    c0 = 0
    for E, d in zip(eye, dims):
        E[:, np.arange(d), c0 + np.arange(d)] = 1.0
        c0 += d
    eq, ef = run(eye)
    G = rng.normal(size=(n, nd + R))
    Jcols = np.concatenate([eq, ef.reshape(n, R, total)], axis=1)
    gT = np.einsum("er,erc->ec", G, Jcols)
    fwd = np.einsum("er,erm->em", G, np.concatenate([dqdd, df.reshape(n, R, 3)], axis=1))
    back = np.einsum("ec,ecm->em", gT, np.concatenate(V, axis=1))
    assert np.abs(fwd - back).max() <= 1e-9 * max(1.0, np.abs(fwd).max())
