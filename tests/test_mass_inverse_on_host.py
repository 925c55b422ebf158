"""The inverse mass matrix M^-1(q) and the operational-space inverse inertia J M^-1 J^T (DESIGN.md section 7.20) on the CPU, from the
kernel SOURCE: the MINV instances of csrc/tds_stepw.cu and the contraction kernel of csrc/tds_mass_inverse.cu compiled for the host
(tests/cpp/mass_inverse_host.cpp, bound by tests/emu_mass_inverse.py) against numpy's inverse of the host-built M and of the C oracle's
M, the forward-dynamics Jacobian on fixed bases, per-environment parameters, J M^-1 J^T assembled in numpy from the host-built point
Jacobians, and the derivatives (against -M^-1 dM M^-1, the product rule, and central differences of the oracle).  Every tolerance on
M^-1 and what is built from it scales with the condition number kappa_2(M): B = 1e-13 kappa max|ref| elementwise.
tests/test_mass_inverse_gpu.py checks the same instances as nvcc builds them."""
import numpy as np
import pytest

from tds_b200.model import param_values, set_param_values
from oracle import port
import emu
import emu_mass
import emu_mass_inverse as emi
import emu_point_motion
from test_mass_matrix_on_host import ORACLE_FIXTURES, OTHER_FIXTURES, _mass_ids, f32, fixture, oracle
from test_params_on_host import all_ids, perturbed

ALL = ORACLE_FIXTURES + OTHER_FIXTURES
MB_WORLDS = ["mb_three_bodies", "mb_racket"]


def kappa(M):
    return float(np.linalg.cond(M).max())


def within_b(X, ref, kap):
    """|X - ref| <= 1e-13 kappa max|ref| elementwise."""
    return bool(np.all(np.abs(X - ref) <= 1e-13 * kap * np.abs(ref).max()))


def points(model):
    """A point table of up to 4 leaf links (and the floating base): links [K], local [K, 3]."""
    nl = int(model[1])
    parents = [int(model[16 + 13 + i * 34]) for i in range(nl)]
    leaves = [i for i in range(nl) if i not in parents][-4:]
    links = leaves + ([-1] if int(model[2]) else [])
    if not links:
        links = [nl - 1]
    local = np.array([[0.1, 0.05, -0.02]] * len(links)) * (1 + np.arange(len(links)))[:, None] * 0.5
    return np.array(links), local


def body_of(model, links):
    """The multibody (index of its root link among the roots) of each point's link."""
    nl = int(model[1])
    roots = [i for i in range(nl) if int(model[16 + 13 + i * 34]) < 0]
    return [max(b for b, r in enumerate(roots) if r <= lk) for lk in links]


@pytest.mark.parametrize("name", ALL)
def test_inverse_of_the_mass_matrix(name):
    """M^-1 against numpy's inverse of the host-built M (and of the C oracle's M), bitwise symmetric, positive definite, M M^-1 = I."""
    model, q = fixture(name)
    M = emu_mass.mass(model, q)
    Mi = emi.mass_inverse(model, q)
    kap = kappa(M)
    assert within_b(Mi, np.linalg.inv(M), kap), (name, kap)
    if name in ORACLE_FIXTURES:
        Mo = oracle(model, q)
        assert within_b(Mi, np.linalg.inv(Mo), kappa(Mo)), name
    assert np.array_equal(Mi, Mi.transpose(0, 2, 1))
    for e in range(Mi.shape[0]):
        np.linalg.cholesky(Mi[e])
    assert np.abs(M @ Mi - np.eye(M.shape[1])).max() <= 1e-13 * kap


@pytest.mark.parametrize("name", MB_WORLDS)
def test_world_is_block_diagonal(name):
    """Exact zeros between the multibodies of a world; each diagonal block is the inverse of its multibody's block of M."""
    model, q = fixture(name)
    M = emu_mass.mass(model, q)
    Mi = emi.mass_inverse(model, q)
    nd = M.shape[1]
    # the multibodies' dof ranges: the connected blocks of M's sparsity
    nz = np.any(M != 0.0, axis=0)
    owner = np.arange(nd)
    for r in range(nd):
        for c in range(r):
            if nz[r, c]:
                owner[owner == owner[r]] = owner[c]
    blocks = [np.flatnonzero(owner == o) for o in np.unique(owner)]
    assert len(blocks) >= 2
    for b in blocks:
        rest = np.setdiff1d(np.arange(nd), b)
        assert np.all(Mi[:, b][:, :, rest] == 0.0)
        Mb = M[:, b][:, :, b]
        assert within_b(Mi[:, b][:, :, b], np.linalg.inv(Mb), kappa(Mb)), name


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "ant", "humanoid_fixed", "pendulum5spherical", "humanoid_spherical",
                                  "mb_three_bodies", "mb_racket"])
def test_equals_the_forward_dynamics_jacobian_on_fixed_bases(name):
    """M^-1 = dqdd/dtau, the MODE_FD dual Jacobian of the same kernel source, within 1e-8 max|M^-1| (fixed bases only: DESIGN.md 7.12)."""
    model, q = fixture(name)
    n_q, n_qd = int(model[3]), int(model[4])
    qd = np.random.default_rng(3).normal(size=(q.shape[0], n_qd)) * 0.3
    J = emu.step(model, 0, q, qd, np.zeros((q.shape[0], n_qd)), jacobian=True)["jac"][:, :, n_q + n_qd:]
    Mi = emi.mass_inverse(model, q)
    assert np.abs(Mi - J).max() <= 1e-8 * np.abs(Mi).max()


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_parameters(name):
    """The model's own values are bit-identical to no set; random +-20 % values per environment are bit-identical to the edited model."""
    model, q = fixture(name)
    ids = all_ids(model)
    assert np.array_equal(emi.mass_inverse(model, q, ids=ids, values=param_values(model)[ids]), emi.mass_inverse(model, q))
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    Mi = emi.mass_inverse(model, q, ids=ids, values=vals)
    for e in range(q.shape[0]):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert np.array_equal(Mi[e:e + 1], emi.mass_inverse(edited, q[e:e + 1])), (name, e)


@pytest.mark.parametrize("name", ALL)
def test_operational_space_inverse_inertia(name):
    """J M^-1 J^T against numpy from the host builds of MOT and MASS, exactly symmetric, positive semi-definite, zero between points on
    different multibodies."""
    model, q = fixture(name)
    links, local = points(model)
    J = emu_point_motion.point_motion(model, q, links, local)[0].reshape(q.shape[0], -1, int(model[4]))
    M = emu_mass.mass(model, q)
    L = emi.osim(J, emi.mass_inverse(model, q))
    ref = J @ np.linalg.inv(M) @ J.transpose(0, 2, 1)
    assert within_b(L, ref, kappa(M)), name
    assert np.array_equal(L, L.transpose(0, 2, 1))
    for e in range(L.shape[0]):
        assert np.linalg.eigvalsh(L[e]).min() >= -1e-12 * np.abs(L[e]).max()
    if name in MB_WORLDS:
        b = np.repeat(body_of(model, links), 6)
        assert np.all(L[:, b[:, None] != b[None, :]] == 0.0)


@pytest.mark.parametrize("name", ["sphere2", "box"])
def test_free_body_at_its_centre_of_mass(name):
    """One free body, the point at its centre of mass: J M^-1 J^T = blockdiag(I_world^-1, 1/m I3), which pins the base columns."""
    model, q = fixture(name)
    pv = param_values(model)
    m, I = pv[2], np.array([[pv[6], pv[7], pv[8]], [pv[7], pv[9], pv[10]], [pv[8], pv[10], pv[11]]])
    com = pv[3:6]
    L = emi.osim(emu_point_motion.point_motion(model, q, [-1], com[None])[0], emi.mass_inverse(model, q))
    for e in range(q.shape[0]):
        R = emu_point_motion.oracle_motion(model, f32(q[e]), None, None)[0][0]
        ref = np.zeros((6, 6))
        ref[:3, :3] = np.linalg.inv(R @ I @ R.T)
        ref[3:, 3:] = np.eye(3) / m
        assert within_b(L[e], ref, kappa(emu_mass.mass(model, q[e:e + 1]))), (name, e, np.abs(L[e] - ref).max())


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_jvp_is_minus_minv_dm_minv(name):
    """dM^-1 = -M^-1 dM M^-1 (dM from the mass matrix's JVP) along q and parameter tangents, and dLambda^-1 = dJ M^-1 J^T + J dM^-1 J^T
    + J M^-1 dJ^T from the point-motion JVP; m tangents in one call bit-identical to single calls."""
    model, q = fixture(name)
    ids = _mass_ids(model)[:12]
    vals = param_values(model)[ids]
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    rng = np.random.default_rng(11)
    vq, vp = rng.normal(size=(n, n_q, 3)), rng.normal(size=(n, len(ids), 3)) * np.maximum(np.abs(vals), 0.01)[None, :, None]
    dMi = emi.mass_inverse_jvp(model, q, vq, vp, ids=ids, values=vals)
    dM = emu_mass.mass_jvp(model, q, vq, vp, ids=ids, values=vals)
    Mi = emi.mass_inverse(model, q)
    kap = kappa(emu_mass.mass(model, q))
    ref = -np.einsum("eij,ejkm,ekl->eilm", Mi, dM, Mi)
    assert np.all(np.abs(dMi - ref) <= 1e-13 * kap * np.abs(Mi).max() ** 2 * np.abs(dM).max()), name
    for j in range(3):
        one = emi.mass_inverse_jvp(model, q, vq[:, :, j:j + 1], vp[:, :, j:j + 1], ids=ids, values=vals)
        assert np.array_equal(one[..., 0], dMi[..., j])
    links, local = points(model)
    K = len(links)
    J = emu_point_motion.point_motion(model, q, links, local)[0].reshape(n, 6 * K, nd)
    tin = np.concatenate([vq, np.zeros((n, 2 * nd, 3))], axis=1)
    dJ = emu_point_motion.point_motion_jvp(model, q, links, local, tin)[:, :6 * K * nd].reshape(n, 6 * K, nd, 3)
    dL = emi.osim(J, Mi, dJ, dMi)
    refL = (np.einsum("eajm,ejk,ebk->eabm", dJ, Mi, J) + np.einsum("eaj,ejkm,ebk->eabm", J, dMi, J)
            + np.einsum("eaj,ejk,ebkm->eabm", J, Mi, dJ))
    assert within_b(dL, refL, kap), name
    assert np.array_equal(dL, dL.transpose(0, 2, 1, 3))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_fixed"])
def test_jvp_against_central_differences_of_the_oracle(name):
    """dM^-1 along random q and parameter tangents against central differences (h = 1e-6) of inv(M) of the C oracle on the edited
    model."""
    model, q = fixture(name)
    q = f32(q[:3])
    ids = _mass_ids(model)
    base = param_values(model)[ids]
    rng = np.random.default_rng(17)
    vq = rng.normal(size=(q.shape[0], q.shape[1]))
    vp = rng.normal(size=(q.shape[0], len(ids))) * np.maximum(np.abs(base), 0.01)
    dMi = emi.mass_inverse_jvp(model, q, vq[:, :, None], vp[:, :, None], ids=ids, values=base)
    h = 1e-6
    for e in range(q.shape[0]):
        inv = lambda s: np.linalg.inv(port.mass_matrix(set_param_values(model, ids, base + s * h * vp[e]), q[e] + s * h * vq[e]))
        fd = (inv(1) - inv(-1)) / (2 * h)
        assert np.all(np.abs(dMi[e, :, :, 0] - fd) <= 1e-6 * max(1.0, np.abs(fd).max())), (name, e)
