"""The joint-space mass matrix M(q) (DESIGN.md section 7.12) on the CPU, from the kernel SOURCE: the MASS instances of csrc/tds_stepw.cu
compiled for the host (tests/cpp/mass_host.cpp, bound by tests/emu_mass.py) against the fp64 C oracle's restatement of mass_matrix.hpp,
structural checks on the models the oracle does not restate (spherical joints, worlds of several multibodies), M times the
forward-dynamics Jacobian in tau, per-environment parameters, and the derivatives (JVP against central differences of the oracle, the
independence of the tangents of one call, JVP / VJP duality).  tests/test_mass_matrix_gpu.py checks the same instances as nvcc builds
them."""
import os

import numpy as np
import pytest

from tds_b200.model import fixture_path, load_model, param_names, param_values, set_param_values
from oracle import port
import emu
import emu_mass
from test_params_on_host import all_ids, perturbed

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
N = 6
ORACLE_FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "laikago", "ant", "humanoid", "humanoid_fixed"]
OTHER_FIXTURES = ["pendulum5spherical", "humanoid_spherical", "mb_three_bodies", "mb_racket"]
HEADER, BASE, LINK = 16, 13, 34


def fixed_base(model):
    """The floating-base model with its base welded at the origin: 7 fewer coordinates, 6 fewer velocity dofs."""
    m = np.array(model, dtype=np.float64)
    n_links = int(m[1])
    m[2], m[3], m[4] = 0, m[3] - 7, m[4] - 6
    for i in range(n_links):
        o = HEADER + BASE + i * LINK
        if m[o + 1] >= 0:   # a moving joint: shift its coordinate indices
            m[o + 2] -= 7
            m[o + 3] -= 6
    return m


def fixture(name):
    """(model, q [N, n_q]) of a fixture at the golden vectors' configurations."""
    if name == "humanoid_fixed":
        model, q = fixture("humanoid")
        return fixed_base(model), q[:, 7:]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    model = g["model"] if name.startswith("mb_") else load_model(fixture_path(name))
    return model, g["q_in"][:N]


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def rel(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def oracle(model, q):
    return np.array([port.mass_matrix(model, x) for x in f32(q)])


@pytest.mark.parametrize("name", ORACLE_FIXTURES)
def test_against_the_c_oracle(name):
    model, q = fixture(name)
    M = emu_mass.mass(model, q)
    Mo = oracle(model, q)
    assert M.shape == Mo.shape == (q.shape[0], int(model[4]), int(model[4]))
    assert np.all(np.abs(M - Mo) <= 1e-10 * np.maximum(1.0, np.abs(Mo).max())), rel(M, Mo)
    assert np.array_equal(M, M.transpose(0, 2, 1))


@pytest.mark.parametrize("name", ORACLE_FIXTURES + OTHER_FIXTURES)
def test_symmetric_and_positive_definite(name):
    model, q = fixture(name)
    M = emu_mass.mass(model, q)
    assert np.array_equal(M, M.transpose(0, 2, 1))
    for e in range(M.shape[0]):
        np.linalg.cholesky(M[e])


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket"])
def test_world_is_block_diagonal_of_its_multibodies(name):
    """Each diagonal block equals the M of the multibody on its own; the blocks between multibodies are zero."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    model, q = g["model"], g["q_in"][:N]
    M = emu_mass.mass(model, q)
    n_bodies = int(model[12])
    assert n_bodies >= 2
    # split the world back into its multibodies (one root link each, links in order)
    n_links = int(model[1])
    links = model[HEADER + BASE:HEADER + BASE + n_links * LINK].reshape(n_links, LINK)
    roots = [i for i in range(n_links) if links[i, 0] < 0] + [n_links]
    qo = do = 0
    for b in range(n_bodies):
        sub = links[roots[b]:roots[b + 1]].copy()
        moving = sub[:, 1] >= 0
        # the body's coordinates run up to the first index of the next body (merge_models concatenates them in order)
        later = links[roots[b + 1]:]
        later = later[later[:, 1] >= 0]
        nq_b = (int(later[:, 2].min()) if later.size else int(model[3])) - qo
        nd_b = (int(later[:, 3].min()) if later.size else int(model[4])) - do
        sub[:, 0] = np.where(sub[:, 0] >= 0, sub[:, 0] - roots[b], -1)
        sub[moving, 2] -= qo
        sub[moving, 3] -= do
        single = np.concatenate([model[:HEADER], model[HEADER:HEADER + BASE], sub.ravel()])
        single[1], single[3], single[4], single[5], single[6], single[7], single[12] = roots[b + 1] - roots[b], nq_b, nd_b, 0, 0, 0, 0
        Mb = emu_mass.mass(single, q[:, qo:qo + nq_b])
        # (equal up to rounding, not bit for bit: the kernel's common-frame origin O of the world is the end of the first multibody's
        # translation chain, the single multibody's is its own)
        assert np.abs(M[:, do:do + nd_b, do:do + nd_b] - Mb).max() <= 1e-12 * max(1.0, np.abs(Mb).max()), (name, b)
        rest = np.ones(M.shape[1], dtype=bool)
        rest[do:do + nd_b] = False
        assert np.all(M[:, do:do + nd_b][:, :, rest] == 0.0)
        qo += nq_b
        do += nd_b
    assert (qo, do) == (int(model[3]), int(model[4]))


def test_inverse_of_the_forward_dynamics_jacobian_on_the_c_oracle():
    """M dqdd/dtau = I on the C oracle (central differences of its forward-dynamics step): the identity the kernel check below relies on.
    It holds for fixed bases only; the reference's floating-base forward dynamics (base-frame quirks, kinematics.hpp:54-61,
    inertia.hpp:302-328) does not invert its mass matrix, so the floating-base humanoid is the counter-example pinned here."""
    P = port.make_params()
    for name, holds in (("pendulum5", True), ("laikago", True), ("humanoid", False)):
        model = load_model(fixture_path(name))
        g = np.load(os.path.join(GOLDEN, name + ".npz"))
        n_qd, fl = int(model[4]), int(model[2])
        n_tau = n_qd - (6 if fl else 0)
        q, qd = g["q_in"][0], g["qd_in"][0]
        M = port.mass_matrix(model, q)
        h, J = 1e-3, np.zeros((n_qd, n_tau))
        for c in range(n_tau):
            t = np.zeros(n_tau)
            t[c] = h
            J[:, c] = (port.step(model, P, 0, q, qd, t)["qdd"] - port.step(model, P, 0, q, qd, -t)["qdd"]) / (2 * h)
        err = np.abs(M @ J - np.eye(n_qd)[:, n_qd - n_tau:]).max()
        assert (err <= 1e-9) == holds, (name, err)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "laikago", "ant", "humanoid_fixed", "pendulum5spherical", "humanoid_spherical",
                                  "mb_three_bodies", "mb_racket"])
def test_inverse_of_the_dual_forward_dynamics_jacobian(name):
    """M dqdd/dtau (the MODE_FD dual Jacobian of the same kernel source) is the identity within 1e-9: fixed-base models only (see the
    oracle check above)."""
    model, q = fixture(name)
    n_q, n_qd = int(model[3]), int(model[4])
    qd = np.random.default_rng(3).normal(size=(q.shape[0], n_qd)) * 0.3
    tau = np.zeros((q.shape[0], n_qd))
    J = emu.step(model, 0, q, qd, tau, jacobian=True)["jac"][:, :, n_q + n_qd:]
    M = emu_mass.mass(model, q)
    assert np.abs(M @ J - np.eye(n_qd)).max() <= 1e-9


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_parameters_at_the_model_values_are_bit_identical(name):
    model, q = fixture(name)
    ids = all_ids(model)
    vals = param_values(model)[ids]
    assert np.array_equal(emu_mass.mass(model, q, ids=ids, values=vals), emu_mass.mass(model, q))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_per_environment_parameters_equal_edited_models(name):
    """Random per-environment values (+-20 %) are bit-identical to the instance without parameters on the flat model edited with those
    values, and within 1e-10 of the oracle on the edited model where the oracle restates it."""
    model, q = fixture(name)
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 9, 0.5, 0.0)
    M = emu_mass.mass(model, q, ids=ids, values=vals)
    for e in range(q.shape[0]):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        assert np.array_equal(M[e:e + 1], emu_mass.mass(edited, q[e:e + 1])), (name, e)
        if name in ORACLE_FIXTURES:
            Mo = port.mass_matrix(edited, f32(q[e]))
            assert np.all(np.abs(M[e] - Mo) <= 1e-10 * max(1.0, np.abs(Mo).max()))


def _mass_ids(model):
    """The parameter ids that enter M: the bodies' masses, centres of mass and inertias (not friction, restitution, stiffness, damping)."""
    names = param_names(model)
    return [i for i in all_ids(model) if names[i].startswith(("base.", "link")) and not names[i].endswith(("stiffness", "damping"))]


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_fixed"])
def test_jvp_against_central_differences_of_the_oracle(name):
    """dM along random q and parameter tangents against (M(x + h v) - M(x - h v)) / 2h of the C oracle on the edited model, h = 1e-6."""
    model, q = fixture(name)
    q = f32(q[:3])
    ids = _mass_ids(model)
    base = param_values(model)[ids]
    rng = np.random.default_rng(17)
    vq = rng.normal(size=(q.shape[0], q.shape[1]))
    vp = rng.normal(size=(q.shape[0], len(ids))) * np.maximum(np.abs(base), 0.01)
    dM = emu_mass.mass_jvp(model, q, vq[:, :, None], vp[:, :, None], ids=ids, values=base)[..., 0]
    h = 1e-6
    for e in range(q.shape[0]):
        Mp = port.mass_matrix(set_param_values(model, ids, base + h * vp[e]), q[e] + h * vq[e])
        Mm = port.mass_matrix(set_param_values(model, ids, base - h * vp[e]), q[e] - h * vq[e])
        fd = (Mp - Mm) / (2 * h)
        assert np.all(np.abs(dM[e] - fd) <= 1e-6 * np.maximum(1.0, np.abs(fd).max())), (name, e, np.abs(dM[e] - fd).max())


@pytest.mark.parametrize("name", ["pendulum5", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_racket"])
def test_tangents_of_one_call_are_independent(name):
    """m tangents in one call are bit-identical to m calls with one tangent each; identity tangents give the value of each column."""
    model, q = fixture(name)
    ids = all_ids(model)[:12]
    vals = perturbed(model, ids, q.shape[0], 4, 0.5, 0.0)
    rng = np.random.default_rng(5)
    vq, vp = rng.normal(size=(q.shape[0], q.shape[1], 3)), rng.normal(size=(q.shape[0], len(ids), 3))
    dM = emu_mass.mass_jvp(model, q, vq, vp, ids=ids, values=vals)
    for j in range(3):
        one = emu_mass.mass_jvp(model, q, vq[:, :, j:j + 1], vp[:, :, j:j + 1], ids=ids, values=vals)
        assert np.array_equal(one[..., 0], dM[..., j])


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "laikago", "humanoid", "humanoid_spherical", "mb_three_bodies"])
def test_vjp_is_the_adjoint_of_the_jvp(name):
    """<G, dM[v]> = <VJP(G), v> within 1e-10, over q and the installed parameters together."""
    model, q = fixture(name)
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 8, 0.5, 0.0)
    rng = np.random.default_rng(6)
    n, nd = q.shape[0], int(model[4])
    G = rng.normal(size=(n, nd, nd))
    vq, vp = rng.normal(size=(n, q.shape[1])), rng.normal(size=(n, len(ids)))
    dM = emu_mass.mass_jvp(model, q, vq[:, :, None], vp[:, :, None], ids=ids, values=vals)[..., 0]
    g_q, g_par = emu_mass.mass_vjp(model, q, G, ids=ids, values=vals)
    fwd = np.einsum("eij,eij->e", G, dM)
    rev = np.einsum("ec,ec->e", g_q, vq) + np.einsum("ek,ek->e", g_par, vp)
    assert rel(fwd, rev) <= 1e-10
    # without installed parameters: g_q alone, the same q part
    g_q0, g_p0 = emu_mass.mass_vjp(model, q, G)
    assert g_p0.shape == (n, 0)
    dM0 = emu_mass.mass_jvp(model, q, vq[:, :, None])[..., 0]
    assert rel(np.einsum("eij,eij->e", G, dM0), np.einsum("ec,ec->e", g_q0, vq)) <= 1e-10
