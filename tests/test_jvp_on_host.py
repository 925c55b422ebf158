"""Forward mode of the step kernels (Jacobian-vector products by the tangent-seeded dual instances, DESIGN.md section 7.10) executed
on the CPU from their SOURCE (tests/cpp/stepw_jvp_host.cpp, tests/cpp/rigid_jvp_host.cpp): identity tangents against the dual-number
Jacobian of the same source, random tangents against J V, independence of the tangents of one call, duality with the taping
instance, central differences of the fp64 C oracle, and the whole-rollout JVP of the rigid-body worlds.  tests/test_jvp_gpu.py checks
the same instances as nvcc builds them."""
import os

import numpy as np
import pytest

import tds_b200.envs as envs
import tds_b200.workloads as wl
from tds_b200.model import fixture_path, load_model
from oracle import port
import emu
import emu_jvp
import emu_params
import emu_vjp
from test_params_on_host import all_ids, fd_case, perturbed
from test_kernel_source_on_host import GOLDEN
from test_vjp_on_host import golden_case, pd_env

FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "cartpole_plane", "pendulum5spherical", "humanoid", "humanoid_spherical",
            "laikago_pd", "ant_pd", "spring_damper", "mb_three_bodies", "mb_racket"]
PARAM_FIXTURES = ["pendulum5", "cartpole", "sphere2", "box", "laikago_pd", "humanoid", "mb_three_bodies", "humanoid_spherical"]
N = 6


def rel(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def case(name):
    """(model, mode, q, qd, tau, kw) of a fixture, N environments; kw holds use_pd / env and the solver parameters."""
    if name in ("laikago_pd", "ant_pd"):   # as tests/test_vjp_on_host.py's PD check
        robot = name[:-3]
        g = np.load(os.path.join(GOLDEN, robot + ".npz"))
        params = dict(dt=1e-3 if robot == "laikago" else envs.ANT_DT, friction=1.0, keep_all_points=True)
        return load_model(fixture_path(robot)), 2, g["q_in"][:N], g["qd_in"][:N], g["action"][:N], dict(use_pd=True, env=pd_env(robot), **params)
    if name == "spring_damper":
        model, _, q, qd, tau, params = golden_case("sphere2")
        law = dict(contact_model=1, spring_k=40000.0, damper_d=3000.0, exponent_n=1.5, v_transition=0.02, hard_contact_condition=True)
        return model, 2, q[:N], qd[:N], None if tau is None else tau[:N], dict(law, **params)
    model, mode, q, qd, tau, params = golden_case(name)
    if name.startswith("mb_"):
        mode = 2
    return model, mode, q[:N], qd[:N], None if tau is None else tau[:N], dict(params)


def rel_jv(out, J, V):
    """|t_out - J V| relative to the size of the products summed, sum_c |J_rc| |V_cj| (at least 1): the rounding bound of a
    contraction, whose terms may cancel."""
    return float(np.max(np.abs(out - np.einsum("erc,ecj->erj", J, V)) / np.maximum(1.0, np.einsum("erc,ecj->erj", np.abs(J), np.abs(V)))))


def jacobian(model, mode, q, qd, tau, kw):
    return emu.step(model, mode, q, qd, tau, jacobian=True, **kw)["jac"]


@pytest.mark.parametrize("name", FIXTURES)
def test_identity_tangents_are_bit_identical_to_the_dual_jacobian(name):
    model, mode, q, qd, tau, kw = case(name)
    J = jacobian(model, mode, q, qd, tau, kw)
    n, rows, cols = J.shape
    eye = np.ascontiguousarray(np.broadcast_to(np.eye(cols), (n, cols, cols)))
    out = emu_jvp.step_jvp(model, mode, q, qd, t_in=eye, tau=tau, **kw)
    assert np.array_equal(out, J), rel(out, J)


@pytest.mark.parametrize("name", FIXTURES)
def test_random_tangents_equal_J_V_and_are_independent(name):
    model, mode, q, qd, tau, kw = case(name)
    J = jacobian(model, mode, q, qd, tau, kw)
    n, rows, cols = J.shape
    V = np.random.default_rng(21).normal(size=(n, cols, 3))
    out = emu_jvp.step_jvp(model, mode, q, qd, t_in=V, tau=tau, **kw)
    assert rel_jv(out, J, V) <= 1e-12
    # m tangents in one call are m calls of one tangent each, bit for bit
    for j in range(3):
        one = emu_jvp.step_jvp(model, mode, q, qd, t_in=V[:, :, j:j + 1], tau=tau, **kw)
        assert np.array_equal(one[:, :, 0], out[:, :, j])


@pytest.mark.parametrize("name", FIXTURES)
def test_duality_with_the_taping_instance(name):
    """<g, J v> of forward mode against <J^T g, v> of reverse mode: two instances of the same source, no Jacobian in between."""
    model, mode, q, qd, tau, kw = case(name)
    n_q, n_qd = int(model[3]), int(model[4])
    rows = n_qd if mode == 0 else n_q + n_qd
    rng = np.random.default_rng(22)
    g = rng.normal(size=(q.shape[0], rows))
    g_in, _ = emu_vjp.step_vjp(model, mode, q, qd, g, tau, **kw)
    v = rng.normal(size=g_in.shape)
    jv = emu_jvp.step_jvp(model, mode, q, qd, t_in=v[:, :, None], tau=tau, **kw)[:, :, 0]
    fwd, rev = np.einsum("er,er->e", g, jv), np.einsum("ec,ec->e", g_in, v)
    assert rel(fwd, rev) <= 1e-10


def param_case(name):
    model, mode, q, qd, tau, params, use_pd, env = fd_case(name)
    if name in ("mb_three_bodies", "humanoid_spherical"):
        mode = 2
    ids = all_ids(model)
    vals = perturbed(model, ids, q.shape[0], 7, params.get("friction", 0.5), params.get("restitution", 0.0))
    return model, mode, q, qd, tau, dict(use_pd=use_pd, env=env, ids=ids, values=vals, **params)


@pytest.mark.parametrize("name", PARAM_FIXTURES)
def test_parameter_tangents(name):
    """Identity tangents over the installed parameters are the dual parameter Jacobian bit for bit; random input and parameter
    tangents together give J V + J_par W; duality with the taping instance's g_in and g_par."""
    model, mode, q, qd, tau, kw = param_case(name)
    k = len(kw["ids"])
    Jp = emu_params.step(model, mode, q, qd, tau, what="param_jacobian", **kw)["jac"]
    Ji = emu_params.step(model, mode, q, qd, tau, what="jacobian", **kw)["jac"]
    n, rows, cols = Ji.shape
    eye = np.ascontiguousarray(np.broadcast_to(np.eye(k), (n, k, k)))
    out = emu_jvp.step_jvp(model, mode, q, qd, t_par=eye, tau=tau, **kw)
    assert np.array_equal(out, Jp), rel(out, Jp)
    rng = np.random.default_rng(23)
    V, W = rng.normal(size=(n, cols, 3)), rng.normal(size=(n, k, 3))
    out = emu_jvp.step_jvp(model, mode, q, qd, t_in=V, t_par=W, tau=tau, **kw)
    assert rel_jv(out, np.concatenate([Ji, Jp], axis=2), np.concatenate([V, W], axis=1)) <= 1e-12
    g = rng.normal(size=(n, rows))
    r = emu_params.step(model, mode, q, qd, tau, what="vjp", g_out=g, **kw)
    fwd = np.einsum("er,er->e", g, out[:, :, 0])
    rev = np.einsum("ec,ec->e", r["g_in"], V[:, :, 0]) + np.einsum("ek,ek->e", r["g_par"], W[:, :, 0])
    assert rel(fwd, rev) <= 1e-10


@pytest.mark.parametrize("name,gen,frac", [("pendulum5", wl.pendulum5, 1.0), ("cartpole", wl.cartpole, 1.0), ("sphere2", wl.sphere2, 0.9)])
def test_jvp_vs_central_differences_of_the_c_oracle(name, gen, frac):
    """J v against (f(x + h v) - f(x - h v)) / 2h of the fp64 C oracle along the same random v, h = 1e-6."""
    n = 20
    model = load_model(fixture_path(name))
    w = gen(n, seed=31)
    mode, tau = w["mode"], w.get("tau")
    n_q, n_qd = int(model[3]), int(model[4])
    n_tau = n_qd - (6 if int(model[2]) else 0)
    t = None if tau is None or not n_tau else tau[:, -n_tau:]
    cols = n_q + n_qd + n_tau
    rng = np.random.default_rng(33)
    V = rng.normal(size=(n, cols))
    jv = emu_jvp.step_jvp(model, mode, w["q"], w["qd"], t_in=V[:, :, None], tau=t, **w["params"])[:, :, 0]
    P = port.make_params(**w["params"])

    def f(x):
        r = port.step(model, P, mode, x[:n_q], x[n_q:n_q + n_qd], x[n_q + n_qd:] if n_tau else None)
        return r["qdd"] if mode == 0 else np.concatenate([r["q"], r["qd"]])
    ok = []
    h = 1e-6
    for e in range(n):
        x0 = np.concatenate([w["q"][e], w["qd"][e], t[e] if t is not None else np.zeros(0)])
        fd = (f(x0 + h * V[e]) - f(x0 - h * V[e])) / (2 * h)
        ok.append(np.all(np.abs(jv[e] - fd) <= 1e-4 * np.maximum(1.0, np.abs(fd))))
    assert np.mean(ok) >= frac, np.mean(ok)


@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3, 20])
def test_rigid_jvp_of_the_whole_rollout(kind, steps):
    w = wl.rigid_world(kind, 6, seed=41)
    out, J = emu.rigid_step(w["bodies"], w["state"], w["force"], steps, jacobian=True, **w["params"])
    n, rows, cols = J.shape
    nb = rows // 13
    # identity tangents over state | force: the dual Jacobian, bit for bit (and the end state of the rollout)
    eye = np.broadcast_to(np.eye(cols), (n, cols, cols))
    ts = eye[:, :rows].reshape(n, nb, 13, cols)
    tf = eye[:, rows:].reshape(n, nb, 3, cols)
    so, to = emu_jvp.rigid_jvp(w["bodies"], w["state"], ts, tf, w["force"], steps, **w["params"])
    assert np.array_equal(to.reshape(n, rows, cols), J)
    assert np.array_equal(so, out)
    # random tangents: J V
    rng = np.random.default_rng(43)
    V = rng.normal(size=(n, cols, 3))
    _, to = emu_jvp.rigid_jvp(w["bodies"], w["state"], V[:, :rows].reshape(n, nb, 13, 3), V[:, rows:].reshape(n, nb, 3, 3), w["force"],
                              steps, **w["params"])
    assert rel_jv(to.reshape(n, rows, 3), J, V) <= 1e-12
    # duality with the checkpointed reverse pass
    g = rng.normal(size=(n, rows))
    gs, gf, _ = emu_vjp.rigid_vjp(w["bodies"], w["state"], g, w["force"], steps, **w["params"])
    fwd = np.einsum("er,er->e", g, to.reshape(n, rows, 3)[:, :, 0])
    rev = np.einsum("ec,ec->e", np.concatenate([gs.reshape(n, -1), gf.reshape(n, -1)], axis=1), V[:, :, 0])
    assert rel(fwd, rev) <= 1e-10
