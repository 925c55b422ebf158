"""Reverse mode of the step kernels (vector-Jacobian products by the taping instance, csrc/tds_tape.cuh) executed on the CPU from
their SOURCE (tests/cpp/stepw_vjp_host.cpp, tests/cpp/rigid_vjp_host.cpp; the dual-number instances through
tests/cpp/stepw_host.cpp, tests/cpp/rigid_host.cpp): against g^T J of the dual-number instance of the same source on
every fixture, against central differences of the fp64 C oracle, tape regrowth, the checkpointed rigid-world rollout and the
billiard optimisation of the reference's python/examples/billiard_optimization.py.  tests/test_vjp_gpu.py checks the same kernels
as nvcc builds them."""
import os

import numpy as np
import pytest

import tds_b200.envs as envs
import tds_b200.workloads as wl
from tds_b200.model import fixture_path, load_model
from oracle import port
import emu
import emu_vjp
from test_kernel_source_on_host import CONFIGS, GOLDEN, params_from_golden

HERE = os.path.dirname(os.path.abspath(__file__))


def vjp_err(v, ref):
    return float(np.max(np.abs(v - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def golden_case(name):
    """(model, mode, q, qd, tau, params) of a golden fixture in its golden mode."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    model = g["model"] if name.startswith("mb_") else load_model(fixture_path(name))
    mode = int(g["mode"]) if "mode" in g.files else 2
    tau = g["tau"] if "tau" in g.files else None
    n_tau = int(model[4]) - (6 if int(model[2]) else 0)
    if tau is not None and tau.shape[1] != n_tau:
        tau = tau[:, -n_tau:]
    return model, mode, g["q_in"], g["qd_in"], tau if n_tau else None, params_from_golden(g)


def check_vjp_vs_dual(model, mode, q, qd, tau, seed, tol=1e-10, **kw):
    J = emu.step(model, mode, q, qd, tau, jacobian=True, **kw)["jac"]
    g = np.random.default_rng(seed).normal(size=J.shape[:2])
    v, st = emu_vjp.step_vjp(model, mode, q, qd, g, tau, **kw)
    ref = np.einsum("er,erc->ec", g, J)
    assert v.shape == ref.shape
    assert vjp_err(v, ref) <= tol, vjp_err(v, ref)
    return st


@pytest.mark.parametrize("name", CONFIGS)
def test_vjp_equals_gT_J_of_the_dual_instance_on_the_fixtures(name):
    model, mode, q, qd, tau, params = golden_case(name)
    check_vjp_vs_dual(model, mode, q, qd, tau, 11, **params)


def pd_env(name):
    poses = envs.LAIKAGO_INITIAL_POSES if name == "laikago" else envs.ANT_INITIAL_POSES
    kp, kd, mf = (envs.LAIKAGO_KP, envs.LAIKAGO_KD, envs.LAIKAGO_MAX_FORCE) if name == "laikago" else (envs.ANT_KP, envs.ANT_KD, envs.ANT_MAX_FORCE)
    return np.array([len(poses), 6, kp, kd, mf, 0.4, *poses])


@pytest.mark.parametrize("name", ["laikago", "ant"])
def test_vjp_with_pd_control_includes_the_gain_columns(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    model = load_model(fixture_path(name))
    params = dict(dt=1e-3 if name == "laikago" else envs.ANT_DT, friction=1.0, keep_all_points=True)
    st = check_vjp_vs_dual(model, 2, g["q_in"], g["qd_in"], g["action"], 12, use_pd=True, env=pd_env(name), **params)
    assert np.all(st["nodes"] > 0)


@pytest.mark.parametrize("name", ["sphere2", "box"])
def test_vjp_through_the_spring_damper_law(name):
    model, mode, q, qd, tau, params = golden_case(name)
    law = dict(contact_model=1, spring_k=40000.0, damper_d=3000.0, exponent_n=1.5, v_transition=0.02, hard_contact_condition=True)
    check_vjp_vs_dual(model, 2, q, qd, tau, 13, **law, **params)


@pytest.mark.parametrize("name", ["mb_three_bodies", "mb_racket", "humanoid_spherical"])
def test_vjp_on_worlds_of_multibodies_and_spherical_joints(name):
    model, mode, q, qd, tau, params = golden_case(name)
    check_vjp_vs_dual(model, 2, q, qd, tau, 14, **params)


@pytest.mark.parametrize("name,gen,frac", [("pendulum5", wl.pendulum5, 1.0), ("cartpole", wl.cartpole, 1.0), ("sphere2", wl.sphere2, 0.9)])
def test_vjp_vs_central_differences_of_the_c_oracle(name, gen, frac):
    """<VJP, v> against g^T (f(x + h v) - f(x - h v)) / 2h of the fp64 C oracle: a check of the gradient that does not go through
    the kernel source's own forward mode."""
    n = 20
    model = load_model(fixture_path(name))
    w = gen(n, seed=31)
    mode, tau = w["mode"], w.get("tau")
    n_q, n_qd = int(model[3]), int(model[4])
    n_tau = n_qd - (6 if int(model[2]) else 0)
    t = None if tau is None or not n_tau else tau[:, -n_tau:]
    rows = n_qd if mode == 0 else n_q + n_qd
    rng = np.random.default_rng(32)
    g = rng.normal(size=(n, rows))
    v_in, _ = emu_vjp.step_vjp(model, mode, w["q"], w["qd"], g, t, **w["params"])
    P = port.make_params(**w["params"])

    def f(x):
        r = port.step(model, P, mode, x[:n_q], x[n_q:n_q + n_qd], x[n_q + n_qd:] if n_tau else None)
        return r["qdd"] if mode == 0 else np.concatenate([r["q"], r["qd"]])
    ok = []
    h = 1e-6
    for e in range(n):
        x0 = np.concatenate([w["q"][e], w["qd"][e], t[e] if t is not None else np.zeros(0)])
        v = rng.normal(size=x0.size)
        fd = g[e] @ (f(x0 + h * v) - f(x0 - h * v)) / (2 * h)
        ad = v_in[e] @ v
        ok.append(abs(ad - fd) <= 1e-4 * max(1.0, abs(fd)))
    assert np.mean(ok) >= frac, np.mean(ok)


def test_tape_regrowth_returns_bit_identical_gradients():
    model, mode, q, qd, tau, params = golden_case("laikago")
    rows = int(model[3]) + int(model[4])
    g = np.random.default_rng(15).normal(size=(q.shape[0], rows))
    big, st_big = emu_vjp.step_vjp(model, mode, q, qd, g, tau, tape_cap=1 << 20, **params)
    small, st_small = emu_vjp.step_vjp(model, mode, q, qd, g, tau, tape_cap=8, **params)
    assert st_big["reruns"] == 0 and st_small["reruns"] > 0 and st_small["cap"] >= int(st_small["nodes"].max())
    assert np.array_equal(big, small)


@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3, 20])
def test_rigid_vjp_equals_gT_J_of_the_dual_instance(kind, steps):
    """The checkpointed reverse pass (one recorded step at a time, the cotangent chained backwards) against g^T J of the dual-number
    instance run over all the steps at once."""
    w = wl.rigid_world(kind, 6, seed=41)
    _, J = emu.rigid_step(w["bodies"], w["state"], w["force"], steps, jacobian=True, **w["params"])
    n = J.shape[0]
    g = np.random.default_rng(42).normal(size=J.shape[:2])
    gs, gf, st = emu_vjp.rigid_vjp(w["bodies"], w["state"], g, w["force"], steps, tape_cap=64, **w["params"])
    assert st["reruns"] > 0
    v = np.concatenate([gs.reshape(n, -1), gf.reshape(n, -1)], axis=1)
    assert vjp_err(v, np.einsum("er,erc->ec", g, J)) <= 1e-12


# ---- the billiard optimisation (python/examples/billiard_optimization.py, three balls) ---------------------------------------------
BILLIARD_STEPS, BILLIARD_ITERS, BILLIARD_LR = 40, 20, 0.8
BILLIARD_GOAL = np.array([1.6, 0.6, 0.0])


def billiard_setup():
    """Cue ball, target ball, a third ball, no gravity (the balls roll on the table plane z = 0), 50 solver sweeps as in the
    reference's example.  The optimised variable is the cue ball's initial velocity in the plane."""
    from tds_b200 import rigid as rg
    bodies = [rg.sphere(1.0, 0.5)] * 3
    state = rg.identity_state(1, 3)
    state[0, 0, :3] = (-2.0, -0.1, 0.0)
    state[0, 1, :3] = (0.0, 0.0, 0.0)
    state[0, 2, :3] = (0.9, 1.6, 0.0)
    params = dict(dt=1.0 / 60.0, gravity=(0.0, 0.0, 0.0), num_solver_iterations=50)
    return bodies, state, params, np.array([4.0, 0.6])


def billiard_loss_grad(step_fn, vjp_fn, state, v):
    """loss = |p_target(T) - goal|^2 and its gradient with respect to the cue velocity (vx, vy)."""
    s = state.copy()
    s[0, 0, 7:9] = v
    out = step_fn(s)
    d = out[0, 1, :3] - BILLIARD_GOAL
    g = np.zeros_like(out)
    g[0, 1, :3] = 2 * d
    gs = vjp_fn(s, g)
    return float(d @ d), gs[0, 0, 7:9]


def billiard_descent(step_fn, vjp_fn):
    bodies, state, params, v = billiard_setup()
    losses = []
    for _ in range(BILLIARD_ITERS):
        loss, grad = billiard_loss_grad(step_fn, vjp_fn, state, v)
        losses.append(loss)
        v = v - BILLIARD_LR * grad
    return np.array(losses), v


def test_billiard_optimisation_on_the_host_build():
    bodies, state, params, _ = billiard_setup()
    step_fn = lambda s: emu.rigid_step(bodies, s, None, BILLIARD_STEPS, **params)
    vjp_fn = lambda s, g: emu_vjp.rigid_vjp(bodies, s, g, None, BILLIARD_STEPS, **params)[0]
    losses, v = billiard_descent(step_fn, vjp_fn)
    # the recorded trajectory of this rehearsal: tests/test_vjp_gpu.py runs the same descent on the device against it
    rehearsal = np.load(os.path.join(GOLDEN, "vjp_billiard_losses.npy"))
    assert np.max(np.abs(losses - rehearsal) / np.maximum(1.0, np.abs(rehearsal))) <= 1e-9
    assert losses[-1] < 0.1 * losses[0]
