"""Per-environment physical parameters (DESIGN.md section 7.9) on the CPU, from the kernel SOURCE: the parameter instances of
csrc/tds_stepw.cu compiled for the host (tests/cpp/stepw_param_host.cpp) against the instances without parameters on the model and
on edited models, their dual-number parameter Jacobian against central differences of the fp64 C oracle, their reverse sweep
against g^T J, and a system identification of a cartpole by descent through a rollout.  tests/test_params_gpu.py checks the same
instances as nvcc builds them."""
import os

import numpy as np
import pytest

import tds_b200.envs as envs
import tds_b200.workloads as wl
from tds_b200.model import fixture_path, load_model, param_names, param_values, set_param_values
from oracle import port
import emu
import emu_params
import emu_vjp
from test_kernel_source_on_host import CONFIGS
from test_vjp_on_host import golden_case, pd_env

HERE = os.path.dirname(os.path.abspath(__file__))
SYSID_GOLDEN = os.path.join(HERE, "golden", "params_sysid_losses.npy")


def all_ids(model):
    """Every id that can be installed on the model (base ids only on a floating base)."""
    names = param_names(model)
    return [i for i, nm in enumerate(names) if int(model[2]) or not nm.startswith("base.")]


def rel(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def perturbed(model, ids, n, seed, friction, restitution):
    """[n, k] values: +-20 % on masses, coms and inertias, friction in [0.3, 1.2], restitution in [0, 0.5], damping in [0, 0.5],
    stiffness in [0, 2] (zero-valued coms get +-0.02)."""
    rng = np.random.default_rng(seed)
    names = param_names(model)
    base = param_values(model, friction, restitution)
    out = np.zeros((n, len(ids)))
    for j, i in enumerate(ids):
        nm, v = names[i], base[i]
        if nm == "friction":
            out[:, j] = rng.uniform(0.3, 1.2, n)
        elif nm == "restitution":
            out[:, j] = rng.uniform(0.0, 0.5, n)
        elif nm.endswith("damping"):
            out[:, j] = rng.uniform(0.0, 0.5, n)
        elif nm.endswith("stiffness"):
            out[:, j] = rng.uniform(0.0, 2.0, n)
        elif ".com." in nm and v == 0.0:
            out[:, j] = rng.uniform(-0.02, 0.02, n)
        else:
            out[:, j] = v * rng.uniform(0.8, 1.2, n)
    return out


@pytest.mark.parametrize("name", CONFIGS + ["mb_three_bodies"])
def test_every_parameter_at_the_model_value_is_bit_identical(name):
    """All ids installed at the model's values reproduce the instance without parameters exactly, in fp64 and mixed precision.  (The
    floating base's inertia is packed per lane by the kernel with the same formula as the host; the host build shows no difference.)"""
    model, mode, q, qd, tau, params = golden_case(name)
    ids = all_ids(model)
    vals = param_values(model, params.get("friction", 0.5), params.get("restitution", 0.0))[ids]
    for prec in (1, 0):
        a = emu.step(model, mode, q, qd, tau, precision=prec, **params)
        b = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, precision=prec, **params)
        keys = ("qdd",) if mode == 0 else ("q", "qd")
        for k in keys:
            assert np.array_equal(a[k], b[k]), (name, prec, k, rel(b[k], a[k]))


@pytest.mark.parametrize("name", CONFIGS + ["mb_three_bodies"])
def test_edited_model_per_environment(name):
    """Environment e with values p_e equals the instance without parameters on the flat model with p_e written in (friction and
    restitution through the solver parameters): bit-identical."""
    model, mode, q, qd, tau, params = golden_case(name)
    n = min(q.shape[0], 6)
    q, qd, tau = q[:n], qd[:n], None if tau is None else tau[:n]
    ids = all_ids(model)
    fr, rs = params.get("friction", 0.5), params.get("restitution", 0.0)
    vals = perturbed(model, ids, n, 5, fr, rs)
    got = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, precision=1, **params)
    for e in range(n):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        kw = dict(params, friction=vals[e, 0], restitution=vals[e, 1])
        ref = emu.step(edited, mode, q[e:e + 1], qd[e:e + 1], None if tau is None else tau[e:e + 1], precision=1, **kw)
        for k in (("qdd",) if mode == 0 else ("q", "qd")):
            assert np.array_equal(got[k][e:e + 1], ref[k]), (name, e, k, rel(got[k][e:e + 1], ref[k]))


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2"])
def test_edited_model_matches_the_c_oracle(name):
    model, mode, q, qd, tau, params = golden_case(name)
    n = min(q.shape[0], 6)
    ids = all_ids(model)
    fr, rs = params.get("friction", 0.5), params.get("restitution", 0.0)
    vals = perturbed(model, ids, n, 6, fr, rs)
    got = emu_params.step(model, mode, q[:n], qd[:n], None if tau is None else tau[:n], ids=ids, values=vals, precision=1, **params)
    n_q = int(model[3])
    for e in range(n):
        edited = set_param_values(model, ids[2:], vals[e, 2:])
        P = port.make_params(**dict(params, friction=vals[e, 0], restitution=vals[e, 1]))
        # the kernel runs on the fp32-rounded state and uses damping / stiffness at fp32
        for i in ids[2:]:
            if param_names(model)[i].endswith(("damping", "stiffness")):
                edited = set_param_values(edited, [i], [float(np.float32(vals[e, ids.index(i)]))])
        r = port.step(edited, P, mode, q[e].astype(np.float32).astype(np.float64), qd[e].astype(np.float32).astype(np.float64),
                      None if tau is None else tau[e].astype(np.float32).astype(np.float64))
        if mode == 0:
            assert rel(got["qdd"][e], r["qdd"]) <= 1e-5
        else:
            assert rel(got["q"][e], r["q"][:n_q]) <= 1e-5 and rel(got["qd"][e], r["qd"]) <= 1e-5


def fd_case(name):
    """(model, mode, q, qd, tau, params, use_pd, env) of the finite-difference fixtures."""
    if name == "laikago_pd":
        g = np.load(os.path.join(HERE, "golden", "laikago.npz"))
        model = load_model(fixture_path("laikago"))
        return model, 2, g["q_in"], g["qd_in"], g["action"], dict(friction=1.0, keep_all_points=True), True, pd_env("laikago")
    gen = {"pendulum5": wl.pendulum5, "cartpole": wl.cartpole, "sphere2": wl.sphere2}.get(name)
    if gen is not None:
        model = load_model(fixture_path(name))
        w = gen(8, seed=41)
        n_qd = int(model[4])
        n_tau = n_qd - (6 if int(model[2]) else 0)
        tau = w.get("tau")
        return model, w["mode"], w["q"], w["qd"], None if tau is None or not n_tau else tau[:, -n_tau:], w["params"], False, None
    model, mode, q, qd, tau, params = golden_case(name)
    return model, 2, q[:8], qd[:8], None if tau is None else tau[:8], params, False, None


def oracle_fn(model, mode, params, use_pd, env):
    """f(edited model, friction, restitution, q, qd, tau) of the fp64 C oracle (the locomotion step with PD)."""
    n_q, n_qd = int(model[3]), int(model[4])

    def f(m, fr, rs, q, qd, tau):
        P = port.make_params(**dict(params, friction=fr, restitution=rs))
        if use_pd:
            x = np.concatenate([q, qd, tau, env[2:5]])[None]
            r = port.locomotion_step(m, P, envs.LAIKAGO_INITIAL_POSES, 6, x, 411)[0]
            return r[:n_q + n_qd]
        r = port.step(m, P, mode, q, qd, tau)
        return r["qdd"] if mode == 0 else np.concatenate([r["q"][:n_q], r["qd"]])
    return f


@pytest.mark.parametrize("name,frac", [("pendulum5", 1.0), ("cartpole", 1.0), ("sphere2", 0.9), ("box", 0.9), ("laikago_pd", 0.9),
                                       ("humanoid", 0.9)])
def test_parameter_jacobian_vs_central_differences_of_the_c_oracle(name, frac):
    """J_par v against (f(p + h v) - f(p - h v)) / 2h of the fp64 C oracle on the edited model, along a random direction v over
    every installable parameter.  (The kernel takes the derivative at the fp32-rounded stiffness and damping, the oracle at the
    fp64 value: a difference far below the tolerance.)  Fixtures the oracle does not restate (spherical joints, worlds of several
    multibodies) are covered by the reverse-mode check against this dual Jacobian below."""
    model, mode, q, qd, tau, params, use_pd, env = fd_case(name)
    n = q.shape[0]
    ids = all_ids(model)
    fr, rs = params.get("friction", 0.5), params.get("restitution", 0.0)
    p0 = param_values(model, fr, rs)[ids]
    J = emu_params.step(model, mode, q, qd, tau, ids=ids, values=p0, what="param_jacobian", use_pd=use_pd, env=env, **params)["jac"]
    f = oracle_fn(model, mode, params, use_pd, env)
    rng = np.random.default_rng(42)
    qf, qdf = q.astype(np.float32).astype(np.float64), qd.astype(np.float32).astype(np.float64)
    tf = None if tau is None else tau.astype(np.float32).astype(np.float64)
    ok = []
    for e in range(n):
        v = rng.normal(size=len(ids)) * np.maximum(np.abs(p0), 0.05)
        h = 1e-6

        def at(s):
            p = p0 + s * v
            return f(set_param_values(model, ids[2:], p[2:]), p[0], p[1], qf[e], qdf[e], None if tf is None else tf[e])
        fd = (at(h) - at(-h)) / (2 * h)
        ad = J[e] @ v
        ok.append(np.all(np.abs(ad - fd) <= 1e-4 * np.maximum(1.0, np.abs(fd))))
    assert np.mean(ok) >= frac, (name, np.mean(ok))


def vjp_case(name):
    if name in ("laikago_pd", "pendulum5", "cartpole", "sphere2", "box", "humanoid"):
        return fd_case(name)
    model, mode, q, qd, tau, params = golden_case(name)
    return model, 2, q[:8], qd[:8], None if tau is None else tau[:8], params, False, None


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "laikago_pd", "humanoid", "mb_three_bodies",
                                  "humanoid_spherical"])
def test_parameter_vjp_equals_gT_J_par_and_keeps_g_in(name):
    model, mode, q, qd, tau, params, use_pd, env = vjp_case(name)
    ids = all_ids(model)
    fr, rs = params.get("friction", 0.5), params.get("restitution", 0.0)
    n = q.shape[0]
    vals = perturbed(model, ids, n, 3, fr, rs)
    kw = dict(use_pd=use_pd, env=env, **params)
    J = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, what="param_jacobian", **kw)["jac"]
    g = np.random.default_rng(17).normal(size=J.shape[:2])
    r = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, what="vjp", g_out=g, **kw)
    assert rel(r["g_par"], np.einsum("er,erk->ek", g, J)) <= 1e-10
    # at the model's values, g_in is that of the VJP without parameters, bit for bit
    p0 = param_values(model, fr, rs)[ids]
    r0 = emu_params.step(model, mode, q, qd, tau, ids=ids, values=p0, what="vjp", g_out=g, **kw)
    g_in, _ = emu_vjp.step_vjp(model, mode, q, qd, g, tau, **kw)
    assert np.array_equal(r0["g_in"], g_in)
    # regrowth from a capacity of 8 nodes gives the same g_par
    r8 = emu_params.step(model, mode, q, qd, tau, ids=ids, values=vals, what="vjp", g_out=g, tape_cap=8, **kw)
    assert r8["reruns"] > 0 and np.array_equal(r8["g_par"], r["g_par"])


def test_parameter_ids_are_checked():
    model = load_model(fixture_path("cartpole"))
    q, qd = np.zeros((1, int(model[3]))), np.zeros((1, int(model[4])))
    n_ids = len(param_names(model))
    assert emu_params.param_count(model) == n_ids
    for bad in ([n_ids], [-1], [3, 3], [2]):   # out of range, negative, twice, base mass on a fixed base
        with pytest.raises(ValueError):
            emu_params.step(model, 1, q, qd, ids=bad, values=np.ones(len(bad)))


# ---- system identification: cartpole masses and joint dampings through a rollout ------------------------------------------------------
SYSID_NAMES = ["link0.mass", "link1.mass", "link0.damping", "link1.damping"]
SYSID_TRUE_DAMPING = (0.3, 0.05)
SYSID_STEPS, SYSID_ENVS, SYSID_ITERS = 40, 8, 150
SYSID_LR, SYSID_DECAY = 0.05, 0.98   # Adam step on log-parameters, decayed per iteration


def sysid_problem():
    """(model, ids, true values, start values, q0, qd0, tau [T][n][n_tau], step kwargs)."""
    model = load_model(fixture_path("cartpole"))
    names = param_names(model)
    ids = [names.index(s) for s in SYSID_NAMES]
    truth = param_values(model)[ids]
    truth[2:] = SYSID_TRUE_DAMPING
    start = truth * np.array([1.3, 0.7, 0.7, 1.3])
    rng = np.random.default_rng(2024)
    n_q = int(model[3])
    q0 = rng.uniform(-0.3, 0.3, (SYSID_ENVS, n_q))
    qd0 = rng.uniform(-0.5, 0.5, (SYSID_ENVS, int(model[4])))
    tau = rng.uniform(-2.0, 2.0, (SYSID_STEPS, SYSID_ENVS, int(model[4])))
    return model, ids, truth, start, q0, qd0, tau, dict(dt=1e-2)


def sysid_host():
    """Adam on log-parameters through a SYSID_STEPS-step rollout of the host-built fp64 instance; loss = mean squared error of
    (q, qd) along the rollout against the rollout at the true values.  Returns (losses, final values)."""
    model, ids, truth, start, q0, qd0, tau, kw = sysid_problem()
    n = SYSID_ENVS

    def rollout(p):
        xs = [(q0, qd0)]
        for t in range(SYSID_STEPS):
            r = emu_params.step(model, 2, xs[-1][0], xs[-1][1], tau[t], ids=ids, values=p, **kw)
            xs.append((r["q"], r["qd"]))
        return xs
    target = rollout(truth)
    z = np.log(start)
    m1, m2 = np.zeros(4), np.zeros(4)
    losses = []
    for it in range(SYSID_ITERS):
        p = np.exp(z)
        xs = rollout(p)
        loss = 0.0
        gq, gqd = np.zeros_like(q0), np.zeros_like(qd0)
        grad = np.zeros(4)
        for t in range(SYSID_STEPS, 0, -1):
            dq, dqd = xs[t][0] - target[t][0], xs[t][1] - target[t][1]
            loss += float(np.sum(dq ** 2) + np.sum(dqd ** 2))
            gq, gqd = gq + 2 * dq, gqd + 2 * dqd
            r = emu_params.step(model, 2, xs[t - 1][0], xs[t - 1][1], tau[t - 1], ids=ids, values=p, what="vjp",
                                g_out=np.concatenate([gq, gqd], axis=1), tape_cap=4096, **kw)
            grad += r["g_par"].sum(axis=0)
            n_q = q0.shape[1]
            gq, gqd = r["g_in"][:, :n_q], r["g_in"][:, n_q:n_q + qd0.shape[1]]
        losses.append(loss / n)
        g = grad * p / n   # d loss / d log p
        m1 = 0.9 * m1 + 0.1 * g
        m2 = 0.999 * m2 + 0.001 * g * g
        z = z - SYSID_LR * SYSID_DECAY ** it * (m1 / (1 - 0.9 ** (it + 1))) / (np.sqrt(m2 / (1 - 0.999 ** (it + 1))) + 1e-12)
    return np.array(losses), np.exp(z), truth


def test_system_identification_of_a_cartpole_by_descent_through_a_rollout():
    losses, final, truth = sysid_host()
    assert np.all(np.abs(final / truth - 1) <= 0.01), final / truth
    assert losses[-1] < 1e-3 * losses[0]
    golden = np.load(SYSID_GOLDEN)
    assert np.max(np.abs(losses - golden) / np.maximum(1.0, np.abs(golden))) <= 1e-9
