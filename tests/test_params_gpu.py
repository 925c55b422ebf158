"""Per-environment physical parameters on the H100 (DESIGN.md section 7.9): the parameter instances of the world-frame kernel against
the instances without parameters and against simulators built from edited models, against the host build of the same source, on
ragged and chunked batches, through the environment layer and through torch.autograd (tds_b200.autograd.step(..., params=)).
The CPU twins are in tests/test_params_on_host.py."""
import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
from tds_b200.model import param_names, param_values, set_param_values
from test_vjp_gpu import _case, rel

pytestmark = pytest.mark.gpu

FLOATING_TOL = 1e-6   # the floating base's inertia is packed per lane on the device (nvcc may contract to FMA there)


def all_ids(model):
    names = param_names(model)
    return [i for i, nm in enumerate(names) if int(model[2]) or not nm.startswith("base.")]


def _world_case(name, n, monkeypatch, seed=2718):
    monkeypatch.setenv("TDS_B200_KERNEL", "world")
    return _case(name, n, seed)


def _friction_restitution(name):
    if name == "laikago_pd":
        return 1.0, 0.0
    if name == "mb_three_bodies":
        return wl.multibody_world("three_bodies", 1)["params"].get("friction", 0.5), 0.0
    p = getattr(wl, name)(1, seed=0)["params"]
    return p.get("friction", 0.5), p.get("restitution", 0.0)


def perturbed(model, ids, n, seed, friction, restitution):
    from test_params_on_host import perturbed as p
    return p(model, ids, n, seed, friction, restitution)


def _same(a, b, floating):
    return rel(a, b) <= FLOATING_TOL if floating else np.array_equal(a, b)


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "humanoid_spherical", "laikago_pd", "mb_three_bodies"])
def test_every_parameter_at_the_model_value_reproduces_the_step(name, monkeypatch):
    n = 40
    sim, mode, q, qd, t, pd = _world_case(name, n, monkeypatch)
    ref = sim.step_host(mode, q, qd, t, use_pd=pd)
    ids = all_ids(sim.model)
    sim.set_physical_params(ids, param_values(sim.model, *_friction_restitution(name))[ids])
    got = sim.step_host(mode, q, qd, t, use_pd=pd)
    for k in ("q", "qd"):
        assert _same(got[k], ref[k], int(sim.model[2])), (name, k, rel(got[k], ref[k]))


@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago_pd"])
def test_edited_model_per_environment_on_the_device(name, monkeypatch):
    n = 4
    sim, mode, q, qd, t, pd = _world_case(name, n, monkeypatch)
    fr, rs = _friction_restitution(name)
    ids = all_ids(sim.model)
    vals = perturbed(sim.model, ids, n, 21, fr, rs)
    sim.set_physical_params(ids, vals)
    got = sim.step_host(mode, q, qd, t, use_pd=pd)
    for e in range(n):
        edited = set_param_values(sim.model, ids[2:], vals[e, 2:])
        if pd:
            one = tds_b200.laikago_sim(1, model=edited)
            one.set_params(dt=1e-3, friction=vals[e, 0], restitution=vals[e, 1], keep_all_points=True)
        else:
            wp = getattr(wl, name)(1, seed=0)["params"]
            one = tds_b200.BatchSim(edited, 1, **wp)
            one.set_params(**dict(wp, friction=vals[e, 0], restitution=vals[e, 1]))
        one.set_precision(sim.precision)
        ref = one.step_host(mode, q[e:e + 1], qd[e:e + 1], None if t is None else t[e:e + 1], use_pd=pd)
        for k in ("q", "qd"):
            assert _same(got[k][e:e + 1], ref[k], int(sim.model[2])), (name, e, k, rel(got[k][e:e + 1], ref[k]))


def test_device_agrees_with_the_host_build():
    """Build agreement (nvcc against the same source compiled for the CPU), not a reference check."""
    import emu_params
    for name in ("sphere2", "humanoid_spherical"):
        n = 8
        sim, mode, q, qd, t, _ = _case(name, n)
        sim.set_precision(tds_b200.sim.PREC_F64)
        w = getattr(wl, name)(n, seed=2718)
        ids = all_ids(sim.model)
        vals = perturbed(sim.model, ids, n, 22, w["params"].get("friction", 0.5), w["params"].get("restitution", 0.0))
        sim.set_physical_params(ids, vals)
        got = sim.step_host(mode, q, qd, t)
        host = emu_params.step(sim.model, mode, q, qd, t, ids=ids, values=vals, precision=1, **w["params"])
        assert rel(got["q"], host["q"]) <= 1e-5 and rel(got["qd"], host["qd"]) <= 1e-5
        J = sim.step_param_jacobian_host(mode, q, qd, t)
        Jh = emu_params.step(sim.model, mode, q, qd, t, ids=ids, values=vals, what="param_jacobian", **w["params"])["jac"]
        assert rel(J, Jh) <= 1e-5
        rows, _ = sim.jacobian_dims(mode)
        g = np.random.default_rng(23).normal(size=(n, rows))
        g_in, g_par = sim.step_vjp_params_host(mode, q, qd, t, g)
        h = emu_params.step(sim.model, mode, q, qd, t, ids=ids, values=vals, what="vjp", g_out=g, **w["params"])
        assert rel(g_par, h["g_par"]) <= 1e-5 and rel(g_in, h["g_in"]) <= 1e-5
        assert rel(g_par, np.einsum("er,erk->ek", g, J)) <= 1e-9


def test_ragged_batches_are_bit_identical_to_a_full_batch():
    n_full = 128
    sim, mode, q, qd, t, pd = _case("laikago_pd", n_full)
    ids = all_ids(sim.model)
    vals = perturbed(sim.model, ids, n_full, 24, 1.0, 0.0)
    sim.set_physical_params(ids, vals)
    full = sim.step_host(mode, q, qd, t, use_pd=pd)
    rows, _ = sim.jacobian_dims(mode, pd)
    g = np.random.default_rng(25).normal(size=(n_full, rows))
    _, gp_full = sim.step_vjp_params_host(mode, q, qd, t, g, use_pd=pd)
    for n in (1, 31, 33, 100):
        small = tds_b200.laikago_sim(n)
        small.set_physical_params(ids, vals[-n:])
        out = small.step_host(mode, q[-n:], qd[-n:], t[-n:], use_pd=pd)
        assert np.array_equal(out["q"], full["q"][-n:]) and np.array_equal(out["qd"], full["qd"][-n:]), n
        _, gp = small.step_vjp_params_host(mode, q[-n:], qd[-n:], t[-n:], g[-n:], use_pd=pd)
        assert np.array_equal(gp, gp_full[-n:]), n


def test_chunked_parameter_vjp_equals_a_small_batch():
    """A humanoid batch of at least two VJP chunks: the parameter values and g_par are offset per chunk like q and qd."""
    probe, mode, q, qd, t, _ = _case("humanoid", 64)
    ids = all_ids(probe.model)
    rows, _ = probe.jacobian_dims(mode)
    probe.set_physical_params(ids, param_values(probe.model)[ids])
    probe.step_vjp_params_host(mode, q, qd, t, np.ones((64, rows)))
    _, per_chunk = probe.vjp_tape_info()
    n = per_chunk + 333
    sim, mode, q, qd, t, _ = _case("humanoid", n, seed=17)
    vals = perturbed(sim.model, ids, n, 26, 0.5, 0.0)
    sim.set_physical_params(ids, vals)
    g = np.random.default_rng(27).normal(size=(n, rows))
    g_in, g_par = sim.step_vjp_params_host(mode, q, qd, t, g)
    assert sim.vjp_tape_info()[1] < n
    idx = np.sort(np.random.default_rng(28).choice(n, 64, replace=False))
    probe.set_physical_params(ids, vals[idx])
    r_in, r_par = probe.step_vjp_params_host(mode, q[idx], qd[idx], t[idx], g[idx])
    assert np.array_equal(g_par[idx], r_par) and np.array_equal(g_in[idx], r_in)


@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago_pd"])
def test_autograd_with_params_through_a_rollout_equals_the_chain_of_jacobians(name):
    import torch
    n, steps = 16, 5
    sim, mode, q, qd, t, pd = _case(name, n)
    md = 2 if mode == 0 else mode
    if t is None:
        t = np.zeros((n, sim.n_act if pd else sim.n_tau))
    fr, rs = _friction_restitution(name)
    names = param_names(sim.model)
    ids = [i for i in all_ids(sim.model) if names[i].endswith(("mass", "damping", "com.z")) or i < 2]
    vals = perturbed(sim.model, ids, n, 29, fr, rs)
    sim.set_physical_params(ids, vals)
    dev = "cuda:0"
    par = torch.tensor(vals, dtype=torch.float64, device=dev, requires_grad=True)
    x = torch.tensor(q, dtype=torch.float32, device=dev)
    xd = torch.tensor(qd, dtype=torch.float32, device=dev)
    tau = torch.tensor(t, dtype=torch.float32, device=dev)
    rng = np.random.default_rng(30)
    wq, wqd = rng.normal(size=(n, sim.n_q)), rng.normal(size=(n, sim.n_qd))
    states = []
    for _ in range(steps):
        states.append((x.detach().cpu().numpy().astype(np.float64), xd.detach().cpu().numpy().astype(np.float64)))
        x, xd = tds_b200.autograd.step(sim, x, xd, tau, mode=md, use_pd=pd, params=par)
    loss = (x * torch.tensor(wq, dtype=torch.float32, device=dev)).sum() + (xd * torch.tensor(wqd, dtype=torch.float32, device=dev)).sum()
    loss.backward()
    g = np.concatenate([wq, wqd], axis=1).astype(np.float32).astype(np.float64)
    g_par = np.zeros(vals.shape)
    nx = sim.n_q + sim.n_qd
    for k in reversed(range(steps)):
        J = sim.step_jacobian_host(md, states[k][0], states[k][1], t, use_pd=pd)
        Jp = sim.step_param_jacobian_host(md, states[k][0], states[k][1], t, use_pd=pd)
        g_par += np.einsum("er,erk->ek", g, Jp)
        g = np.einsum("er,erc->ec", g, J)[:, :nx].astype(np.float32).astype(np.float64)
    assert par.grad.dtype == torch.float64
    assert rel(par.grad.cpu().numpy(), g_par) <= 1e-6


def test_environment_layer_uses_the_installed_values():
    import torch
    n = 64
    sim, mode, q, qd, t, pd = _case("laikago_pd", n)
    ids = all_ids(sim.model)
    vals = perturbed(sim.model, ids, n, 31, 1.0, 0.0)
    sim.set_physical_params(ids, vals)
    ref = sim.step_host(2, q, qd, t, use_pd=True)
    sim.env_set_state(q, qd)
    acts = torch.tensor(t, dtype=torch.float32).pin_memory()
    obs = torch.zeros((n, sim.n_q + sim.n_qd), dtype=torch.float32).pin_memory()
    rew = torch.zeros(n, dtype=torch.float32).pin_memory()
    done = torch.zeros(n, dtype=torch.float32).pin_memory()
    sim.env_step_host(acts, obs, rew, done)
    o = obs.numpy().astype(np.float64)
    assert np.array_equal(o[:, :sim.n_q], ref["q"]) and np.array_equal(o[:, sim.n_q:], ref["qd"])


def test_clearing_the_set_restores_the_kernel_and_the_outputs():
    n = 64
    fresh, mode, q, qd, t, pd = _case("laikago_pd", n)
    ref = fresh.step_host(mode, q, qd, t, use_pd=pd)
    sim, *_ = _case("laikago_pd", n)
    ids = all_ids(sim.model)
    sim.set_physical_params(ids, perturbed(sim.model, ids, n, 32, 1.0, 0.0))
    sim.step_host(mode, q, qd, t, use_pd=pd)
    assert sim.kernel_name().startswith("tds_stepw_kernel")
    sim.set_physical_params(None)
    out = sim.step_host(mode, q, qd, t, use_pd=pd)
    assert sim.kernel_name() == fresh.kernel_name()
    assert np.array_equal(out["q"], ref["q"]) and np.array_equal(out["qd"], ref["qd"])


def test_system_identification_through_autograd_reproduces_the_host_descent():
    """The host descent of tests/test_params_on_host.py through tds_b200.autograd.step.  Both carry the state in fp32 between steps;
    autograd also rounds the state cotangents to fp32, and nvcc contracts to FMA where the host build does not, so a step's state
    may differ in its last fp32 bit (~6e-8).  While the loss is well above that noise (>= 1e-4 of the first one) the trajectories
    agree to 1e-3 relative; near convergence the loss is of the order of the rounding noise itself, so there only the end point is
    checked: within 1 % of the generating parameters."""
    import torch
    from test_params_on_host import (SYSID_DECAY, SYSID_ENVS, SYSID_GOLDEN, SYSID_ITERS, SYSID_LR, SYSID_STEPS, sysid_problem)
    model, ids, truth, start, q0, qd0, tau, kw = sysid_problem()
    n, dev = SYSID_ENVS, "cuda:0"
    sim = tds_b200.BatchSim(model, n, **kw)
    sim.set_physical_params(ids, start)
    tau_t = [torch.tensor(tau[k], dtype=torch.float32, device=dev) for k in range(SYSID_STEPS)]
    x0 = torch.tensor(q0, dtype=torch.float32, device=dev)
    xd0 = torch.tensor(qd0, dtype=torch.float32, device=dev)

    def rollout(p):
        xs, x, xd = [], x0, xd0
        for k in range(SYSID_STEPS):
            x, xd = tds_b200.autograd.step(sim, x, xd, tau_t[k], params=p.unsqueeze(0).expand(n, -1).contiguous())
            xs.append((x, xd))
        return xs
    with torch.no_grad():
        target = [(a.detach(), b.detach()) for a, b in rollout(torch.tensor(truth, dtype=torch.float64, device=dev))]
    z = torch.tensor(np.log(start), dtype=torch.float64, device=dev)
    m1, m2 = torch.zeros(4, dtype=torch.float64, device=dev), torch.zeros(4, dtype=torch.float64, device=dev)
    losses = []
    for it in range(SYSID_ITERS):
        zz = z.clone().requires_grad_(True)
        xs = rollout(torch.exp(zz))
        loss = sum(((a.double() - ta.double()) ** 2).sum() + ((b.double() - tb.double()) ** 2).sum() for (a, b), (ta, tb) in zip(xs, target)) / n
        loss.backward()
        losses.append(float(loss.detach()))
        g = zz.grad
        m1 = 0.9 * m1 + 0.1 * g
        m2 = 0.999 * m2 + 0.001 * g * g
        z = z - SYSID_LR * SYSID_DECAY ** it * (m1 / (1 - 0.9 ** (it + 1))) / (torch.sqrt(m2 / (1 - 0.999 ** (it + 1))) + 1e-12)
    final = np.exp(z.cpu().numpy())
    host = np.load(SYSID_GOLDEN)
    losses = np.array(losses)
    big = host >= 1e-4 * host[0]
    assert big.sum() >= 20
    assert np.max(np.abs(losses[big] - host[big]) / host[big]) <= 1e-3
    assert losses[-1] < 1e-3 * losses[0]
    assert np.all(np.abs(final / truth - 1) <= 0.01), final / truth
