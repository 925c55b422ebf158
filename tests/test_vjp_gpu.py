"""Reverse mode on the H100: the vector-Jacobian products of the step (taping instance of the world-frame kernel) and of the
rigid-body world, against g^T J of the dual-number instance on the device, against the host build of the same source, on ragged
and chunked batches, and through torch.autograd (tds_b200.autograd).  The CPU twins are in tests/test_vjp_on_host.py."""
import os

import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
from tds_b200.model import fixture_path, load_model

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref)))) if ref.size else 0.0


def _case(name, n, seed=2718):
    """(sim, mode, q, qd, tau_or_action, use_pd) of a workload."""
    if name == "laikago_pd":
        w = wl.laikago_perturbed(n, seed=seed)
        return tds_b200.laikago_sim(n), 2, w["q"], w["qd"], w["action"], True
    if name in ("mb_three_bodies",):
        w = wl.multibody_world(name[3:], n, seed=seed)
        return tds_b200.BatchSim(w["model"], n, **w["params"]), 2, w["q"], w["qd"], w["tau"], False
    gen = getattr(wl, name)
    w = gen(n, seed=seed)
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, **w["params"])
    tau = w.get("tau")
    t = None if tau is None or not sim.n_tau else tau[:, -sim.n_tau:]
    return sim, w["mode"], w["q"], w["qd"], t, False


@pytest.mark.parametrize("name", ["pendulum5", "cartpole", "sphere2", "box", "humanoid", "laikago_pd", "mb_three_bodies",
                                  "humanoid_spherical"])
def test_vjp_equals_gT_J_on_the_device(name):
    n = 24
    sim, mode, q, qd, t, pd = _case(name, n)
    J = sim.step_jacobian_host(mode, q, qd, t, use_pd=pd)
    g = np.random.default_rng(3).normal(size=J.shape[:2])
    v = sim.step_vjp_host(mode, q, qd, t, g, use_pd=pd)
    assert rel(v, np.einsum("er,erc->ec", g, J)) <= 1e-9


def test_device_vjp_agrees_with_the_host_build():
    """Build agreement (the nvcc build against the same kernel source compiled for the CPU), not a reference check."""
    import emu_vjp
    for name in ("sphere2", "humanoid_spherical"):
        sim, mode, q, qd, t, _ = _case(name, 8)
        w = getattr(wl, name)(8, seed=2718)
        rows, _ = sim.jacobian_dims(mode)
        g = np.random.default_rng(4).normal(size=(8, rows))
        v = sim.step_vjp_host(mode, q, qd, t, g)
        vh, _ = emu_vjp.step_vjp(sim.model, mode, q, qd, g, t, **w["params"])
        assert rel(v, vh) <= 1e-5


def test_ragged_batches_are_bit_identical_to_a_full_batch():
    n_full = 128
    sim, mode, q, qd, t, pd = _case("laikago_pd", n_full)
    rows, _ = sim.jacobian_dims(mode, pd)
    g = np.random.default_rng(5).normal(size=(n_full, rows))
    full = sim.step_vjp_host(mode, q, qd, t, g, use_pd=pd)
    for n in (1, 31, 33, 100):
        small = tds_b200.laikago_sim(n)
        v = small.step_vjp_host(mode, q[-n:], qd[-n:], t[-n:], g[-n:], use_pd=pd)
        assert np.array_equal(v, full[-n:]), n


def test_chunked_batch_equals_a_small_batch():
    """A humanoid batch sized from the tape length so that the VJP runs in at least two chunks of environments."""
    probe, mode, q, qd, t, _ = _case("humanoid", 64)
    rows, _ = probe.jacobian_dims(mode)
    probe.step_vjp_host(mode, q, qd, t, np.ones((64, rows)))
    _, per_chunk = probe.vjp_tape_info()
    n = per_chunk + 333
    sim, mode, q, qd, t, _ = _case("humanoid", n, seed=17)
    g = np.random.default_rng(6).normal(size=(n, rows))
    v = sim.step_vjp_host(mode, q, qd, t, g)
    cap, per_chunk2 = sim.vjp_tape_info()
    assert per_chunk2 < n and cap >= 32768
    idx = np.sort(np.random.default_rng(7).choice(n, 64, replace=False))
    ref = probe.step_vjp_host(mode, q[idx], qd[idx], t[idx], g[idx])
    assert np.array_equal(v[idx], ref)


@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago_pd"])
def test_autograd_through_a_rollout_equals_the_chain_of_jacobians(name):
    import torch
    n, steps = 16, 5
    sim, mode, q, qd, t, pd = _case(name, n)
    if t is None:
        t = np.zeros((n, sim.n_act if pd else sim.n_tau))
    dev = "cuda:0"
    q0 = torch.tensor(q, dtype=torch.float32, device=dev, requires_grad=True)
    qd0 = torch.tensor(qd, dtype=torch.float32, device=dev, requires_grad=True)
    tau = torch.tensor(t, dtype=torch.float32, device=dev, requires_grad=True)
    rng = np.random.default_rng(8)
    wq, wqd = rng.normal(size=(n, sim.n_q)), rng.normal(size=(n, sim.n_qd))
    states = []
    x, xd = q0, qd0
    for _ in range(steps):
        states.append((x.detach().cpu().numpy().astype(np.float64), xd.detach().cpu().numpy().astype(np.float64)))
        x, xd = tds_b200.autograd.step(sim, x, xd, tau, mode=2 if mode == 0 else mode, use_pd=pd)
    loss = (x * torch.tensor(wq, dtype=torch.float32, device=dev)).sum() + (xd * torch.tensor(wqd, dtype=torch.float32, device=dev)).sum()
    loss.backward()
    # the same chain by hand: g^T J at the recorded states, the cotangent rounded to float32 between steps as autograd does
    md = 2 if mode == 0 else mode
    g = np.concatenate([wq, wqd], axis=1).astype(np.float32).astype(np.float64)
    g_tau = np.zeros(t.shape, dtype=np.float32)
    nx = sim.n_q + sim.n_qd
    for k in reversed(range(steps)):
        J = sim.step_jacobian_host(md, states[k][0], states[k][1], t, use_pd=pd)
        gin = np.einsum("er,erc->ec", g, J)
        g_tau = g_tau + gin[:, nx:nx + t.shape[1]].astype(np.float32)
        g = gin[:, :nx].astype(np.float32).astype(np.float64)
    assert rel(q0.grad.cpu().numpy().astype(np.float64), g[:, :sim.n_q]) <= 1e-6
    assert rel(qd0.grad.cpu().numpy().astype(np.float64), g[:, sim.n_q:]) <= 1e-6
    assert rel(tau.grad.cpu().numpy().astype(np.float64), g_tau.astype(np.float64)) <= 1e-6


@pytest.mark.parametrize("steps", [1, 20])
def test_rigid_vjp_equals_gT_J_on_the_device(steps):
    n = 40
    w = wl.rigid_world("billiard", n, seed=9)
    world = tds_b200.RigidWorld(w["bodies"], n, **w["params"])
    _, J = world.step_jacobian(w["state"], w["force"], steps)
    g = np.random.default_rng(10).normal(size=J.shape[:2])
    gs, gf = world.step_vjp(w["state"], w["force"], g.reshape(w["state"].shape), steps)
    v = np.concatenate([gs.reshape(n, -1), gf.reshape(n, -1)], axis=1)
    # 20 chained steps: the dual instance and the checkpointed states may round differently where nvcc contracts to FMA
    assert rel(v, np.einsum("er,erc->ec", g, J)) <= (1e-12 if steps == 1 else 1e-9)


def test_billiard_optimisation_through_autograd_reproduces_the_host_rehearsal():
    import torch
    from test_vjp_on_host import BILLIARD_GOAL, BILLIARD_ITERS, BILLIARD_LR, BILLIARD_STEPS, billiard_setup
    bodies, state, params, v0 = billiard_setup()
    world = tds_b200.RigidWorld(bodies, 1, **params)
    goal = torch.tensor(BILLIARD_GOAL, dtype=torch.float64, device="cuda:0")
    base = torch.tensor(state, dtype=torch.float64, device="cuda:0")
    v = torch.tensor(v0, dtype=torch.float64, device="cuda:0")
    losses = []
    for _ in range(BILLIARD_ITERS):
        vv = v.clone().requires_grad_(True)
        s = base.clone()
        s[0, 0, 7:9] = vv
        out = tds_b200.autograd.rigid_step(world, s, None, BILLIARD_STEPS)
        loss = ((out[0, 1, :3] - goal) ** 2).sum()
        loss.backward()
        losses.append(float(loss))
        v = (vv - BILLIARD_LR * vv.grad).detach()
    losses = np.array(losses)
    rehearsal = np.load(os.path.join(GOLDEN, "vjp_billiard_losses.npy"))
    assert rel(losses, rehearsal) <= 1e-6
    assert losses[-1] / losses[0] <= rehearsal[-1] / rehearsal[0] * (1 + 1e-6)
