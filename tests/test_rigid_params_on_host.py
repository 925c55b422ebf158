"""Per-world physical parameters of the rigid-body world (DESIGN.md section 7.11) executed on the CPU from the kernel's SOURCE
(tests/cpp/rigid_param_host.cpp, bound by tests/emu_rigid_params.py): parameters installed at the description's values against the
instances without parameters, bit for bit; per-world values against the kernel run on an edited description, bit for bit; the
parameter Jacobian against central differences; forward mode, reverse mode and the Jacobian against each other; the tape regrowth of
the chunked reverse pass; the refused ids and values; and a system identification of two ball masses and the restitution.
tests/test_rigid_params_gpu.py checks the same instances as nvcc builds them."""
import os

import numpy as np
import pytest

import tds_b200.rigid as rg
import tds_b200.workloads as wl
import emu
import emu_jvp
import emu_rigid_params as erp
import emu_vjp
from test_jvp_on_host import rel, rel_jv
from test_kernel_source_on_host import GOLDEN

N = 6
STEPS = [1, 3, 20]


def world(kind, n=N, seed=41):
    w = wl.rigid_world(kind, n, seed=seed)
    return w, w["bodies"], all_ids(w["bodies"])


def all_ids(desc):
    return rg.param_ids(desc, rg.param_names(desc))


def model_values(w):
    return rg.param_values(w["bodies"], friction=w["params"].get("friction", 0.5), restitution=w["params"].get("restitution", 0.0))


def random_values(w, ids, n, seed):
    """Per-world values: +-20 % on masses and sizes, friction in [0, 1], restitution in [0, 0.9]."""
    r = np.random.default_rng(seed)
    v = model_values(w)[None, :] * r.uniform(0.8, 1.2, (n, len(ids)))
    for j, i in enumerate(ids):
        if i == 0:
            v[:, j] = r.uniform(0.0, 1.0, n)
        elif i == 1:
            v[:, j] = r.uniform(0.0, 0.9, n)
    return v


def edited(w, ids, vals):
    """(description, World parameters) with the parameters ids set to vals [k] (friction and restitution: through set_params)."""
    d = np.array(w["bodies"], dtype=np.float64)
    p = dict(w["params"])
    for i, v in zip(ids, vals):
        if i == 0:
            p["friction"] = v
        elif i == 1:
            p["restitution"] = v
        else:
            b, c = divmod(i - 2, 4)
            d[b, 0 if c == 0 else 1 + c] = v
    return d, p


# ---- 1. installed at the description's values: the instances without parameters, bit for bit ------------------------------------------
@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", STEPS)
def test_model_values_are_bit_identical_to_the_instances_without_parameters(kind, steps):
    w, desc, ids = world(kind)
    vals = model_values(w)
    out, J = emu.rigid_step(desc, w["state"], w["force"], steps, jacobian=True, **w["params"])
    r = erp.step(desc, w["state"], ids, vals, w["force"], steps, jac_in=True, **w["params"])
    assert np.array_equal(r["state"], emu.rigid_step(desc, w["state"], w["force"], steps, **w["params"]))
    assert np.array_equal(r["jac"], J)
    n, rows, cols = J.shape
    nb = rows // 13
    g = np.random.default_rng(5).normal(size=(n, rows))
    gs0, gf0, _ = emu_vjp.rigid_vjp(desc, w["state"], g, w["force"], steps, **w["params"])
    gs1, gf1, _, _ = erp.vjp(desc, w["state"], ids, vals, g, w["force"], steps, **w["params"])
    assert np.array_equal(gs1, gs0) and np.array_equal(gf1, gf0)
    V = np.random.default_rng(6).normal(size=(n, cols, 2))
    ts, tf = V[:, :rows].reshape(n, nb, 13, 2), V[:, rows:].reshape(n, nb, 3, 2)
    so0, to0 = emu_jvp.rigid_jvp(desc, w["state"], ts, tf, w["force"], steps, **w["params"])
    so1, to1 = erp.jvp(desc, w["state"], ids, vals, ts, tf, None, w["force"], steps, **w["params"])
    assert np.array_equal(so1, so0) and np.array_equal(to1, to0)


# ---- 2. per-world values: the kernel on a description edited with the world's values, bit for bit -------------------------------------
@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", STEPS)
def test_per_world_values_equal_edited_descriptions(kind, steps):
    w, desc, ids = world(kind)
    vals = random_values(w, ids, N, 7)
    r = erp.step(desc, w["state"], ids, vals, w["force"], steps, jac_in=steps < 20, **w["params"])
    for e in range(N):
        d, p = edited(w, ids, vals[e])
        out = emu.rigid_step(d, w["state"][e:e + 1], w["force"][e:e + 1], steps, jacobian=steps < 20, **p)
        if steps < 20:
            assert np.array_equal(r["state"][e], out[0][0]) and np.array_equal(r["jac"][e], out[1][0])
        else:
            assert np.array_equal(r["state"][e], out[0])


# ---- 3. the parameter Jacobian against central differences of the fp64 forward instance --------------------------------------------
@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3])
def test_param_jacobian_vs_central_differences(kind, steps):
    w, desc, ids = world(kind)
    vals = random_values(w, ids, N, 8)
    Jp = erp.step(desc, w["state"], ids, vals, w["force"], steps, jac_par=True, **w["params"])["jac_par"]
    h = 1e-6
    ok = []
    for e in range(N):
        fd = np.zeros_like(Jp[e])
        for j in range(len(ids)):
            f = []
            for sgn in (1.0, -1.0):
                v = vals[e].copy()
                v[j] += sgn * h
                d, p = edited(w, ids, v)
                f.append(emu.rigid_step(d, w["state"][e:e + 1], w["force"][e:e + 1], steps, **p)[0].reshape(-1))
            fd[:, j] = (f[0] - f[1]) / (2 * h)
        ok.append(np.all(np.abs(Jp[e] - fd) <= 1e-5 * np.maximum(1.0, np.abs(Jp[e]))))
    # (the bar of test_rigid_jacobian_by_dual_numbers_vs_central_differences: a contact switching within +-h breaks a few worlds)
    assert np.mean(ok) >= 0.75, np.mean(ok)


# ---- 4. forward mode --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", STEPS)
def test_parameter_tangents(kind, steps):
    w, desc, ids = world(kind)
    k = len(ids)
    vals = random_values(w, ids, N, 9)
    r = erp.step(desc, w["state"], ids, vals, w["force"], steps, jac_in=True, jac_par=True, **w["params"])
    J, Jp = r["jac"], r["jac_par"]
    n, rows, cols = J.shape
    nb = rows // 13
    # identity parameter tangents: the parameter Jacobian, bit for bit
    eye = np.ascontiguousarray(np.broadcast_to(np.eye(k), (n, k, k)))
    so, to = erp.jvp(desc, w["state"], ids, vals, t_par=eye, force=w["force"], steps=steps, **w["params"])
    assert np.array_equal(to.reshape(n, rows, k), Jp)
    assert np.array_equal(so, r["state"])
    # random input and parameter tangents together: J V + J_par W
    rng = np.random.default_rng(10)
    V, Wt = rng.normal(size=(n, cols, 3)), rng.normal(size=(n, k, 3))
    ts, tf = V[:, :rows].reshape(n, nb, 13, 3), V[:, rows:].reshape(n, nb, 3, 3)
    _, to = erp.jvp(desc, w["state"], ids, vals, ts, tf, Wt, w["force"], steps, **w["params"])
    assert rel_jv(to.reshape(n, rows, 3), np.concatenate([J, Jp], axis=2), np.concatenate([V, Wt], axis=1)) <= 1e-12
    # m tangents in one call are m calls of one tangent each, bit for bit
    for j in range(3):
        _, one = erp.jvp(desc, w["state"], ids, vals, ts[..., j:j + 1], tf[..., j:j + 1], Wt[..., j:j + 1], w["force"], steps, **w["params"])
        assert np.array_equal(one[..., 0], to[..., j])


# ---- 5. reverse mode --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", STEPS)
def test_parameter_vjp(kind, steps):
    w, desc, ids = world(kind)
    k = len(ids)
    vals = random_values(w, ids, N, 11)
    Jp = erp.step(desc, w["state"], ids, vals, w["force"], steps, jac_par=True, **w["params"])["jac_par"]
    n, rows, _ = Jp.shape
    rng = np.random.default_rng(12)
    g = rng.normal(size=(n, rows))
    gs, gf, gp, st = erp.vjp(desc, w["state"], ids, vals, g, w["force"], steps, tape_cap=1 << 16, **w["params"])
    # g_par = g^T J_par of the dual instance over all the steps
    ref = np.einsum("er,erk->ek", g, Jp)
    assert np.max(np.abs(gp - ref) / np.maximum(1.0, np.einsum("er,erk->ek", np.abs(g), np.abs(Jp)))) <= 1e-12
    # duality with forward mode: <g, J_par w> = <g_par, w>
    wv = rng.normal(size=(n, k, 1))
    _, to = erp.jvp(desc, w["state"], ids, vals, t_par=wv, force=w["force"], steps=steps, **w["params"])
    assert rel(np.einsum("er,er->e", g, to.reshape(n, rows)), np.einsum("ek,ek->e", gp, wv[..., 0])) <= 1e-10
    # chunks rerun from a 64-node tape: bit-identical to a run that never regrew (the staging of g_par counts a rerun chunk once)
    gs2, gf2, gp2, st2 = erp.vjp(desc, w["state"], ids, vals, g, w["force"], steps, tape_cap=64, chunk=2, **w["params"])
    assert st["reruns"] == 0 and st2["reruns"] > 0
    assert np.array_equal(gs2, gs) and np.array_equal(gf2, gf) and np.array_equal(gp2, gp)


# ---- 6. refused ids and values ----------------------------------------------------------------------------------------------------
REFUSALS = [
    ("id out of range", "stack", [2 + 4 * 5], None, -2),
    ("negative id", "stack", [-1], None, -2),
    ("duplicate", "stack", [0, 3, 0], None, -2),
    ("static mass", "static", [2 + 4 * 1], None, -2),
    ("sphere length", "stack", [2 + 4 * 1 + 2], None, -2),
    ("capsule extent_z", "stack", [2 + 4 * 3 + 3], None, -2),
    ("plane mass", "stack", [2], None, -2),
    ("plane normal", "stack", [3], None, -2),
    ("zero mass", "stack", [6], [0.0], -3),
    ("negative radius", "stack", [7], [-0.3], -3),
    ("negative friction", "stack", [0], [-0.1], -3),
    ("negative restitution", "stack", [1], [-0.5], -3),
    ("nan", "stack", [0], [np.nan], -3),
    ("inf size", "stack", [19], [np.inf], -3),
]


def refusal_bodies(kind):
    if kind == "static":   # a static sphere (model mass 0) among dynamic ones
        return np.asarray([rg.sphere(1.0, 0.5), rg.sphere(0.0, 0.5), rg.sphere(2.0, 0.3)], dtype=np.float64)
    return wl.rigid_world(kind, 1)["bodies"]


@pytest.mark.parametrize("what,kind,ids,values,rc", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refused_ids_and_values(what, kind, ids, values, rc):
    with pytest.raises(erp.Refused) as ex:
        erp.check(refusal_bodies(kind), ids, values)
    assert ex.value.rc == rc
    if values is not None:   # the ids themselves are accepted
        erp.check(refusal_bodies(kind), ids)


def test_accepted_ids_and_names():
    desc = wl.rigid_world("stack", 1)["bodies"]
    names = rg.param_names(desc)
    assert names == ["friction", "restitution", "body1.mass", "body1.radius", "body2.mass", "body2.radius", "body3.mass", "body3.radius",
                     "body3.length", "body4.mass", "body4.extent_x", "body4.extent_y", "body4.extent_z"]
    ids = all_ids(desc)
    assert ids == [0, 1, 6, 7, 10, 11, 14, 15, 16, 18, 19, 20, 21]
    erp.check(desc, ids, rg.param_values(desc))
    assert np.allclose(rg.param_values(desc, friction=0.6), [0.6, 0.0, 1.0, 0.3, 2.0, 0.2, 1.5, 0.15, 0.6, 2.0, 0.4, 0.3, 0.2])
    erp.check(refusal_bodies("static"), rg.param_ids(refusal_bodies("static"), ["body1.radius", "body2.mass"]))
    with pytest.raises(ValueError):
        rg.param_ids(desc, ["body0.mass"])


# ---- 7. system identification: two ball masses and the restitution from observed collisions ------------------------------------------
SYSID_STEPS, SYSID_ITERS, SYSID_LR = 30, 120, 0.05
SYSID_NAMES = ["body1.mass", "body2.mass", "restitution"]
SYSID_TRUE = np.array([1.7, 0.6, 0.5])
SYSID_START = np.array([1.25, 0.8, 0.35])      # 26 %, 33 % and 30 % off


def sysid_setup(n=4):
    """Billiard worlds (no gravity, 50 solver sweeps, the balls roll on the table plane z = 0): a cue ball of known mass 1 runs into
    ball 1, which runs into ball 2; each world with its own cue velocity and offsets.  Returns (bodies, states, World parameters)."""
    bodies = np.asarray([rg.sphere(1.0, 0.5)] * 3, dtype=np.float64)
    r = np.random.default_rng(71)
    state = rg.identity_state(n, 3)
    state[:, 0, 0] = -1.4
    state[:, 0, 1] = r.uniform(-0.15, 0.15, n)
    state[:, 2, 0] = 1.15
    state[:, 2, 1] = r.uniform(-0.15, 0.15, n)
    state[:, 0, 7] = r.uniform(2.5, 3.5, n)
    state[:, 0, 8] = r.uniform(-0.3, 0.3, n)
    params = dict(gravity=(0.0, 0.0, 0.0), num_solver_iterations=50)
    return bodies, state, params


def adam(theta, grad, mom, it, lr=SYSID_LR, b1=0.9, b2=0.999, eps=1e-12):
    m, v = mom
    m = b1 * m + (1 - b1) * grad
    v = b2 * v + (1 - b2) * grad * grad
    step = lr * (m / (1 - b1 ** (it + 1))) / (np.sqrt(v / (1 - b2 ** (it + 1))) + eps)
    return theta - step, (m, v)


def sysid_descent(loss_grad):
    """Adam on the log-parameters; loss_grad(p [3]) -> (loss, dloss / dp [3]).  Returns (losses, final parameters)."""
    theta = np.log(SYSID_START)
    mom = (np.zeros(3), np.zeros(3))
    losses = []
    for it in range(SYSID_ITERS):
        p = np.exp(theta)
        loss, g = loss_grad(p)
        losses.append(loss)
        theta, mom = adam(theta, g * p, mom, it)
    return np.array(losses), np.exp(theta)


def sysid_host_loss_grad():
    bodies, state, params = sysid_setup()
    ids = rg.param_ids(bodies, SYSID_NAMES)
    n = state.shape[0]
    obs = erp.step(bodies, state, ids, SYSID_TRUE, None, SYSID_STEPS, **params)["state"]

    def loss_grad(p):
        out = erp.step(bodies, state, ids, p, None, SYSID_STEPS, **params)["state"]
        d = out - obs
        _, _, gp, _ = erp.vjp(bodies, state, ids, p, 2 * d.reshape(n, -1), None, SYSID_STEPS, **params)
        return float(np.sum(d * d)), gp.sum(axis=0)
    return loss_grad


def test_system_identification_on_the_host_build():
    losses, p = sysid_descent(sysid_host_loss_grad())
    assert np.all(np.abs(p - SYSID_TRUE) <= 0.01 * SYSID_TRUE), p
    # the recorded trajectory of this rehearsal: tests/test_rigid_params_gpu.py runs the same descent through autograd against it
    rehearsal = np.load(os.path.join(GOLDEN, "rigid_sysid_losses.npy"))
    assert np.max(np.abs(losses - rehearsal) / np.maximum(1e-12, np.abs(rehearsal))) <= 1e-9
