"""Per-world physical parameters of the rigid-body world on the H100 (DESIGN.md section 7.11): the PAR instances of csrc/tds_rigid.cu as
nvcc builds them, through the C-ABI, RigidWorld and tds_b200.autograd.rigid_step.  Different nvcc instances may contract FMAs
differently, so device results are compared within 1e-12 (forward) or 1e-10 (derivatives); results of the same instance bit for bit.
tests/test_rigid_params_on_host.py checks the same kernel source on the CPU."""
import ctypes
import os

import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
import emu_rigid_params as erp
from test_rigid_params_on_host import (SYSID_ITERS, SYSID_NAMES, SYSID_START, SYSID_STEPS, SYSID_TRUE, all_ids, edited, model_values,
                                       random_values, sysid_descent, sysid_setup)
from test_kernel_source_on_host import GOLDEN
from test_vjp_gpu import rel

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def make(kind, n, seed=41):
    w = wl.rigid_world(kind, n, seed=seed)
    return w, tds_b200.RigidWorld(w["bodies"], n, **w["params"]), all_ids(w["bodies"])


def everything(world, w, steps, g, V, Wt=None):
    """Forward, input Jacobian, VJP and JVP of the world as it is installed (plus the parameter derivatives when Wt is given)."""
    n, nb = world.n_worlds, world.n_bodies
    rows = 13 * nb
    out = dict(state=world.step(w["state"], w["force"], steps))
    out["jac"] = world.step_jacobian(w["state"], w["force"], steps)[1]
    out["gs"], out["gf"] = world.step_vjp(w["state"], w["force"], g, steps)
    ts, tf = V[:, :rows].reshape(n, nb, 13, -1), V[:, rows:].reshape(n, nb, 3, -1)
    out["jvp"] = world.step_jvp(w["state"], w["force"], ts, tf, steps)[1]
    if Wt is not None:
        out["jac_par"] = world.step_param_jacobian(w["state"], w["force"], steps)[1]
        out["gs_p"], out["gf_p"], out["gp"] = world.step_vjp_params(w["state"], w["force"], g, steps)
        out["jvp_p"] = world.step_jvp(w["state"], w["force"], ts, tf, steps, t_par=Wt)[1]
    return out


def inputs(w, nb, seed):
    n = w["state"].shape[0]
    rng = np.random.default_rng(seed)
    return rng.normal(size=(n, 13 * nb)).reshape(n, nb, 13), rng.normal(size=(n, 16 * nb, 2))


@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3])
def test_model_values_and_clearing(kind, steps):
    """Every id installed at the description's values against the instances without parameters (1e-12), and clearing the set gives
    the results before the install back bit for bit."""
    w, world, ids = make(kind, 40)
    g, V = inputs(w, world.n_bodies, 3)
    before = everything(world, w, steps, g, V)
    world.set_physical_params(ids, model_values(w))
    inst = everything(world, w, steps, g, V)
    for key in before:
        assert rel(inst[key], before[key]) <= 1e-12, key
    world.set_physical_params(None)
    after = everything(world, w, steps, g, V)
    for key in before:
        assert np.array_equal(after[key], before[key]), key


@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3])
def test_per_world_values_equal_edited_worlds(kind, steps):
    n = 8
    w, world, ids = make(kind, n)
    vals = random_values(w, ids, n, 4)
    world.set_physical_params(ids, vals)
    out = world.step(w["state"], w["force"], steps)
    _, J = world.step_jacobian(w["state"], w["force"], steps)
    for e in range(n):
        d, p = edited(w, ids, vals[e])
        one = tds_b200.RigidWorld(d, 1, **p)
        assert rel(out[e], one.step(w["state"][e:e + 1], w["force"][e:e + 1], steps)[0]) <= 1e-12
        assert rel(J[e], one.step_jacobian(w["state"][e:e + 1], w["force"][e:e + 1], steps)[1][0]) <= 1e-12


@pytest.mark.parametrize("kind", wl.RIGID_WORLDS)
@pytest.mark.parametrize("steps", [1, 3, 20])
def test_device_against_the_host_build(kind, steps):
    n = 12
    w, world, ids = make(kind, n)
    k = len(ids)
    vals = random_values(w, ids, n, 5)
    world.set_physical_params(ids, vals)
    g, V = inputs(w, world.n_bodies, 6)
    Wt = np.random.default_rng(7).normal(size=(n, k, 2))
    dev = everything(world, w, steps, g, V, Wt)
    rows = 13 * world.n_bodies
    host = erp.step(w["bodies"], w["state"], ids, vals, w["force"], steps, jac_in=True, jac_par=True, **w["params"])
    assert rel(dev["state"], host["state"]) <= 1e-12
    assert rel(dev["jac"], host["jac"]) <= 1e-10 and rel(dev["jac_par"], host["jac_par"]) <= 1e-10
    gs, gf, gp, _ = erp.vjp(w["bodies"], w["state"], ids, vals, g, w["force"], steps, tape_cap=1 << 16, **w["params"])
    assert rel(dev["gs_p"], gs) <= 1e-10 and rel(dev["gf_p"], gf) <= 1e-10 and rel(dev["gp"], gp) <= 1e-10
    assert np.array_equal(dev["gs_p"], dev["gs"]) and np.array_equal(dev["gf_p"], dev["gf"])
    ts, tf = V[:, :rows].reshape(n, -1, 13, 2), V[:, rows:].reshape(n, -1, 3, 2)
    _, to = erp.jvp(w["bodies"], w["state"], ids, vals, ts, tf, Wt, w["force"], steps, **w["params"])
    assert rel(dev["jvp_p"], to) <= 1e-10


def test_ragged_batches_are_bit_identical_to_a_full_batch():
    full_n, steps = 100, 3
    w, world, ids = make("stack", full_n, seed=8)
    k = len(ids)
    vals = random_values(w, ids, full_n, 9)
    g, _ = inputs(w, world.n_bodies, 10)
    Wt = np.random.default_rng(11).normal(size=(full_n, k, 1))

    def run(wd, n):
        wd.set_physical_params(ids, vals[:n])
        s, f = w["state"][:n], w["force"][:n]
        return (wd.step(s, f, steps), wd.step_param_jacobian(s, f, steps)[1], wd.step_vjp_params(s, f, g[:n], steps),
                wd.step_jvp(s, f, None, None, steps, t_par=Wt[:n])[1])
    ref = run(world, full_n)
    for n in (1, 31, 33, 100):
        got = run(tds_b200.RigidWorld(w["bodies"], n, **w["params"]), n)
        assert np.array_equal(got[0], ref[0][:n]) and np.array_equal(got[1], ref[1][:n]) and np.array_equal(got[3], ref[3][:n])
        for a, b in zip(got[2], ref[2]):
            assert np.array_equal(a, b[:n])


def test_4096_world_billiard_vjp_regrows_its_tape():
    """The chunked, checkpointed reverse pass of 4096 billiard worlds with parameters, from a tape that has to grow (its chunks rerun),
    against the host build on every 128th world."""
    import torch
    n, steps = 4096, 3
    w, world, ids = make("billiard", n, seed=12)
    vals = random_values(w, ids, n, 13)
    world.set_physical_params(ids, vals)
    g = np.random.default_rng(14).normal(size=(n, 13 * world.n_bodies))
    ns, nb = world.n_stride, world.n_bodies
    soa = lambda a, d: torch.tensor(np.pad(a.reshape(n, d).T, ((0, 0), (0, ns - n))), dtype=torch.float64, device=DEV).contiguous()
    s, f, go = soa(w["state"], 13 * nb), soa(w["force"], 3 * nb), soa(g, 13 * nb)
    gs, gf = torch.zeros_like(s), torch.zeros_like(f)
    gp = torch.zeros((len(ids), ns), dtype=torch.float64, device=DEV)
    world.step_vjp_params_device(s, f, go, gs, gf, gp, steps)
    torch.cuda.synchronize()
    sub = np.arange(0, n, 128)
    hs, hf, hp, st = erp.vjp(w["bodies"], w["state"][sub], ids, vals[sub], g[sub], w["force"][sub], steps, tape_cap=4096, **w["params"])
    assert st["reruns"] > 0          # (the world starts at the same 4096 nodes)
    assert rel(gs.cpu().numpy()[:, sub].T.reshape(len(sub), nb, 13), hs) <= 1e-10
    assert rel(gf.cpu().numpy()[:, sub].T.reshape(len(sub), nb, 3), hf) <= 1e-10
    assert rel(gp.cpu().numpy()[:, sub].T, hp) <= 1e-10


def test_autograd_backward_over_chained_calls():
    import torch
    n = 24
    w, world, ids = make("swapped", n, seed=15)
    k = len(ids)
    v1, v2 = random_values(w, ids, n, 16), random_values(w, ids, 1, 17)[0]
    world.set_physical_params(ids, v1)
    s0 = torch.tensor(w["state"], device=DEV, requires_grad=True)
    f0 = torch.tensor(w["force"], device=DEV, requires_grad=True)
    p1 = torch.tensor(v1, device=DEV, requires_grad=True)
    p2 = torch.tensor(v2, device=DEV, requires_grad=True)          # one value for all worlds: a [k] leaf expanded
    s1 = tds_b200.autograd.rigid_step(world, s0, f0, 2, params=p1)
    s2 = tds_b200.autograd.rigid_step(world, s1, None, 3, params=p2.expand(n, k))
    g = np.random.default_rng(18).normal(size=(n, world.n_bodies, 13))
    (s2 * torch.tensor(g, device=DEV)).sum().backward()
    # the chain of step_vjp_params, each with the values of its call
    world.set_physical_params(ids, v2)
    gs1, _, gp2 = world.step_vjp_params(s1.detach().cpu().numpy(), None, g, 3)
    world.set_physical_params(ids, v1)
    gs0, gf0, gp1 = world.step_vjp_params(w["state"], w["force"], gs1, 2)
    assert rel(s0.grad.cpu().numpy(), gs0) <= 1e-12 and rel(f0.grad.cpu().numpy(), gf0) <= 1e-12
    assert rel(p1.grad.cpu().numpy(), gp1) <= 1e-12
    assert rel(p2.grad.cpu().numpy(), gp2.sum(axis=0)) <= 1e-12


def test_forward_mode_with_parameter_tangents():
    import torch
    import torch.autograd.forward_ad as fwAD
    n, steps = 16, 5
    w, world, ids = make("stack", n, seed=19)
    k = len(ids)
    vals = random_values(w, ids, n, 20)
    world.set_physical_params(ids, vals)
    rng = np.random.default_rng(21)
    ts, tf, tp = rng.normal(size=(n, world.n_bodies, 13)), rng.normal(size=(n, world.n_bodies, 3)), rng.normal(size=(n, k))
    _, ref = world.step_jvp(w["state"], w["force"], ts, tf, steps, t_par=tp)
    _, ref_p = world.step_jvp(w["state"], w["force"], None, None, steps, t_par=tp)
    s, f, p = (torch.tensor(a, device=DEV) for a in (w["state"], w["force"], vals))
    vs, vf, vp = (torch.tensor(a, device=DEV) for a in (ts, tf, tp))
    world.set_physical_params(ids, model_values(w))       # the rules install the values of their own call
    with fwAD.dual_level():
        out = tds_b200.autograd.rigid_step(world, fwAD.make_dual(s, vs), fwAD.make_dual(f, vf), steps, params=fwAD.make_dual(p, vp))
        tan = fwAD.unpack_dual(out).tangent.clone().cpu().numpy()
        out = tds_b200.autograd.rigid_step(world, s, f, steps, params=fwAD.make_dual(p, vp))
        tan_p = fwAD.unpack_dual(out).tangent.clone().cpu().numpy()
    assert rel(tan, ref) <= 1e-12 and rel(tan_p, ref_p) <= 1e-12
    _, (ft,) = torch.func.jvp(lambda a, b, c: (tds_b200.autograd.rigid_step(world, a, b, steps, params=c),), (s, f, p), (vs, vf, vp))
    assert rel(ft.cpu().numpy(), ref) <= 1e-12


def test_system_identification_through_autograd():
    """The descent of tests/test_rigid_params_on_host.py with the gradient from loss.backward() through rigid_step(..., params=)."""
    import torch
    bodies, state, params = sysid_setup()
    n = state.shape[0]
    world = tds_b200.RigidWorld(bodies, n, **params)
    world.set_physical_params(SYSID_NAMES, SYSID_TRUE)
    obs = torch.tensor(world.step(state, None, SYSID_STEPS), device=DEV)
    world.set_physical_params(SYSID_NAMES, SYSID_START)
    s = torch.tensor(state, device=DEV)

    def loss_grad(pv):
        p = torch.tensor(pv, device=DEV, requires_grad=True)
        out = tds_b200.autograd.rigid_step(world, s, None, SYSID_STEPS, params=p.expand(n, 3))
        loss = ((out - obs) ** 2).sum()
        loss.backward()
        return float(loss), p.grad.cpu().numpy()
    losses, p = sysid_descent(loss_grad)
    rehearsal = np.load(os.path.join(GOLDEN, "rigid_sysid_losses.npy"))
    assert len(losses) == SYSID_ITERS
    assert np.max(np.abs(losses - rehearsal) / np.abs(rehearsal)) <= 1e-6
    assert np.all(np.abs(p - SYSID_TRUE) <= 0.01 * SYSID_TRUE), p


def test_argument_checks():
    import torch
    L = tds_b200._lib.lib()
    w, world, ids = make("stack", 4)
    h, nb, ns = world._h, world.n_bodies, world.n_stride
    rows = 13 * nb
    p = lambda a: ctypes.c_void_p(a.data_ptr()) if a is not None else None
    hp = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
    idv = np.asarray(ids[:3], dtype=np.int32)
    assert L.tds_b200_rigid_param_count(None) == -1 and L.tds_b200_rigid_param_count(h) == 2 + 4 * nb
    # installation
    sh = lambda k, i, v: L.tds_b200_rigid_set_physical_params_host(h, k, hp(i), hp(v))
    good = np.ascontiguousarray(np.broadcast_to(model_values(w)[:3], (4, 3)))
    assert L.tds_b200_rigid_set_physical_params_host(None, 3, hp(idv), hp(good)) == -1
    assert sh(3, None, good) == -1 and sh(3, idv, None) == -1 and sh(-1, idv, good) == -1
    assert sh(1, np.asarray([22], dtype=np.int32), good) == -2 and "out of range" in tds_b200._lib.last_error()
    assert sh(2, np.asarray([0, 0], dtype=np.int32), good) == -2 and "twice" in tds_b200._lib.last_error()
    assert sh(1, np.asarray([2], dtype=np.int32), good) == -2 and "plane" in tds_b200._lib.last_error()
    assert sh(1, np.asarray([8], dtype=np.int32), good) == -2 and "size component" in tds_b200._lib.last_error()
    bad = good.copy(); bad[2, 2] = 0.0
    assert sh(3, idv, bad) == -3
    vd = torch.full((3, ns), -1.0, dtype=torch.float64, device=DEV)     # the device entry copies without checking the values
    assert L.tds_b200_rigid_set_physical_params_device(h, 3, hp(np.asarray([0, 1, 2], dtype=np.int32)), p(vd), None) == -2
    assert L.tds_b200_rigid_set_physical_params_device(h, 3, hp(idv), p(vd), None) == 0
    assert sh(0, None, None) == 0
    # derivative entries: argument checks (-1), then -4 without a set
    s, f = np.ascontiguousarray(w["state"]), np.ascontiguousarray(w["force"])
    jac, gs, gf, gp = np.zeros((4, rows, 3)), np.zeros_like(s), np.zeros_like(f), np.zeros((4, 3))
    to, tpar = np.zeros((4, rows, 1)), np.zeros((4, 3, 1))
    pj = lambda j, st=1: L.tds_b200_rigid_param_jacobian_host(h, hp(s), hp(f), st, None, hp(j))
    vh = lambda g_par, st=1: L.tds_b200_rigid_vjp_params_host(h, hp(s), hp(f), st, hp(s), hp(gs), hp(gf), hp(g_par))
    jh = lambda m, tp, t_out=to: L.tds_b200_rigid_jvp_params_host(h, hp(s), hp(f), 1, m, None, None, hp(tp), None, hp(t_out))
    ds = torch.zeros((rows, ns), dtype=torch.float64, device=DEV)
    dgs, dgp = torch.zeros_like(ds), torch.zeros((3, ns), dtype=torch.float64, device=DEV)
    dto, dtp = torch.zeros((rows, ns), dtype=torch.float64, device=DEV), torch.zeros((3, ns), dtype=torch.float64, device=DEV)
    vd_ = lambda g_par, st=1: L.tds_b200_rigid_vjp_params_device(h, p(ds), None, st, p(ds), p(dgs), None, p(g_par), None)
    jd = lambda m, tp, so=None: L.tds_b200_rigid_jvp_params_device(h, p(ds), None, 1, m, None, None, p(tp), p(so), p(dto), None)
    for rc_fn in (lambda: pj(jac), lambda: vh(gp), lambda: jh(1, tpar), lambda: vd_(dgp), lambda: jd(1, dtp)):
        assert rc_fn() == -4 and "no physical parameters" in tds_b200._lib.last_error()
    assert pj(None) == -1 and pj(jac, -1) == -1
    assert vh(None) == -1 and vh(gp, -1) == -1 and vd_(None) == -1 and vd_(dgp, -1) == -1
    assert jh(0, tpar) == -1 and jh(1, None) == -1 and jh(1, tpar, None) == -1
    assert jd(0, dtp) == -1 and jd(1, None) == -1 and jd(1, dtp, ds) == -1      # state_out aliasing state
    assert sh(3, idv, good) == 0
    assert pj(jac) == 0 and vh(gp) == 0 and jh(1, tpar) == 0 and vd_(dgp) == 0 and jd(1, dtp) == 0
    # the existing entries run with a set installed too (the VJP without g_par)
    assert L.tds_b200_rigid_vjp_device(h, p(ds), None, 1, p(ds), p(dgs), None, None) == 0
    torch.cuda.synchronize()
