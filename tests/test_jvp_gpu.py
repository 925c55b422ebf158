"""Forward mode on the H100 (DESIGN.md section 7.10): the Jacobian-vector products of the step (tangent-seeded dual instances of the
world-frame kernel) and of the rigid-body world, against the host build of the same source, against the device Jacobian, on ragged
and chunked batches, through torch.autograd.forward_ad and torch.func.jvp, and in a system identification gradient.  The CPU twins
are in tests/test_jvp_on_host.py."""
import ctypes

import numpy as np
import pytest

import tds_b200
import tds_b200.workloads as wl
from tds_b200.model import param_names
from test_vjp_gpu import _case, rel

pytestmark = pytest.mark.gpu

CASES = ["pendulum5", "cartpole", "sphere2", "box", "humanoid", "laikago_pd", "mb_three_bodies", "humanoid_spherical"]


def rel_jv(out, J, V):
    """|t_out - J V| relative to sum_c |J_rc| |V_cj| (at least 1), the rounding bound of the contraction."""
    return float(np.max(np.abs(out - np.einsum("erc,ecj->erj", J, V)) / np.maximum(1.0, np.einsum("erc,ecj->erj", np.abs(J), np.abs(V)))))


def all_ids(model):
    names = param_names(model)
    return [i for i, nm in enumerate(names) if int(model[2]) or not nm.startswith("base.")]


def _params_of(name):
    if name == "laikago_pd":
        return 1.0, 0.0
    if name == "mb_three_bodies":
        return wl.multibody_world("three_bodies", 1)["params"].get("friction", 0.5), 0.0
    p = getattr(wl, name)(1, seed=0)["params"]
    return p.get("friction", 0.5), p.get("restitution", 0.0)


def _install(sim, name, n, seed):
    from test_params_on_host import perturbed
    ids = all_ids(sim.model)
    vals = perturbed(sim.model, ids, n, seed, *_params_of(name))
    sim.set_physical_params(ids, vals)
    return ids, vals


@pytest.mark.parametrize("name", CASES)
def test_jvp_against_the_device_jacobian(name):
    """Identity tangents against the dual Jacobian of the device (another instance: nvcc may contract differently, hence 1e-12 and
    not bit identity); random tangents against J V."""
    n = 24
    sim, mode, q, qd, t, pd = _case(name, n)
    J = sim.step_jacobian_host(mode, q, qd, t, use_pd=pd)
    _, rows, cols = J.shape
    eye = np.broadcast_to(np.eye(cols), (n, cols, cols))
    assert rel(sim.step_jvp_host(mode, q, qd, t, eye, use_pd=pd), J) <= 1e-12
    V = np.random.default_rng(1).normal(size=(n, cols, 3))
    assert rel_jv(sim.step_jvp_host(mode, q, qd, t, V, use_pd=pd), J, V) <= 1e-10
    # one tangent as [n, cols]: [n, rows]
    one = sim.step_jvp_host(mode, q, qd, t, V[:, :, 0], use_pd=pd)
    assert one.shape == (n, rows) and rel_jv(one[:, :, None], J, V[:, :, :1]) <= 1e-10


@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago_pd", "humanoid_spherical"])
def test_parameter_tangents_against_the_device_parameter_jacobian(name):
    n = 24
    sim, mode, q, qd, t, pd = _case(name, n)
    ids, _ = _install(sim, name, n, 2)
    k = len(ids)
    Jp = sim.step_param_jacobian_host(mode, q, qd, t, use_pd=pd)
    Ji = sim.step_jacobian_host(mode, q, qd, t, use_pd=pd)
    assert rel(sim.step_jvp_host(mode, q, qd, t, None, np.broadcast_to(np.eye(k), (n, k, k)), use_pd=pd), Jp) <= 1e-12
    rng = np.random.default_rng(3)
    V, W = rng.normal(size=(n, Ji.shape[2], 3)), rng.normal(size=(n, k, 3))
    out = sim.step_jvp_host(mode, q, qd, t, V, W, use_pd=pd)
    assert rel_jv(out, np.concatenate([Ji, Jp], axis=2), np.concatenate([V, W], axis=1)) <= 1e-10


def test_device_jvp_agrees_with_the_host_build():
    """Build agreement (the nvcc build against the same kernel source compiled for the CPU), not a reference check."""
    import emu_jvp
    for name in ("sphere2", "humanoid_spherical"):
        n = 8
        sim, mode, q, qd, t, _ = _case(name, n)
        w = getattr(wl, name)(n, seed=2718)
        _, cols = sim.jacobian_dims(mode)
        rng = np.random.default_rng(4)
        V = rng.normal(size=(n, cols, 3))
        assert rel(sim.step_jvp_host(mode, q, qd, t, V), emu_jvp.step_jvp(sim.model, mode, q, qd, t_in=V, tau=t, **w["params"])) <= 1e-5
        ids, vals = _install(sim, name, n, 5)
        W = rng.normal(size=(n, len(ids), 3))
        host = emu_jvp.step_jvp(sim.model, mode, q, qd, t_in=V, t_par=W, tau=t, ids=ids, values=vals, **w["params"])
        assert rel(sim.step_jvp_host(mode, q, qd, t, V, W), host) <= 1e-5


def test_ragged_batches_are_bit_identical_to_a_full_batch():
    n_full = 128
    sim, mode, q, qd, t, pd = _case("laikago_pd", n_full)
    _, cols = sim.jacobian_dims(mode, pd)
    V = np.random.default_rng(6).normal(size=(n_full, cols, 4))
    full = sim.step_jvp_host(mode, q, qd, t, V, use_pd=pd)
    for n in (1, 31, 33, 100):
        small = tds_b200.laikago_sim(n)
        out = small.step_jvp_host(mode, q[-n:], qd[-n:], t[-n:], V[-n:], use_pd=pd)
        assert np.array_equal(out, full[-n:]), n


def test_chunked_tangents_equal_single_chunk_calls():
    """A humanoid batch sized from the arena bound (2 GB of dual-number scratch per launch) so that the m tangents run in at least
    two launches; every tangent equals the same tangent computed in a call of one chunk."""
    probe, *_ = _case("humanoid", 32)
    per_warp = probe.jacobian_chunk()            # directions per launch with one warp of environments
    warps = per_warp // 3 + 1                      # -> at most 3 directions per launch
    n = 32 * warps
    sim, mode, q, qd, t, _ = _case("humanoid", n, seed=19)
    chunk = sim.jacobian_chunk()
    m = 2 * chunk + 1
    assert 1 <= chunk < m
    _, cols = sim.jacobian_dims(mode)
    V = np.random.default_rng(7).normal(size=(n, cols, m))
    out = sim.step_jvp_host(mode, q, qd, t, V)
    for j0 in range(0, m, chunk):
        part = sim.step_jvp_host(mode, q, qd, t, V[:, :, j0:j0 + chunk])
        assert np.array_equal(part, out[:, :, j0:j0 + chunk]), j0


def _rollout_setup(name, n, with_params, seed):
    import torch
    sim, mode, q, qd, t, pd = _case(name, n)
    md = 2 if mode == 0 else mode
    if t is None:
        t = np.zeros((n, sim.n_act if pd else sim.n_tau))
    dev = "cuda:0"
    vals = None
    if with_params:
        names = param_names(sim.model)
        ids = [i for i in all_ids(sim.model) if names[i].endswith(("mass", "damping", "com.z")) or i < 2]
        from test_params_on_host import perturbed
        vals = perturbed(sim.model, ids, n, 29, *_params_of(name))
        sim.set_physical_params(ids, vals)
    rng = np.random.default_rng(seed)
    x = dict(q=torch.tensor(q, dtype=torch.float32, device=dev), qd=torch.tensor(qd, dtype=torch.float32, device=dev),
             tau=torch.tensor(t, dtype=torch.float32, device=dev),
             par=None if vals is None else torch.tensor(vals, dtype=torch.float64, device=dev))
    v = {k: None if a is None else torch.tensor(rng.normal(size=tuple(a.shape)), dtype=a.dtype, device=dev) for k, a in x.items()}
    return sim, md, pd, x, v


def _roll(sim, md, pd, steps, q, qd, tau, par):
    for _ in range(steps):
        q, qd = tds_b200.autograd.step(sim, q, qd, tau, mode=md, use_pd=pd, params=par)
    return q, qd


@pytest.mark.parametrize("with_params", [False, True])
@pytest.mark.parametrize("name", ["cartpole", "sphere2", "laikago_pd"])
def test_forward_mode_autograd_through_a_rollout(name, with_params):
    import torch
    import torch.autograd.forward_ad as fwAD
    n, steps = 16, 5
    sim, md, pd, x, v = _rollout_setup(name, n, with_params, 8)
    keys = ("q", "qd", "tau", "par") if with_params else ("q", "qd", "tau")
    # 1. torch.autograd.forward_ad
    states = []
    with fwAD.dual_level():
        d = {k: fwAD.make_dual(x[k], v[k]) for k in keys}
        q, qd = d["q"], d["qd"]
        for _ in range(steps):
            states.append((fwAD.unpack_dual(q).primal.cpu().numpy().astype(np.float64), fwAD.unpack_dual(qd).primal.cpu().numpy().astype(np.float64)))
            q, qd = tds_b200.autograd.step(sim, q, qd, d["tau"], mode=md, use_pd=pd, params=d.get("par"))
        tq, tqd = fwAD.unpack_dual(q).tangent.clone(), fwAD.unpack_dual(qd).tangent.clone()
    assert tq.dtype == torch.float32 and tqd.dtype == torch.float32
    # the chain of Jacobians by hand, the state tangent rounded to float32 between steps as the rule returns it
    nx = sim.n_q + sim.n_qd
    vs = np.concatenate([v["q"].cpu().numpy(), v["qd"].cpu().numpy()], axis=1).astype(np.float64)
    vt = v["tau"].cpu().numpy().astype(np.float64)
    vp = v["par"].cpu().numpy() if with_params else None
    t_np = x["tau"].cpu().numpy().astype(np.float64)
    for k in range(steps):
        J = sim.step_jacobian_host(md, states[k][0], states[k][1], t_np, use_pd=pd)
        vin = np.concatenate([vs, vt, np.zeros((n, J.shape[2] - nx - vt.shape[1]))], axis=1)
        jv = np.einsum("erc,ec->er", J, vin)
        if with_params:
            jv += np.einsum("erk,ek->er", sim.step_param_jacobian_host(md, states[k][0], states[k][1], t_np, use_pd=pd), vp)
        vs = jv.astype(np.float32).astype(np.float64)
    got = np.concatenate([tq.cpu().numpy(), tqd.cpu().numpy()], axis=1).astype(np.float64)
    assert rel(got, vs) <= 1e-6
    # 2. torch.func.jvp: the same rule
    prim = tuple(x[k] for k in keys)
    tang = tuple(v[k] for k in keys)
    fn = lambda *a: _roll(sim, md, pd, steps, a[0], a[1], a[2], a[3] if with_params else None)
    _, (fq, fqd) = torch.func.jvp(fn, prim, tang)
    assert rel(torch.cat([fq, fqd], 1).cpu().numpy().astype(np.float64), got) <= 1e-12
    # 3. forward and backward through the same rollout: <g, J v> = <J^T g, v>
    req = {k: x[k].clone().requires_grad_(True) for k in keys}
    q, qd = _roll(sim, md, pd, steps, req["q"], req["qd"], req["tau"], req.get("par"))
    rng = np.random.default_rng(9)
    wq = torch.tensor(rng.normal(size=(n, sim.n_q)), dtype=torch.float32, device="cuda:0")
    wqd = torch.tensor(rng.normal(size=(n, sim.n_qd)), dtype=torch.float32, device="cuda:0")
    ((q * wq).sum() + (qd * wqd).sum()).backward()
    fwd = float((tq.double() * wq.double()).sum() + (tqd.double() * wqd.double()).sum())
    rev = sum(float((req[k].grad.double() * v[k].double()).sum()) for k in keys)
    assert abs(fwd - rev) <= 1e-5 * max(1.0, abs(rev)), (fwd, rev)


def test_rigid_jvp_on_the_device():
    import torch
    import torch.autograd.forward_ad as fwAD
    import emu_jvp
    n, steps = 40, 20
    w = wl.rigid_world("billiard", n, seed=9)
    world = tds_b200.RigidWorld(w["bodies"], n, **w["params"])
    nb = world.n_bodies
    rng = np.random.default_rng(10)
    ts, tf = rng.normal(size=(n, nb, 13, 3)), rng.normal(size=(n, nb, 3, 3))
    so, to = world.step_jvp(w["state"], w["force"], ts, tf, steps)
    hso, hto = emu_jvp.rigid_jvp(w["bodies"], w["state"], ts, tf, w["force"], steps, **w["params"])
    assert rel(to, hto) <= 1e-12 and rel(so, hso) <= 1e-12
    # forward mode through rigid_step against J v of the dual Jacobian
    _, J = world.step_jacobian(w["state"], w["force"], steps)
    dev = "cuda:0"
    s = torch.tensor(w["state"], dtype=torch.float64, device=dev)
    f = torch.tensor(w["force"], dtype=torch.float64, device=dev)
    vs, vf = torch.tensor(ts[..., 0], device=dev), torch.tensor(tf[..., 0], device=dev)
    with fwAD.dual_level():
        out = tds_b200.autograd.rigid_step(world, fwAD.make_dual(s, vs), fwAD.make_dual(f, vf), steps)
        tan = fwAD.unpack_dual(out).tangent.clone().cpu().numpy()
    V = np.concatenate([ts[..., 0].reshape(n, -1), tf[..., 0].reshape(n, -1)], axis=1)
    assert rel_jv(tan.reshape(n, -1, 1), J, V[:, :, None]) <= 1e-10
    _, (ft,) = torch.func.jvp(lambda a, b: (tds_b200.autograd.rigid_step(world, a, b, steps),), (s, f), (vs, vf))
    assert rel(ft.cpu().numpy(), tan) <= 1e-12


def test_system_identification_gradient_by_forward_mode():
    """At the start point of the cartpole system identification (tests/test_params_on_host.py), the gradient of the rollout loss
    with respect to the 4 parameters by forward mode (m = 4 tangents carried in fp64 between steps through step_jvp_device) against
    params.grad of reverse-mode autograd."""
    import torch
    from test_params_on_host import SYSID_ENVS, SYSID_STEPS, sysid_problem
    model, ids, truth, start, q0, qd0, tau, kw = sysid_problem()
    n, dev, k = SYSID_ENVS, "cuda:0", 4
    sim = tds_b200.BatchSim(model, n, **kw)
    sim.set_physical_params(ids, start)
    ns, n_q, n_qd = sim.n_stride, sim.n_q, sim.n_qd
    rows, cols = sim.jacobian_dims(2)
    tau_t = [torch.tensor(tau[s], dtype=torch.float32, device=dev) for s in range(SYSID_STEPS)]
    x0 = torch.tensor(q0, dtype=torch.float32, device=dev)
    xd0 = torch.tensor(qd0, dtype=torch.float32, device=dev)

    def rollout(p):
        xs, x, xd = [], x0, xd0
        for s in range(SYSID_STEPS):
            x, xd = tds_b200.autograd.step(sim, x, xd, tau_t[s], params=p.unsqueeze(0).expand(n, -1).contiguous())
            xs.append((x, xd))
        return xs
    with torch.no_grad():
        target = [(a.detach().double(), b.detach().double()) for a, b in rollout(torch.tensor(truth, dtype=torch.float64, device=dev))]
    p = torch.tensor(start, dtype=torch.float64, device=dev, requires_grad=True)
    xs = rollout(p)
    loss = sum(((a.double() - ta) ** 2).sum() + ((b.double() - tb) ** 2).sum() for (a, b), (ta, tb) in zip(xs, target)) / n
    loss.backward()
    # forward mode: T = d state / d p [rows * k][ns] carried in fp64; parameter tangent j = the unit vector j in every environment
    sim.set_physical_params(ids, start)
    qs = torch.zeros((n_q, ns), dtype=torch.float32, device=dev); qs[:, :n] = x0.t()
    qds = torch.zeros((n_qd, ns), dtype=torch.float32, device=dev); qds[:, :n] = xd0.t()
    T = torch.zeros((rows * k, ns), dtype=torch.float64, device=dev)
    t_par = torch.zeros((k * k, ns), dtype=torch.float64, device=dev)
    for j in range(k):
        t_par[j * k + j, :n] = 1.0
    grad = torch.zeros(k, dtype=torch.float64, device=dev)
    for s in range(SYSID_STEPS):
        ts = torch.zeros((sim.n_tau, ns), dtype=torch.float32, device=dev); ts[:, :n] = tau_t[s].t()
        t_in = torch.zeros((cols * k, ns), dtype=torch.float64, device=dev)
        t_in[:rows * k] = T
        T = torch.zeros((rows * k, ns), dtype=torch.float64, device=dev)
        sim.step_jvp_device(2, qs, qds, ts, k, t_in, t_par, T)
        q1, qd1 = torch.empty_like(qs), torch.empty_like(qds)
        sim.step_device(2, qs, qds, ts, q_out=q1, qd_out=qd1)
        qs, qds = q1, qd1
        res = torch.cat([qs[:, :n].double() - target[s][0].t(), qds[:, :n].double() - target[s][1].t()], 0)   # [rows][n]
        grad += 2 * (T[:, :n].reshape(rows, k, n) * res[:, None, :]).sum(dim=(0, 2)) / n
    g_rev = p.grad.cpu().numpy()
    g_fwd = grad.cpu().numpy()
    assert np.max(np.abs(g_fwd - g_rev)) <= 1e-5 * np.max(np.abs(g_rev)), (g_fwd, g_rev)


def test_argument_checks():
    import torch
    L = tds_b200._lib.lib()
    dev = "cuda:0"
    sim, *_ = _case("cartpole", 8)
    ns = sim.n_stride
    rows, cols = sim.jacobian_dims(2)
    p = lambda a: ctypes.c_void_p(a.data_ptr()) if a is not None else None
    f32 = lambda d: torch.zeros((max(d, 1), ns), dtype=torch.float32, device=dev)
    q, qd, tau = f32(sim.n_q), f32(sim.n_qd), f32(sim.n_tau)
    t_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    t_out = torch.zeros((rows, ns), dtype=torch.float64, device=dev)
    t_par = torch.zeros((1, ns), dtype=torch.float64, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    dv = lambda mode, pd, a, b, c, m, ti, tp, to: L.tds_b200_step_jvp_device(sim._h, mode, pd, p(a), p(b), p(c), m, p(ti), p(tp), p(to), st)
    assert dv(3, 0, q, qd, tau, 1, t_in, None, t_out) == -2                  # mode WORLD
    assert dv(2, 1, q, qd, tau, 1, t_in, None, t_out) == -3                  # use_pd without set_env
    assert dv(2, 0, None, qd, tau, 1, t_in, None, t_out) == -1               # null q
    assert dv(2, 0, q, qd, tau, 1, t_in, None, None) == -1                   # null t_out
    assert dv(2, 0, q, qd, tau, 0, t_in, None, t_out) == -1                  # m < 1
    assert dv(2, 0, q, qd, tau, 1, None, None, t_out) == -1                  # both tangents null
    assert dv(2, 0, q, qd, tau, 1, t_in, t_par, t_out) == -4                 # parameter tangents without a set
    assert dv(2, 0, q, qd, tau, 1, t_in, None, t_out) == 0
    torch.cuda.synchronize()
    h = np.zeros((8, sim.n_q))
    hd = np.zeros((8, sim.n_qd))
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double)) if a is not None else None
    ti, to, tp = np.zeros((8, cols, 1)), np.zeros((8, rows, 1)), np.zeros((8, 1, 1))
    act = np.zeros((8, 1))
    hv = lambda mode, pd, m, a, b, c, t=None: L.tds_b200_step_jvp_host(sim._h, mode, pd, dp(h), dp(hd), dp(t), m, dp(a), dp(b), dp(c))
    assert hv(3, 0, 1, ti, None, to) == -2
    assert hv(2, 1, 1, ti, None, to) == -1                                    # use_pd needs the action
    assert hv(2, 1, 1, ti, None, to, act) == -3
    assert hv(2, 0, 0, ti, None, to) == -1
    assert hv(2, 0, 1, None, None, to) == -1
    assert hv(2, 0, 1, ti, tp, to) == -4
    w = wl.rigid_world("billiard", 4, seed=1)
    world = tds_b200.RigidWorld(w["bodies"], 4, **w["params"])
    nb, wns = world.n_bodies, world.n_stride
    s = torch.zeros((13 * nb, wns), dtype=torch.float64, device=dev)
    ts = torch.zeros((13 * nb, wns), dtype=torch.float64, device=dev)
    to_ = torch.zeros((13 * nb, wns), dtype=torch.float64, device=dev)
    rj = lambda m, a, b, so: L.tds_b200_rigid_jvp_device(world._h, p(s), None, 1, m, p(a), p(b), p(so), p(to_), None)
    assert rj(0, ts, None, None) == -1
    assert rj(1, None, None, None) == -1
    assert rj(1, ts, None, s) == -1                                           # state_out aliasing state
    assert rj(1, ts, None, None) == 0
    torch.cuda.synchronize()
