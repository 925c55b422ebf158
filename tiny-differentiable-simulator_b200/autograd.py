"""torch.autograd bindings of the batched step (reverse mode, DESIGN.md section 7.8).

    q1, qd1 = tds_b200.autograd.step(sim, q, qd, tau)          # [n_envs, dim] float32 CUDA tensors
    loss = ((q1 - target) ** 2).sum(); loss.backward()           # q.grad, qd.grad, tau.grad

The forward is the simulator's own step (BatchSim.step_device at its precision: Laikago keeps its fast mixed kernel).  The
backward is the vector-Jacobian product of the step at the saved inputs (BatchSim.step_vjp_device): the gradient of the fp64
world-frame step at the fp32-rounded inputs, and the gradient of the branch taken (contact set, clamps of the PD controller and
of the Gauss-Seidel sweep), as with any operator-overloading AD.  Gradients come back as float32.  The PD gains are simulator
settings, not autograd inputs; their cotangents are available from step_vjp_host / step_vjp_device.

With params (a float64 CUDA tensor [n_envs, k] of values for the physical parameters installed by BatchSim.set_physical_params,
DESIGN.md section 7.9) the forward installs those values and steps, and the backward also returns params.grad (float64): system
identification by gradient descent through rollouts.

rigid_step does the same for a batch of rigid-body worlds (RigidWorld) on float64 [n_worlds, n_bodies, 13] / [..., 3] tensors:
the reverse pass checkpoints the states of the rollout on the device and sweeps one step at a time.  Its params (float64 [n_worlds,
k], for the masses, shape sizes, friction and restitution installed by RigidWorld.set_physical_params, DESIGN.md section 7.11) get
their gradient summed over the rollout's steps.

Both functions also have forward-mode rules (DESIGN.md section 7.10), for torch.autograd.forward_ad dual tensors and torch.func.jvp:
the tangent of the outputs is the Jacobian-vector product of the same derivative (BatchSim.step_jvp_device, RigidWorld.step_jvp_device),
run with the parameter values of the same call.  Tangents of q, qd, tau_or_action and of the outputs are float32, those of params
float64; the PD gains have zero tangent.  rigid_step's forward mode runs the whole rollout in one launch.

mass_matrix(sim, q, params=None) is the joint-space mass matrix M(q) [n_envs, n_qd, n_qd] (float64, DESIGN.md section 7.12) with a
backward rule (BatchSim.mass_matrix_vjp_device: float32 q.grad, float64 params.grad) and a forward-mode rule
(BatchSim.mass_matrix_jvp_device).

inverse_dynamics(sim, q, qd, qdd=None, params=None) is tau = ID(q, qd, qdd) [n_envs, n_qd] (float64, DESIGN.md section 7.14) with a
backward rule (BatchSim.inverse_dynamics_vjp_device: float32 q.grad, qd.grad, qdd.grad, float64 params.grad) and a forward-mode rule
(BatchSim.inverse_dynamics_jvp_device).

step_contacts(sim, q, qd, tau_or_action=None, mode=MODE_FULL, use_pd=False, params=None) is the step that also reports its contacts
(DESIGN.md section 7.15): (q', qd', C) with C [n_envs, n_contact_points, 10] float32 (normal on b, point on b, distance, impulse on b),
on the world-frame kernel at the simulator's precision.  Its backward rule (BatchSim.step_contacts_vjp_device) takes cotangents of all
three outputs (float32 q.grad, qd.grad, tau_or_action.grad, float64 params.grad) and its forward-mode rule runs
BatchSim.step_contacts_jvp_device; both in MODE_FULL.  step itself is unchanged.

centroidal(sim, q, qd=None, params=None) is the body record, centroidal momentum matrix and its bias (DESIGN.md section 7.16): (m, c,
I_G, A, bias) float64, with a backward rule (BatchSim.centroidal_vjp_device: cotangents of all five outputs; float32 q.grad, qd.grad,
float64 params.grad) and a forward-mode rule (BatchSim.centroidal_jvp_device).

forward_kinematics(sim, q, links, local) is every link's world transform and every point's world position and linear Jacobian (float64,
DESIGN.md section 7.13) with a backward rule (BatchSim.kinematics_vjp_device: float32 q.grad) and a forward-mode rule
(BatchSim.kinematics_jvp_device).

point_motion(sim, q, qd, links, local, qdd=None) is every point's spatial Jacobian, velocity and acceleration J qdd + J' qd (float64,
DESIGN.md section 7.17) with a backward rule (BatchSim.point_motion_vjp_device: float32 q.grad, qd.grad, qdd.grad) and a forward-mode
rule (BatchSim.point_motion_jvp_device).

step_wrench(sim, q, qd, tau_or_action, links, local, W, mode=MODE_FULL, use_pd=False, params=None) is the step with a wrench [n; f] per
environment at every point of a point table (DESIGN.md section 7.18), on the world-frame kernel at the simulator's precision, with a
backward rule (BatchSim.step_wrench_vjp_device: float32 q.grad, qd.grad, tau_or_action.grad, W.grad, float64 params.grad) and a
forward-mode rule (BatchSim.step_wrench_jvp_device).

regressor(sim, q, qd=None, qdd=None) is the joint-torque regressor Y and the energy regressors yT, yV of the inertial parameters (float64,
DESIGN.md section 7.19) with a backward rule (BatchSim.regressor_vjp_device: float32 q.grad, qd.grad, qdd.grad) and a forward-mode rule
(BatchSim.regressor_jvp_device).

constrained_dynamics(sim, q, qd=None, tau=None, links=None, local=None, dims=3, damping=0.0, params=None) is the forward dynamics qdd with
the points of a table held in place and the constraint forces f (float64, DESIGN.md section 7.21), with a backward rule
(BatchSim.constrained_dynamics_vjp_device: float32 q.grad, qd.grad, tau.grad, float64 params.grad) and a forward-mode rule
(BatchSim.constrained_dynamics_jvp_device).

coriolis(sim, q, qd=None, params=None) is the Coriolis matrix C(q, qd) [n_envs, n_qd, n_qd] (float64, DESIGN.md section 7.22) with a
backward rule (BatchSim.coriolis_vjp_device: float32 q.grad, qd.grad, float64 params.grad) and a forward-mode rule
(BatchSim.coriolis_jvp_device).

inverse_dynamics_derivatives(sim, q, qd=None, qdd=None, params=None) is (d tau / dq, d tau / dqd) [n_envs, n_qd, n_qd] of the inverse
dynamics (float64, DESIGN.md section 7.23) with a backward rule (BatchSim.inverse_dynamics_derivatives_vjp_device: float32 q.grad, qd.grad,
qdd.grad, float64 params.grad) and a forward-mode rule (BatchSim.inverse_dynamics_derivatives_jvp_device).

forward_dynamics_derivatives(sim, q, qd=None, tau=None, params=None) is (qdd [n_envs, n_qd], d qdd / dq, d qdd / dqd, d qdd / dtau
[n_envs, n_qd, n_qd]) of the forward dynamics (float64, DESIGN.md section 7.24) with a backward rule
(BatchSim.forward_dynamics_derivatives_vjp_device: float32 q.grad, qd.grad, tau.grad, float64 params.grad) and a forward-mode rule
(BatchSim.forward_dynamics_derivatives_jvp_device).
"""
from collections import namedtuple

import numpy as np
import torch

from .sim import MODE_FD, MODE_FULL


def _soa(x, n_stride, dtype):
    """[n, dim] -> [max(dim, 1), n_stride] contiguous, padding environments zero."""
    n, dim = x.shape
    out = torch.zeros((max(dim, 1), n_stride), dtype=dtype, device=x.device)
    if dim:
        out[:dim, :n] = x.detach().to(dtype).t()
    return out


def _plain(t):
    """The tensor under torch.func's wrappers.  Under torch.func.jvp the forward-mode rules below receive the tangents wrapped for the
    transform's levels; they unwrap them and run with the transforms switched off (torch._C._DisableFuncTorch), so that the tensors
    handed to the C-ABI have storage."""
    from torch._C._functorch import get_unwrapped, is_functorch_wrapped_tensor
    while t is not None and is_functorch_wrapped_tensor(t):
        t = get_unwrapped(t)
    return t


def _check_params(sim, params):
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")


class _Step(torch.autograd.Function):
    @staticmethod
    def forward(sim, mode, use_pd, q, qd, tau, params):
        n, ns = sim.n_envs, sim.n_stride
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32)
        ts = None if tau is None else _soa(tau, ns, torch.float32)
        q_out, qd_out = torch.empty_like(qs), torch.empty_like(qds)
        qdd_out = torch.empty_like(qds) if mode == MODE_FD else None
        sim.step_device(mode, qs, qds, ts, q_out=q_out, qd_out=qd_out, qdd_out=qdd_out, use_pd=use_pd)
        if mode == MODE_FD:
            return qdd_out[:sim.n_qd, :n].t().contiguous()
        return q_out[:sim.n_q, :n].t().contiguous(), qd_out[:sim.n_qd, :n].t().contiguous()

    @staticmethod
    def setup_context(ctx, inputs, output):
        # (separate from forward so that torch.func transforms accept the Function; the SoA inputs are rebuilt here, the values
        # forward stepped)
        sim, mode, use_pd, q, qd, tau, params = inputs
        ns = sim.n_stride
        qs, qds = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32)
        ts = None if tau is None else _soa(tau, ns, torch.float32)
        ctx.sim, ctx.mode, ctx.use_pd, ctx.has_tau, ctx.has_params = sim, mode, use_pd, tau is not None, params is not None
        ctx.save_for_backward(qs, qds, ts if ts is not None else qs, params.detach() if params is not None else qs)
        ctx.jvp_inputs = (qs, qds, ts, params.detach() if params is not None else None)

    @staticmethod
    def backward(ctx, *grads):
        sim, mode = ctx.sim, ctx.mode
        qs, qds, ts, par = ctx.saved_tensors
        n, ns = sim.n_envs, sim.n_stride
        rows, cols = sim.jacobian_dims(mode, ctx.use_pd)
        dims = [sim.n_qd] if mode == MODE_FD else [sim.n_q, sim.n_qd]
        g_out = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        r = 0
        for g, d in zip(grads, dims):
            if g is not None:
                g_out[r:r + d, :n] = g.to(torch.float64).t()
            r += d
        g_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
        gp = None
        if ctx.has_params:
            # the values of this step (a later step of the graph may have installed others)
            sim.set_physical_params(sim.param_ids, par)
            g_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device)
            sim.step_vjp_params_device(mode, qs, qds, ts if ctx.has_tau else None, g_out, g_in, g_par, use_pd=ctx.use_pd)
            gp = g_par[:, :n].t().contiguous()
        else:
            sim.step_vjp_device(mode, qs, qds, ts if ctx.has_tau else None, g_out, g_in, use_pd=ctx.use_pd)
        gq = g_in[:sim.n_q, :n].t().to(torch.float32)
        gqd = g_in[sim.n_q:sim.n_q + sim.n_qd, :n].t().to(torch.float32)
        gt = None
        if ctx.has_tau:
            k0 = sim.n_q + sim.n_qd
            gt = g_in[k0:k0 + (sim.n_act if ctx.use_pd else sim.n_tau), :n].t().to(torch.float32)
        return None, None, None, gq, gqd, gt, gp

    @staticmethod
    def jvp(ctx, _sim, _mode, _use_pd, *tangents):
        with torch._C._DisableFuncTorch():
            return _Step._jvp(ctx, *(_plain(t) for t in tangents))

    @staticmethod
    def _jvp(ctx, tq, tqd, ttau, tpar):
        # forward mode: the m = 1 Jacobian-vector product of the fp64 world-frame step at the same inputs and parameter values
        sim, mode, use_pd = ctx.sim, ctx.mode, ctx.use_pd
        qs, qds, ts, par = (_plain(t) for t in ctx.jvp_inputs)
        n, ns = sim.n_envs, sim.n_stride
        rows, cols = sim.jacobian_dims(mode, use_pd)
        t_in = t_par = None
        if tq is not None or tqd is not None or (ttau is not None and ctx.has_tau):
            t_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
            k0 = sim.n_q + sim.n_qd
            for t, r0 in ((tq, 0), (tqd, sim.n_q), (ttau if ctx.has_tau else None, k0)):   # the PD gains: zero tangent
                if t is not None and t.shape[1]:
                    t_in[r0:r0 + t.shape[1], :n] = t.to(torch.float64).t()
        if tpar is not None and ctx.has_params:
            t_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device)
            t_par[:, :n] = tpar.to(torch.float64).t()
        t_out = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        if t_in is not None or t_par is not None:
            if ctx.has_params:
                sim.set_physical_params(sim.param_ids, par)   # the values of this step
            sim.step_jvp_device(mode, qs, qds, ts, 1, t_in, t_par, t_out, use_pd=use_pd)
        if mode == MODE_FD:
            return t_out[:sim.n_qd, :n].t().to(torch.float32).contiguous()
        return (t_out[:sim.n_q, :n].t().to(torch.float32).contiguous(),
                t_out[sim.n_q:sim.n_q + sim.n_qd, :n].t().to(torch.float32).contiguous())


def step(sim, q, qd, tau_or_action=None, mode=MODE_FULL, use_pd=False, params=None):
    """One differentiable step of every environment of `sim` (a BatchSim).  q [n_envs, n_q], qd [n_envs, n_qd], tau_or_action
    [n_envs, n_tau] (or [n_envs, n_act] with use_pd) float32 CUDA tensors.  Returns (q', qd'), or qdd in MODE_FD.  The gradient
    is that of the fp64 world-frame step at the fp32-rounded inputs, of the branch taken; see the module docstring.  params: None,
    or a float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also
    differentiated)."""
    for name, t in (("q", q), ("qd", qd), ("tau_or_action", tau_or_action)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or t.shape[0] != sim.n_envs):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, dim] is expected")
    _check_params(sim, params)
    return _Step.apply(sim, int(mode), bool(use_pd), q, qd, tau_or_action, params)


def _on_side_stream(dev, fn, tensors):
    """The rigid-world C-ABI reads a NULL stream as the world's own stream, and torch's default stream has the handle NULL: run
    fn(stream) on a side stream ordered after and before torch's current stream instead."""
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(cur)
    fn(side)
    cur.wait_stream(side)
    for t in tensors:
        if t is not None:
            t.record_stream(side)


class _RigidStep(torch.autograd.Function):
    @staticmethod
    def forward(world, steps, state, force, params):
        n, nb, ns = world.n_worlds, world.n_bodies, world.n_stride
        s = _soa(state.reshape(n, 13 * nb), ns, torch.float64)
        f = None if force is None else _soa(force.reshape(n, 3 * nb), ns, torch.float64)
        out = torch.empty_like(s)

        def run(st):
            if params is not None:
                world.set_physical_params(world.param_ids, params.detach(), stream=st)
            world.step_device(s, out, f, steps, stream=st)
        _on_side_stream(state.device, run, (s, out, f))
        return out[:, :n].t().reshape(n, nb, 13).contiguous()

    @staticmethod
    def setup_context(ctx, inputs, output):
        world, steps, state, force, params = inputs
        n, nb, ns = world.n_worlds, world.n_bodies, world.n_stride
        s = _soa(state.reshape(n, 13 * nb), ns, torch.float64)
        f = None if force is None else _soa(force.reshape(n, 3 * nb), ns, torch.float64)
        par = params.detach() if params is not None else None
        ctx.world, ctx.steps, ctx.has_force, ctx.has_params = world, steps, force is not None, params is not None
        ctx.save_for_backward(s, f if f is not None else s, par if par is not None else s)
        ctx.jvp_inputs = (s, f, par)

    @staticmethod
    def backward(ctx, g):
        world = ctx.world
        s, f, par = ctx.saved_tensors
        n, nb, ns = world.n_worlds, world.n_bodies, world.n_stride
        g_out = _soa(g.reshape(n, 13 * nb), ns, torch.float64)
        g_state = torch.zeros_like(g_out)
        g_force = torch.zeros((3 * nb, ns), dtype=torch.float64, device=g.device) if ctx.has_force else None
        fs = f if ctx.has_force else None
        g_par = None
        if ctx.has_params:
            g_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=g.device)

            def run(st):
                # the values of this call (a later call of the graph may have installed others)
                world.set_physical_params(world.param_ids, par, stream=st)
                world.step_vjp_params_device(s, fs, g_out, g_state, g_force, g_par, ctx.steps, stream=st)
        else:
            def run(st):
                world.step_vjp_device(s, fs, g_out, g_state, g_force, ctx.steps, stream=st)
        _on_side_stream(g.device, run, (s, f, g_out, g_state, g_force, g_par))
        gs = g_state[:, :n].t().reshape(n, nb, 13)
        gf = g_force[:, :n].t().reshape(n, nb, 3) if ctx.has_force else None
        gp = g_par[:, :n].t().contiguous() if ctx.has_params else None
        return None, None, gs, gf, gp

    @staticmethod
    def jvp(ctx, _world, _steps, t_state, t_force, t_params):
        with torch._C._DisableFuncTorch():
            return _RigidStep._jvp(ctx, _plain(t_state), _plain(t_force), _plain(t_params))

    @staticmethod
    def _jvp(ctx, t_state, t_force, t_params):
        # forward mode: the whole rollout in one launch of the tangent-seeded rigid kernel, with the parameter values of this call
        world = ctx.world
        s, f, par = (_plain(t) for t in ctx.jvp_inputs)
        n, nb, ns = world.n_worlds, world.n_bodies, world.n_stride
        ts = None if t_state is None else _soa(t_state.reshape(n, 13 * nb), ns, torch.float64)
        tf = None if t_force is None or not ctx.has_force else _soa(t_force.reshape(n, 3 * nb), ns, torch.float64)
        tp = None if t_params is None or not ctx.has_params else _soa(t_params, ns, torch.float64)
        t_out = torch.zeros_like(s)
        if ts is not None or tf is not None or tp is not None:
            def run(st):
                if ctx.has_params:
                    world.set_physical_params(world.param_ids, par, stream=st)
                world.step_jvp_device(s, f, 1, ts, tf, None, t_out, ctx.steps, stream=st, t_par=tp)
            _on_side_stream(s.device, run, (s, f, ts, tf, tp, t_out))
        return t_out[:, :n].t().reshape(n, nb, 13).contiguous()


def rigid_step(world, state, force=None, steps=1, params=None):
    """`steps` differentiable World::step calls of every world of `world` (a RigidWorld).  state [n_worlds, n_bodies, 13], force
    [n_worlds, n_bodies, 3] (applied before the first step) float64 CUDA tensors.  Returns the new state.  params: None, or a float64
    CUDA tensor [n_worlds, k] of values for the parameters installed by world.set_physical_params (then also differentiated; a [k]
    leaf expanded to [n_worlds, k] gets the gradient summed over the worlds)."""
    for name, t in (("state", state), ("force", force)):
        if t is not None and (t.dtype != torch.float64 or not t.is_cuda or t.shape[:2] != (world.n_worlds, world.n_bodies)):
            raise ValueError(f"{name}: a float64 CUDA tensor [n_worlds, n_bodies, dim] is expected")
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or not world.param_ids or
                               tuple(params.shape) != (world.n_worlds, len(world.param_ids))):
        raise ValueError("params: a float64 CUDA tensor [n_worlds, k] for the k parameters installed by set_physical_params is expected")
    return _RigidStep.apply(world, int(steps), state, force, params)


_In = namedtuple("_In", "q qd qdd params")   # a query's inputs, and their tangents or gradients, in _Query.apply's order

# What one dynamics query adds to _Query; p is the call's point table _Points, or None for a query without one:
#   rows(sim, p)                  row counts of the output buffers [rows, n_stride] (float64)
#   unpack(sim, p, *views)        views [n_envs, rows] of those buffers -> the outputs the user gets
#   pack(sim, p, *grads)          the outputs' cotangents -> the device's cotangent buffers, the inverse of unpack
#   value(sim, p, x, out, st)     the BatchSim value entry on the SoA inputs x (an _In; absent inputs None) and output buffers
#   jvp(sim, p, x, t, out, st)    the m = 1 JVP entry along the SoA tangents t (an _In; None: zero)
#   vjp(sim, p, x, G, g, st)      the VJP entry from the cotangent buffers G into the gradient buffers g (an _In; None: not computed)
# The three entries keep their own argument orders; st is the side stream they run on.
_QuerySpec = namedtuple("_QuerySpec", "rows unpack pack value jvp vjp")
_Points = namedtuple("_Points", "links local K")   # sim._points(links, local): int32 [K], float64 [K, 3], K


def _zeros(sim, rows, device):
    return torch.zeros((max(rows, 1), sim.n_stride), dtype=torch.float64, device=device)


def _cot(g, sim):
    """Cotangent [n_envs, ...] -> [rows, n_stride] float64."""
    return _soa(g.flatten(1), sim.n_stride, torch.float64)


def _check_state(sim, q, qd=None, qdd=None):
    for name, t, dim in (("q", q, "n_q"), ("qd", qd, "n_qd"), ("qdd", qdd, "n_qd")):
        if t is None and name != "q":
            continue
        if t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or tuple(t.shape) != (sim.n_envs, getattr(sim, dim)):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, {dim}] is expected")


def _state_soa(sim, q, qd, qdd):
    return [None if x is None else _soa(x, sim.n_stride, torch.float32) for x in (q, qd, qdd)]


class _Query(torch.autograd.Function):
    """The dynamics queries (mass_matrix, inverse_dynamics, centroidal, forward_kinematics, point_motion, regressor, mass_inverse,
    constrained_dynamics, coriolis, inverse_dynamics_derivatives, forward_dynamics_derivatives) as one Function over a _QuerySpec: the inputs in the SoA layout (float32 state, float64 tangents, environments padded with zeros to n_stride), zeroed
    float64 output buffers, every C-ABI call ordered on a side stream, and the gradients as float32 (q, qd, qdd) and float64 (params).
    An input the query does not take, or the call leaves out, is None and gets no gradient; a tangent on it is ignored.  With params
    the forward installs their values, and the backward and forward-mode rule reinstall the values of this call (a later call of the
    graph may have installed others)."""

    @staticmethod
    def forward(spec, sim, points, q, qd, qdd, params):
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        x = _state_soa(sim, q, qd, qdd)
        rows = spec.rows(sim, points)
        out = [_zeros(sim, r, q.device) for r in rows]
        _on_side_stream(q.device, lambda st: spec.value(sim, points, _In(*x, None), out, st), (*x, *out))
        return spec.unpack(sim, points, *(b[:r, :sim.n_envs].t() for b, r in zip(out, rows)))

    @staticmethod
    def setup_context(ctx, inputs, output):
        # (separate from forward so that torch.func transforms accept the Function; the SoA inputs are rebuilt here, the values
        # forward used)
        spec, sim, points, q, qd, qdd, params = inputs
        x = _In(*_state_soa(sim, q, qd, qdd), None if params is None else params.detach())
        ctx.spec, ctx.sim, ctx.points, ctx.has = spec, sim, points, [t is not None for t in x]
        ctx.save_for_backward(*(x.q if t is None else t for t in x))
        ctx.jvp_inputs = x

    @staticmethod
    def backward(ctx, *grads):
        spec, sim, p = ctx.spec, ctx.sim, ctx.points
        x = _In(*(t if has else None for t, has in zip(ctx.saved_tensors, ctx.has)))
        n, dev = sim.n_envs, x.q.device
        G = spec.pack(sim, p, *grads)
        dims = (sim.n_q, sim.n_qd, sim.n_qd, 0 if x.params is None else x.params.shape[1])
        g = _In(*(None if t is None else _zeros(sim, d, dev) for t, d in zip(x, dims)))
        if x.params is not None:
            sim.set_physical_params(sim.param_ids, x.params)
        _on_side_stream(dev, lambda st: spec.vjp(sim, p, x, G, g, st), (x.q, x.qd, x.qdd, *G, *g))
        dtypes = (torch.float32, torch.float32, torch.float32, torch.float64)
        return (None, None, None) + tuple(None if t is None else t[:d, :n].t().to(dt).contiguous() for t, d, dt in zip(g, dims, dtypes))

    @staticmethod
    def jvp(ctx, _spec, _sim, _points, *tangents):
        with torch._C._DisableFuncTorch():
            return _Query._jvp(ctx, *(_plain(t) for t in tangents))

    @staticmethod
    def _jvp(ctx, *tangents):
        spec, sim, p = ctx.spec, ctx.sim, ctx.points
        x = _In(*(_plain(t) for t in ctx.jvp_inputs))
        t = _In(*(None if v is None or xi is None else _soa(v, sim.n_stride, torch.float64) for v, xi in zip(tangents, x)))
        rows = spec.rows(sim, p)
        out = [_zeros(sim, r, x.q.device) for r in rows]
        if any(v is not None for v in t):
            if x.params is not None:
                sim.set_physical_params(sim.param_ids, x.params)
            _on_side_stream(x.q.device, lambda st: spec.jvp(sim, p, x, t, out, st), (x.q, x.qd, x.qdd, *t, *out))
        return spec.unpack(sim, p, *(b[:r, :sim.n_envs].t() for b, r in zip(out, rows)))


_MASS_MATRIX = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd * sim.n_qd],
    unpack=lambda sim, p, M: M.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous(),
    pack=lambda sim, p, gM: [_cot(gM, sim)],
    value=lambda sim, p, x, out, st: sim.mass_matrix_device(x.q, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.mass_matrix_jvp_device(x.q, 1, t.q, t.params, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.mass_matrix_vjp_device(x.q, *G, g.q, g.params, stream=st))


def mass_matrix(sim, q, params=None):
    """The joint-space mass matrix M(q) of every environment of `sim` (a BatchSim): [n_envs, n_qd, n_qd] float64, from q [n_envs, n_q]
    float32 CUDA tensor (fp64 CRBA at the fp32-rounded q).  params: None, or a float64 CUDA tensor [n_envs, k] of values for the
    parameters installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse and forward mode."""
    _check_state(sim, q)
    _check_params(sim, params)
    return _Query.apply(_MASS_MATRIX, sim, None, q, None, None, params)


_INVERSE_DYNAMICS = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd],
    unpack=lambda sim, p, tau: tau.contiguous(),
    pack=lambda sim, p, gtau: [_cot(gtau, sim)],
    value=lambda sim, p, x, out, st: sim.inverse_dynamics_device(x.q, x.qd, x.qdd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.inverse_dynamics_jvp_device(x.q, x.qd, x.qdd, 1, *t, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.inverse_dynamics_vjp_device(x.q, x.qd, x.qdd, *G, *g, stream=st))


def inverse_dynamics(sim, q, qd, qdd=None, params=None):
    """Inverse dynamics of every environment of `sim` (a BatchSim): tau [n_envs, n_qd] float64, the joint forces for which the
    multibodies have the accelerations qdd at (q, qd) under the simulator's gravity (DESIGN.md section 7.14), by the recursive
    Newton-Euler algorithm in fp64 at the fp32-rounded inputs.  q [n_envs, n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors; qd or
    qdd None: zero (the bias forces h(q, qd) are inverse_dynamics(sim, q, qd)).  Fixed base: the inverse of the MODE_FD step, stiffness
    and damping terms included.  Floating base: rows 0..5 are the wrench on the base in the base frame for the base-frame spatial
    acceleration qdd[0:6], with gravity rotated into the base frame - the textbook RNEA in the coordinates of mass_matrix, not the
    inverse of the reference's floating-base forward dynamics.  params: None, or a float64 CUDA tensor [n_envs, k] of values for the
    parameters installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse and forward mode."""
    _check_state(sim, q, qd, qdd)
    _check_params(sim, params)
    return _Query.apply(_INVERSE_DYNAMICS, sim, None, q, qd, qdd, params)


_SYM = [0, 1, 2, 1, 3, 4, 2, 4, 5]   # [3, 3] from the components xx, xy, xz, yy, yz, zz


def _fold_sym(g):
    """Cotangent [n, 3, 3] of a symmetric matrix read by _SYM -> [n, 6]: an off-diagonal component collects both of its entries."""
    g = g.flatten(1)
    return torch.stack([g[:, 0], g[:, 1] + g[:, 3], g[:, 2] + g[:, 6], g[:, 4], g[:, 5] + g[:, 7], g[:, 8]], dim=1)


# the com record [10, n_stride]: m, c, I_G xx xy xz yy yz zz
_CENTROIDAL = _QuerySpec(
    rows=lambda sim, p: [10, 6 * sim.n_qd, 6],
    unpack=lambda sim, p, com, A, bias: (com[:, 0].contiguous(), com[:, 1:4].contiguous(),
                                         com[:, 4:10][:, _SYM].reshape(sim.n_envs, 3, 3).contiguous(),
                                         A.reshape(sim.n_envs, 6, sim.n_qd).contiguous(), bias.contiguous()),
    pack=lambda sim, p, gm, gc, gI, gA, gbias: [_cot(torch.cat([gm[:, None], gc, _fold_sym(gI)], dim=1), sim), _cot(gA, sim),
                                                _cot(gbias, sim)],
    value=lambda sim, p, x, out, st: sim.centroidal_device(x.q, x.qd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.centroidal_jvp_device(x.q, x.qd, 1, t.q, t.qd, t.params, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.centroidal_vjp_device(x.q, x.qd, *G, g.q, g.qd, g.params, stream=st))


def centroidal(sim, q, qd=None, params=None):
    """The centroidal quantities of every environment of `sim` (a BatchSim), DESIGN.md section 7.16, in fp64 at the fp32-rounded inputs:
    (m [n_envs], c [n_envs, 3], I_G [n_envs, 3, 3], A [n_envs, 6, n_qd], bias [n_envs, 6]) float64 - the total mass of the links and a
    floating base, their centre of mass in world coordinates, the rotational inertia about it in world axes, the centroidal momentum
    matrix (h_G = A qd, rows [angular about c; linear] in world axes, columns in the coordinates of mass_matrix) and its bias A' qd (the
    rate of h_G at qdd = 0, without gravity).  q [n_envs, n_q], qd [n_envs, n_qd] float32 CUDA tensors (qd None: zero).  params: None, or
    a float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also differentiated).
    Differentiable in reverse and forward mode."""
    _check_state(sim, q, qd)
    _check_params(sim, params)
    return _Query.apply(_CENTROIDAL, sim, None, q, qd, None, params)


# xf [12 n_links, n_stride]: per link R row-major | p.  Without points (K = 0) the entries get None for x and J and their cotangents.
_KINEMATICS = _QuerySpec(
    rows=lambda sim, p: [12 * sim.n_links, 3 * p.K, 3 * p.K * sim.n_qd],
    unpack=lambda sim, p, xf, x, J: (xf.reshape(sim.n_envs, sim.n_links, 4, 3)[:, :, :3].contiguous(),
                                     xf.reshape(sim.n_envs, sim.n_links, 4, 3)[:, :, 3].contiguous(),
                                     x.reshape(sim.n_envs, p.K, 3).contiguous(), J.reshape(sim.n_envs, p.K, 3, sim.n_qd).contiguous()),
    pack=lambda sim, p, gR, gp, gx, gJ: [_cot(torch.cat([gR, gp[:, :, None]], dim=2), sim), _cot(gx, sim) if p.K else None,
                                         _cot(gJ, sim) if p.K and sim.n_qd else None],
    value=lambda sim, p, x, out, st: sim.kinematics_device(x.q, p.links, p.local, out[0], *(out[1:] if p.K else (None, None)), stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.kinematics_jvp_device(x.q, p.links, p.local, 1, t.q, out[0], *(out[1:] if p.K else (None, None)),
                                                                stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.kinematics_vjp_device(x.q, p.links, p.local, *G, g.q, stream=st))


def forward_kinematics(sim, q, links, local):
    """Forward kinematics and linear point Jacobians of every environment of `sim` (a BatchSim) at q [n_envs, n_q] float32 CUDA tensor
    (fp64 at the fp32-rounded q), for the point table links [K] (-1: the base) / local [K, 3] (coordinates in the link's frame; both
    constants of the call): (R [n_envs, n_links, 3, 3], p [n_envs, n_links, 3], x [n_envs, K, 3], J [n_envs, K, 3, n_qd]), float64 world
    coordinates.  Differentiable along q in reverse mode (float32 q.grad from the cotangents of all four outputs) and forward mode."""
    _check_state(sim, q)
    return _Query.apply(_KINEMATICS, sim, _Points(*sim._points(links, local)), q, None, None, None)


_POINT_MOTION = _QuerySpec(
    rows=lambda sim, p: [6 * p.K * sim.n_qd, 6 * p.K, 6 * p.K],
    unpack=lambda sim, p, J, vel, acc: (J.reshape(sim.n_envs, p.K, 6, sim.n_qd).contiguous(), vel.reshape(sim.n_envs, p.K, 6).contiguous(),
                                        acc.reshape(sim.n_envs, p.K, 6).contiguous()),
    pack=lambda sim, p, gJ, gvel, gacc: [_cot(gJ, sim), _cot(gvel, sim), _cot(gacc, sim)],
    value=lambda sim, p, x, out, st: sim.point_motion_device(x.q, x.qd, x.qdd, p.links, p.local, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.point_motion_jvp_device(x.q, x.qd, x.qdd, p.links, p.local, 1, t.q, t.qd, t.qdd, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.point_motion_vjp_device(x.q, x.qd, x.qdd, p.links, p.local, *G, g.q, g.qd, g.qdd, stream=st))


def point_motion(sim, q, qd, links, local, qdd=None):
    """Spatial point Jacobians, point velocities and accelerations of every environment of `sim` (a BatchSim), DESIGN.md section 7.17,
    in fp64 at the fp32-rounded inputs, for the point table links [K] (-1: the base) / local [K, 3] (coordinates in the link's frame; both
    constants of the call): (J [n_envs, K, 6, n_qd], vel [n_envs, K, 6], acc [n_envs, K, 6]) float64, world axes, rows [w; x'] (the
    angular velocity of the point's link and the velocity of the point's world position), vel = J qd and acc = [w'; x''] = J qdd + J' qd
    (the drift J' qd when qdd is None).  Columns in the coordinates of mass_matrix and inverse_dynamics: a floating base's qd[0:6] is the
    base-frame twist, so J composes with M, h and A (its base columns differ from forward_kinematics' J, which ignores the base
    rotation).  q [n_envs, n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors (qd or qdd None: zero).  Gravity and installed physical
    parameters do not enter.  Differentiable along q, qd and qdd in reverse mode (float32 gradients from the cotangents of all three
    outputs) and forward mode."""
    _check_state(sim, q, qd, qdd)
    return _Query.apply(_POINT_MOTION, sim, _Points(*sim._points(links, local)), q, qd, qdd, None)


class _StepContacts(torch.autograd.Function):
    @staticmethod
    def forward(sim, mode, use_pd, q, qd, tau, params):
        n, ns, npts = sim.n_envs, sim.n_stride, sim.n_contact_points
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), None if tau is None else _soa(tau, ns, torch.float32)
        q_out, qd_out = torch.empty_like(qs), torch.empty_like(qds)
        C = torch.zeros((max(10 * npts, 1), ns), dtype=torch.float32, device=q.device)
        _on_side_stream(q.device, lambda st: sim.step_contacts_device(mode, qs, qds, ts, q_out, qd_out, C, use_pd=use_pd, stream=st),
                        (qs, qds, ts, q_out, qd_out, C))
        return (q_out[:sim.n_q, :n].t().contiguous(), qd_out[:sim.n_qd, :n].t().contiguous(),
                C[:10 * npts, :n].t().reshape(n, npts, 10).contiguous())

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, mode, use_pd, q, qd, tau, params = inputs
        ns = sim.n_stride
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), None if tau is None else _soa(tau, ns, torch.float32)
        par = params.detach() if params is not None else None
        ctx.sim, ctx.mode, ctx.use_pd, ctx.has_tau, ctx.has_params = sim, mode, use_pd, tau is not None, params is not None
        ctx.save_for_backward(qs, qds, ts if ts is not None else qs, par if par is not None else qs)
        ctx.jvp_inputs = (qs, qds, ts, par)

    @staticmethod
    def backward(ctx, gq_out, gqd_out, gC):
        sim, mode, use_pd = ctx.sim, ctx.mode, ctx.use_pd
        qs, qds, ts, par = ctx.saved_tensors
        ts = ts if ctx.has_tau else None
        n, ns, nq, nd, npts = sim.n_envs, sim.n_stride, sim.n_q, sim.n_qd, sim.n_contact_points
        rows, cols = sim.contact_rows(mode, use_pd)
        G = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        for g, r0, d in ((gq_out, 0, nq), (gqd_out, nq, nd), (None if gC is None else gC.reshape(n, 10 * npts), nq + nd, 10 * npts)):
            if g is not None and d:
                G[r0:r0 + d, :n] = g.to(torch.float64).t()
        g_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
        g_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device) if ctx.has_params else None
        if ctx.has_params:
            sim.set_physical_params(sim.param_ids, par)   # the values of this call
        _on_side_stream(qs.device, lambda st: sim.step_contacts_vjp_device(mode, qs, qds, ts, G, g_in, g_par, use_pd=use_pd, stream=st),
                        (qs, qds, ts, G, g_in, g_par))
        gt = None
        if ctx.has_tau:
            k0 = nq + nd
            gt = g_in[k0:k0 + (sim.n_act if use_pd else sim.n_tau), :n].t().to(torch.float32).contiguous()
        gp = g_par[:, :n].t().contiguous() if ctx.has_params else None
        return (None, None, None, g_in[:nq, :n].t().to(torch.float32).contiguous(), g_in[nq:nq + nd, :n].t().to(torch.float32).contiguous(),
                gt, gp)

    @staticmethod
    def jvp(ctx, _sim, _mode, _use_pd, *tangents):
        with torch._C._DisableFuncTorch():
            return _StepContacts._jvp(ctx, *(_plain(t) for t in tangents))

    @staticmethod
    def _jvp(ctx, tq, tqd, ttau, tpar):
        sim, mode, use_pd = ctx.sim, ctx.mode, ctx.use_pd
        qs, qds, ts, par = (_plain(t) for t in ctx.jvp_inputs)
        n, ns, nq, nd, npts = sim.n_envs, sim.n_stride, sim.n_q, sim.n_qd, sim.n_contact_points
        rows, cols = sim.contact_rows(mode, use_pd)
        t_in = t_par = None
        if tq is not None or tqd is not None or (ttau is not None and ctx.has_tau):
            t_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
            for t, r0 in ((tq, 0), (tqd, nq), (ttau if ctx.has_tau else None, nq + nd)):   # the PD gains: zero tangent
                if t is not None and t.shape[1]:
                    t_in[r0:r0 + t.shape[1], :n] = t.to(torch.float64).t()
        if tpar is not None and ctx.has_params:
            t_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device)
            t_par[:, :n] = tpar.to(torch.float64).t()
        t_out = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        if t_in is not None or t_par is not None:
            if ctx.has_params:
                sim.set_physical_params(sim.param_ids, par)   # the values of this call
            _on_side_stream(qs.device, lambda st: sim.step_contacts_jvp_device(mode, qs, qds, ts, 1, t_in, t_par, t_out, use_pd=use_pd,
                                                                               stream=st), (qs, qds, ts, t_in, t_par, t_out))
        out = lambda r0, d: t_out[r0:r0 + d, :n].t().to(torch.float32).contiguous()
        return out(0, nq), out(nq, nd), out(nq + nd, 10 * npts).reshape(n, npts, 10)


def step_contacts(sim, q, qd, tau_or_action=None, mode=MODE_FULL, use_pd=False, params=None):
    """One differentiable step of every environment of `sim` (a BatchSim) that also reports its contacts: (q' [n_envs, n_q], qd'
    [n_envs, n_qd], C [n_envs, n_contact_points, 10]) float32, a record per contact candidate - normal on b [3], point on b [3],
    distance, impulse on body b [3] in N s - in world coordinates (DESIGN.md section 7.15).  The step runs on the world-frame kernel at
    the simulator's precision (mode MODE_FULL or MODE_WORLD); q' and qd' are those of that kernel's step.  Inputs as for step.  The
    derivatives (MODE_FULL) are those of the fp64 world-frame step at the fp32-rounded inputs, of the branch taken (contact set,
    clamps of the Gauss-Seidel sweep), with cotangents or tangents of all three outputs."""
    for name, t in (("q", q), ("qd", qd), ("tau_or_action", tau_or_action)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or t.shape[0] != sim.n_envs):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, dim] is expected")
    _check_params(sim, params)
    return _StepContacts.apply(sim, int(mode), bool(use_pd), q, qd, tau_or_action, params)


class _StepWrench(torch.autograd.Function):
    @staticmethod
    def forward(sim, mode, use_pd, links, local, q, qd, tau, W, params):
        n, ns = sim.n_envs, sim.n_stride
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), None if tau is None else _soa(tau, ns, torch.float32)
        Ws = _soa(W.reshape(n, -1), ns, torch.float32)
        fd = mode == MODE_FD
        q_out = None if fd else torch.empty_like(qs)
        qd_out = None if fd else torch.empty_like(qds)
        qdd_out = torch.empty_like(qds) if fd else None
        _on_side_stream(q.device, lambda st: sim.step_wrench_device(mode, qs, qds, ts, links, local, Ws, q_out, qd_out, qdd_out, use_pd=use_pd,
                                                                    stream=st), (qs, qds, ts, Ws, q_out, qd_out, qdd_out))
        if fd:
            return qdd_out[:sim.n_qd, :n].t().contiguous()
        return q_out[:sim.n_q, :n].t().contiguous(), qd_out[:sim.n_qd, :n].t().contiguous()

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, mode, use_pd, links, local, q, qd, tau, W, params = inputs
        ns = sim.n_stride
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), None if tau is None else _soa(tau, ns, torch.float32)
        Ws = _soa(W.reshape(sim.n_envs, -1), ns, torch.float32)
        par = params.detach() if params is not None else None
        ctx.sim, ctx.mode, ctx.use_pd, ctx.links, ctx.local = sim, mode, use_pd, links, local
        ctx.has_tau, ctx.has_params, ctx.K = tau is not None, params is not None, len(links)
        ctx.save_for_backward(qs, qds, ts if ts is not None else qs, Ws, par if par is not None else qs)
        ctx.jvp_inputs = (qs, qds, ts, Ws, par)

    @staticmethod
    def backward(ctx, *grads):
        sim, mode, use_pd, K = ctx.sim, ctx.mode, ctx.use_pd, ctx.K
        qs, qds, ts, Ws, par = ctx.saved_tensors
        ts = ts if ctx.has_tau else None
        n, ns, nq, nd = sim.n_envs, sim.n_stride, sim.n_q, sim.n_qd
        rows, cols = sim.jacobian_dims(mode, use_pd)
        dims = [(0, nd)] if mode == MODE_FD else [(0, nq), (nq, nd)]
        G = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        for g, (r0, d) in zip(grads, dims):
            if g is not None and d:
                G[r0:r0 + d, :n] = g.to(torch.float64).t()
        g_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
        g_W = torch.zeros((max(6 * K, 1), ns), dtype=torch.float64, device=qs.device)
        g_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device) if ctx.has_params else None
        if ctx.has_params:
            sim.set_physical_params(sim.param_ids, par)   # the values of this call
        _on_side_stream(qs.device, lambda st: sim.step_wrench_vjp_device(mode, qs, qds, ts, ctx.links, ctx.local, Ws, G, g_in, g_W, g_par,
                                                                         use_pd=use_pd, stream=st), (qs, qds, ts, Ws, G, g_in, g_W, g_par))
        gt = None
        if ctx.has_tau:
            k0 = nq + nd
            gt = g_in[k0:k0 + (sim.n_act if use_pd else sim.n_tau), :n].t().to(torch.float32).contiguous()
        gW = g_W[:6 * K, :n].t().to(torch.float32).reshape(n, K, 6).contiguous()
        gp = g_par[:, :n].t().contiguous() if ctx.has_params else None
        return (None, None, None, None, None, g_in[:nq, :n].t().to(torch.float32).contiguous(),
                g_in[nq:nq + nd, :n].t().to(torch.float32).contiguous(), gt, gW, gp)

    @staticmethod
    def jvp(ctx, _sim, _mode, _use_pd, _links, _local, *tangents):
        with torch._C._DisableFuncTorch():
            return _StepWrench._jvp(ctx, *(_plain(t) for t in tangents))

    @staticmethod
    def _jvp(ctx, tq, tqd, ttau, tW, tpar):
        sim, mode, use_pd, K = ctx.sim, ctx.mode, ctx.use_pd, ctx.K
        qs, qds, ts, Ws, par = (_plain(t) for t in ctx.jvp_inputs)
        n, ns, nq, nd = sim.n_envs, sim.n_stride, sim.n_q, sim.n_qd
        rows, cols = sim.jacobian_dims(mode, use_pd)
        t_in = t_W = t_par = None
        if tq is not None or tqd is not None or (ttau is not None and ctx.has_tau):
            t_in = torch.zeros((cols, ns), dtype=torch.float64, device=qs.device)
            for t, r0 in ((tq, 0), (tqd, nq), (ttau if ctx.has_tau else None, nq + nd)):   # the PD gains: zero tangent
                if t is not None and t.shape[1]:
                    t_in[r0:r0 + t.shape[1], :n] = t.to(torch.float64).t()
        if tW is not None and K:
            t_W = _soa(tW.reshape(n, 6 * K), ns, torch.float64)
        if tpar is not None and ctx.has_params:
            t_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=qs.device)
            t_par[:, :n] = tpar.to(torch.float64).t()
        t_out = torch.zeros((rows, ns), dtype=torch.float64, device=qs.device)
        if t_in is not None or t_W is not None or t_par is not None:
            if ctx.has_params:
                sim.set_physical_params(sim.param_ids, par)   # the values of this call
            _on_side_stream(qs.device, lambda st: sim.step_wrench_jvp_device(mode, qs, qds, ts, ctx.links, ctx.local, Ws, 1, t_in, t_W, t_par,
                                                                             t_out, use_pd=use_pd, stream=st),
                            (qs, qds, ts, Ws, t_in, t_W, t_par, t_out))
        out = lambda r0, d: t_out[r0:r0 + d, :n].t().to(torch.float32).contiguous()
        if mode == MODE_FD:
            return out(0, nd)
        return out(0, nq), out(nq, nd)


def step_wrench(sim, q, qd, tau_or_action, links, local, W, mode=MODE_FULL, use_pd=False, params=None):
    """One differentiable step of every environment of `sim` (a BatchSim) with external wrenches (DESIGN.md section 7.18): W float32 CUDA
    tensor [n_envs, K, 6], W[e, k] = [n; f] in world axes at point k of the table links [K] (-1: the base) / local [K, 3] (the force acts
    along a line through the point, n is a pure moment).  Returns (q', qd'), or qdd in MODE_FD, float32.  The step runs on the world-frame
    kernel at the simulator's precision; other inputs as for step.  The derivatives are those of the fp64 world-frame step at the
    fp32-rounded inputs, of the branch taken, along q, qd, tau_or_action, W and params (backward rule BatchSim.step_wrench_vjp_device,
    forward-mode rule BatchSim.step_wrench_jvp_device)."""
    for name, t in (("q", q), ("qd", qd), ("tau_or_action", tau_or_action)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or t.shape[0] != sim.n_envs):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, dim] is expected")
    lk = tuple(int(x) for x in torch.as_tensor(links).reshape(-1).tolist())
    lc = tuple(tuple(float(v) for v in row) for row in torch.as_tensor(local, dtype=torch.float64).reshape(-1, 3).tolist())
    if len(lc) != len(lk):
        raise ValueError("links [K] and local [K, 3] expected")
    if W.dtype != torch.float32 or not W.is_cuda or tuple(W.shape) != (sim.n_envs, len(lk), 6):
        raise ValueError("W: a float32 CUDA tensor [n_envs, K, 6] is expected")
    _check_params(sim, params)
    return _StepWrench.apply(sim, int(mode), bool(use_pd), lk, lc, q, qd, tau_or_action, W, params)


_REGRESSOR = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd * sim.n_pi, sim.n_pi, sim.n_pi],
    unpack=lambda sim, p, Y, yT, yV: (Y.reshape(sim.n_envs, sim.n_qd, sim.n_pi).contiguous(), yT.contiguous(), yV.contiguous()),
    pack=lambda sim, p, gY, gT, gV: [_cot(gY, sim), _cot(gT, sim), _cot(gV, sim)],
    value=lambda sim, p, x, out, st: sim.regressor_device(x.q, x.qd, x.qdd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.regressor_jvp_device(x.q, x.qd, x.qdd, 1, t.q, t.qd, t.qdd, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.regressor_vjp_device(x.q, x.qd, x.qdd, *G, g.q, g.qd, g.qdd, stream=st))


def regressor(sim, q, qd=None, qdd=None):
    """The regressors of the inertial parameters of every environment of `sim` (a BatchSim), DESIGN.md section 7.19, in fp64 at the
    fp32-rounded inputs: (Y [n_envs, n_qd, n_pi], yT [n_envs, n_pi], yV [n_envs, n_pi]) float64 with inverse_dynamics(sim, q, qd, qdd) =
    Y @ pi, the kinetic energy 1/2 qd^T M qd = yT . pi and the potential energy yV . pi, for pi of tds_b200.model.inertial_parameters
    (per body: mass, first moment m c and inertia about the body-frame origin; per joint: stiffness and damping; column names from
    tds_b200.model.regressor_names).  q [n_envs, n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors (qd or qdd None: zero).  Installed
    physical parameters do not enter.  Differentiable along q, qd and qdd in reverse mode (float32 gradients from the cotangents of all
    three outputs) and forward mode."""
    _check_state(sim, q, qd, qdd)
    return _Query.apply(_REGRESSOR, sim, None, q, qd, qdd, None)


# Without points (K = 0) the entries get None for Linv and its cotangent, and the Function's Linv is [n_envs, 0, 0].
_MASS_INVERSE = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd * sim.n_qd, 36 * p.K * p.K],
    unpack=lambda sim, p, Minv, Linv: (Minv.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous(),
                                       Linv.reshape(sim.n_envs, 6 * p.K, 6 * p.K).contiguous()),
    pack=lambda sim, p, gMinv, gLinv: [_cot(gMinv, sim), _cot(gLinv, sim) if p.K else None],
    value=lambda sim, p, x, out, st: sim.mass_inverse_device(x.q, p.links, p.local, out[0], out[1] if p.K else None, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.mass_inverse_jvp_device(x.q, p.links, p.local, 1, t.q, t.params, out[0], out[1] if p.K else None,
                                                                  stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.mass_inverse_vjp_device(x.q, p.links, p.local, *G, g.q, g.params, stream=st))


def mass_inverse(sim, q, links=None, local=None, params=None):
    """The inverse mass matrix and the operational-space inverse inertia of every environment of `sim` (a BatchSim), DESIGN.md section
    7.20, in fp64 at the fp32-rounded q [n_envs, n_q] float32 CUDA tensor: (Minv [n_envs, n_qd, n_qd], Linv [n_envs, 6K, 6K] or None
    without points) float64.  Minv is the inverse of mass_matrix(sim, q, params), bitwise symmetric (for a floating base it is not the
    forward dynamics' dqdd/dtau); Linv = J Minv J^T for the point table links [K] (-1: the base) / local [K, 3] (K <= 16; constants of
    the call), J the spatial point Jacobian of point_motion ([n_envs, K, 6, n_qd] as 6K rows), so that Lambda = Linv^-1 (rank-deficient
    where a point's chain has fewer than 6 dofs: the caller chooses how to invert it).  A solve with M is Minv @ b.  params: None, or a
    float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also differentiated).
    Differentiable in reverse mode (float32 q.grad, float64 params.grad) and forward mode."""
    _check_state(sim, q)
    _check_params(sim, params)
    p = _Points(*sim._points([] if links is None else links, np.zeros((0, 3)) if local is None else local))
    Minv, Linv = _Query.apply(_MASS_INVERSE, sim, p, q, None, None, params)
    return Minv, (Linv if p.K else None)


_CdPoints = namedtuple("_CdPoints", "links local K dims damping")   # the point table of _Points with the constraint's dims and damping

# tau rides in the qdd slot (n_qd float32, as qdd).  Without points (K = 0) the entries get None for f and its cotangent, and the
# Function's f is [n_envs, 0, dims].
_CONSTRAINED_DYNAMICS = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd, p.dims * p.K],
    unpack=lambda sim, p, qdd, f: (qdd.contiguous(), f.reshape(sim.n_envs, p.K, p.dims).contiguous()),
    pack=lambda sim, p, gqdd, gf: [_cot(gqdd, sim), _cot(gf, sim) if p.K else None],
    value=lambda sim, p, x, out, st: sim.constrained_dynamics_device(x.q, x.qd, x.qdd, p.links, p.local, p.dims, p.damping, out[0],
                                                                     out[1] if p.K else None, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.constrained_dynamics_jvp_device(x.q, x.qd, x.qdd, p.links, p.local, p.dims, p.damping, 1, t.q,
                                                                         t.qd, t.qdd, t.params, out[0], out[1] if p.K else None,
                                                                         stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.constrained_dynamics_vjp_device(x.q, x.qd, x.qdd, p.links, p.local, p.dims, p.damping, *G, g.q,
                                                                       g.qd, g.qdd, g.params, stream=st))


def constrained_dynamics(sim, q, qd=None, tau=None, links=None, local=None, dims=3, damping=0.0, params=None):
    """The point-constrained forward dynamics of every environment of `sim` (a BatchSim), DESIGN.md section 7.21, in fp64 at the
    fp32-rounded q [n_envs, n_q], qd and tau [n_envs, n_qd] float32 CUDA tensors (qd or tau None: zero; a floating base's tau[0:6] is a
    wrench on the base in the base frame, as for inverse_dynamics): (qdd [n_envs, n_qd], f [n_envs, K, dims] or None without points)
    float64 with M qdd - J_c^T f = tau - h and J_c qdd = -d_c - damping f, for M = mass_matrix(sim, q, params), h = inverse_dynamics(sim,
    q, qd, params=params) and J, d = point_motion(sim, q, qd, links, local)'s J and acc, J_c and d_c their rows held by the constraint:
    the 3 linear rows of each point (dims 3, a point contact that neither slips nor lifts off) or all 6 (dims 6, a welded frame).  f is the
    force (or wrench [n; f]) the constraint applies to the robot at each point, in world axes, as step_wrench's W.  The point table links
    [K] (-1: the base) / local [K, 3] (K <= 16), dims and damping >= 0 are constants of the call; K = 0 is the unconstrained forward
    dynamics M^-1 (tau - h).  An environment whose J_c M^-1 J_c^T + damping I has a pivot <= 0 gets NaN outputs.  params: None, or a
    float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also differentiated).
    Differentiable in reverse mode (float32 q.grad, qd.grad, tau.grad, float64 params.grad) and forward mode."""
    _check_state(sim, q, qd)
    if tau is not None and (tau.dtype != torch.float32 or not tau.is_cuda or tuple(tau.shape) != (sim.n_envs, sim.n_qd)):
        raise ValueError("tau: a float32 CUDA tensor [n_envs, n_qd] is expected")
    _check_params(sim, params)
    if dims not in (3, 6):
        raise ValueError("dims: 3 (the points' linear rows) or 6 (all six rows) is expected")
    p = _CdPoints(*sim._points([] if links is None else links, np.zeros((0, 3)) if local is None else local), int(dims), float(damping))
    qdd, f = _Query.apply(_CONSTRAINED_DYNAMICS, sim, p, q, qd, tau, params)
    return qdd, (f if p.K else None)


_CORIOLIS = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd * sim.n_qd],
    unpack=lambda sim, p, C: C.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous(),
    pack=lambda sim, p, gC: [_cot(gC, sim)],
    value=lambda sim, p, x, out, st: sim.coriolis_device(x.q, x.qd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.coriolis_jvp_device(x.q, x.qd, 1, t.q, t.qd, t.params, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.coriolis_vjp_device(x.q, x.qd, *G, g.q, g.qd, g.params, stream=st))


def coriolis(sim, q, qd=None, params=None):
    """The Coriolis matrix C(q, qd) of every environment of `sim` (a BatchSim), DESIGN.md section 7.22: [n_envs, n_qd, n_qd] float64 in
    the coordinates of mass_matrix, in fp64 at the fp32-rounded q [n_envs, n_q] and qd [n_envs, n_qd] float32 CUDA tensors (qd None:
    zero, C = 0).  C is Echeandia & Wensing's factorisation, so C qd is the velocity part of the bias forces (inverse_dynamics(sim, q, qd)
    - inverse_dynamics(sim, q) without joint damping) and C + C^T is the time derivative of M along qd (M' - 2 C is skew-symmetric).
    params: None, or a float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also
    differentiated).  Differentiable in reverse mode (float32 q.grad, qd.grad, float64 params.grad) and forward mode."""
    _check_state(sim, q, qd)
    _check_params(sim, params)
    return _Query.apply(_CORIOLIS, sim, None, q, qd, None, params)


_INVERSE_DYNAMICS_DERIVATIVES = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd * sim.n_qd, sim.n_qd * sim.n_qd],
    unpack=lambda sim, p, a, b: (a.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous(), b.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous()),
    pack=lambda sim, p, ga, gb: [_cot(ga, sim), _cot(gb, sim)],
    value=lambda sim, p, x, out, st: sim.inverse_dynamics_derivatives_device(x.q, x.qd, x.qdd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.inverse_dynamics_derivatives_jvp_device(x.q, x.qd, x.qdd, 1, *t, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.inverse_dynamics_derivatives_vjp_device(x.q, x.qd, x.qdd, *G, *g, stream=st))


def inverse_dynamics_derivatives(sim, q, qd=None, qdd=None, params=None):
    """The derivatives (d tau / dq, d tau / dqd) of inverse_dynamics(sim, q, qd, qdd, params) for every environment of `sim` (a
    BatchSim), DESIGN.md section 7.23: two [n_envs, n_qd, n_qd] float64 tensors, row r = tau_r, in fp64 at the fp32-rounded q [n_envs,
    n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors (qd or qdd None: zero).  The columns are in the coordinates of mass_matrix: column
    k of d tau / dq is the derivative along the motion with velocity e_k (include/tds_b200.h), so the matrices compose with M, C and the
    point Jacobians; d tau / dqdd is mass_matrix(sim, q).  params: None, or a float64 CUDA tensor [n_envs, k] of values for the parameters
    installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse mode (float32 q.grad, qd.grad, qdd.grad,
    float64 params.grad: second-order terms) and forward mode."""
    _check_state(sim, q, qd, qdd)
    _check_params(sim, params)
    return _Query.apply(_INVERSE_DYNAMICS_DERIVATIVES, sim, None, q, qd, qdd, params)


def _square(sim, x):
    return x.reshape(sim.n_envs, sim.n_qd, sim.n_qd).contiguous()


_FORWARD_DYNAMICS_DERIVATIVES = _QuerySpec(
    rows=lambda sim, p: [sim.n_qd] + [sim.n_qd * sim.n_qd] * 3,
    unpack=lambda sim, p, qdd, a, b, c: (qdd.contiguous(), _square(sim, a), _square(sim, b), _square(sim, c)),
    pack=lambda sim, p, *G: [_cot(g, sim) for g in G],
    value=lambda sim, p, x, out, st: sim.forward_dynamics_derivatives_device(x.q, x.qd, x.qdd, *out, stream=st),
    jvp=lambda sim, p, x, t, out, st: sim.forward_dynamics_derivatives_jvp_device(x.q, x.qd, x.qdd, 1, *t, *out, stream=st),
    vjp=lambda sim, p, x, G, g, st: sim.forward_dynamics_derivatives_vjp_device(x.q, x.qd, x.qdd, *G, *g, stream=st))


def forward_dynamics_derivatives(sim, q, qd=None, tau=None, params=None):
    """The forward dynamics qdd = M^-1 (tau - h) and its derivatives (d qdd / dq, d qdd / dqd, d qdd / dtau) for every environment of
    `sim` (a BatchSim), DESIGN.md section 7.24: qdd [n_envs, n_qd] and three [n_envs, n_qd, n_qd] float64 tensors, row r = qdd_r, in fp64
    at the fp32-rounded q [n_envs, n_q], qd and tau [n_envs, n_qd] float32 CUDA tensors (qd or tau None: zero).  qdd is
    constrained_dynamics(sim, q, qd, tau)'s, d qdd / dtau is mass_inverse(sim, q)'s M^-1, and d qdd / dq = -M^-1 d tau / dq, d qdd / dqd =
    -M^-1 d tau / dqd with the inverse dynamics' derivatives at that qdd in fp64.  The columns are in the coordinates of mass_matrix: column
    k of d qdd / dq is the derivative along the motion with velocity e_k (include/tds_b200.h).  A floating base's tau rows 0..5 are the
    base wrench in the base frame (this qdd is not the MODE_FD step's there).  params: None, or a float64 CUDA tensor [n_envs, k] of values
    for the parameters installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse mode (float32 q.grad,
    qd.grad, tau.grad, float64 params.grad: second-order terms) and forward mode."""
    _check_state(sim, q, qd)
    if tau is not None and (tau.dtype != torch.float32 or not tau.is_cuda or tuple(tau.shape) != (sim.n_envs, sim.n_qd)):
        raise ValueError("tau: a float32 CUDA tensor [n_envs, n_qd] is expected")
    _check_params(sim, params)
    return _Query.apply(_FORWARD_DYNAMICS_DERIVATIVES, sim, None, q, qd, tau, params)
