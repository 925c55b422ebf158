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
"""
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
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
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


class _MassMatrix(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, params):
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs = _soa(q, ns, torch.float32)
        M = torch.zeros((max(nd * nd, 1), ns), dtype=torch.float64, device=q.device)
        _on_side_stream(q.device, lambda st: sim.mass_matrix_device(qs, M, stream=st), (qs, M))
        return M[:nd * nd, :n].t().reshape(n, nd, nd).contiguous()

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, params = inputs
        qs = _soa(q, sim.n_stride, torch.float32)
        par = params.detach() if params is not None else None
        ctx.sim, ctx.has_params = sim, params is not None
        ctx.save_for_backward(qs, par if par is not None else qs)
        ctx.jvp_inputs = (qs, par)

    @staticmethod
    def backward(ctx, g):
        sim = ctx.sim
        qs, par = ctx.saved_tensors
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        G = _soa(g.reshape(n, nd * nd), ns, torch.float64)
        g_q = torch.zeros((max(sim.n_q, 1), ns), dtype=torch.float64, device=g.device)
        g_par = torch.zeros((par.shape[1], ns), dtype=torch.float64, device=g.device) if ctx.has_params else None
        if ctx.has_params:
            sim.set_physical_params(sim.param_ids, par)   # the values of this call
        _on_side_stream(g.device, lambda st: sim.mass_matrix_vjp_device(qs, G, g_q, g_par, stream=st), (qs, G, g_q, g_par))
        gq = g_q[:sim.n_q, :n].t().to(torch.float32)
        gp = g_par[:, :n].t().contiguous() if ctx.has_params else None
        return None, gq, gp

    @staticmethod
    def jvp(ctx, _sim, t_q, t_params):
        with torch._C._DisableFuncTorch():
            return _MassMatrix._jvp(ctx, _plain(t_q), _plain(t_params))

    @staticmethod
    def _jvp(ctx, t_q, t_params):
        sim = ctx.sim
        qs, par = (_plain(t) for t in ctx.jvp_inputs)
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        tq = None if t_q is None else _soa(t_q, ns, torch.float64)
        tp = None if t_params is None or not ctx.has_params else _soa(t_params, ns, torch.float64)
        t_M = torch.zeros((max(nd * nd, 1), ns), dtype=torch.float64, device=qs.device)
        if tq is not None or tp is not None:
            if ctx.has_params:
                sim.set_physical_params(sim.param_ids, par)   # the values of this call
            _on_side_stream(qs.device, lambda st: sim.mass_matrix_jvp_device(qs, 1, tq, tp, t_M, stream=st), (qs, tq, tp, t_M))
        return t_M[:nd * nd, :n].t().reshape(n, nd, nd).contiguous()


def mass_matrix(sim, q, params=None):
    """The joint-space mass matrix M(q) of every environment of `sim` (a BatchSim): [n_envs, n_qd, n_qd] float64, from q [n_envs, n_q]
    float32 CUDA tensor (fp64 CRBA at the fp32-rounded q).  params: None, or a float64 CUDA tensor [n_envs, k] of values for the
    parameters installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse and forward mode."""
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
    return _MassMatrix.apply(sim, q, params)


class _InverseDynamics(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, qd, qdd, params):
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        tau = torch.zeros((max(nd, 1), ns), dtype=torch.float64, device=q.device)
        _on_side_stream(q.device, lambda st: sim.inverse_dynamics_device(qs, qds, qdds, tau, stream=st), (qs, qds, qdds, tau))
        return tau[:nd, :n].t().contiguous()

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, qd, qdd, params = inputs
        ns = sim.n_stride
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        par = params.detach() if params is not None else None
        ctx.sim, ctx.has = sim, (qd is not None, qdd is not None, params is not None)
        ctx.save_for_backward(qs, *(t if t is not None else qs for t in (qds, qdds, par)))
        ctx.jvp_inputs = (qs, qds, qdds, par)

    @staticmethod
    def backward(ctx, g):
        sim = ctx.sim
        has_qd, has_qdd, has_par = ctx.has
        qs, qds, qdds, par = ctx.saved_tensors
        qds, qdds = (qds if has_qd else None), (qdds if has_qdd else None)
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        G = _soa(g, ns, torch.float64)
        z = lambda rows: torch.zeros((max(rows, 1), ns), dtype=torch.float64, device=g.device)
        g_q, g_qd, g_qdd = z(sim.n_q), (z(nd) if has_qd else None), (z(nd) if has_qdd else None)
        g_par = z(par.shape[1]) if has_par else None
        if has_par:
            sim.set_physical_params(sim.param_ids, par)   # the values of this call
        _on_side_stream(g.device, lambda st: sim.inverse_dynamics_vjp_device(qs, qds, qdds, G, g_q, g_qd, g_qdd, g_par, stream=st),
                        (qs, qds, qdds, G, g_q, g_qd, g_qdd, g_par))
        out = lambda t, rows, dt: None if t is None else t[:rows, :n].t().to(dt).contiguous()
        return None, out(g_q, sim.n_q, torch.float32), out(g_qd, nd, torch.float32), out(g_qdd, nd, torch.float32), \
            out(g_par, par.shape[1], torch.float64)

    @staticmethod
    def jvp(ctx, _sim, t_q, t_qd, t_qdd, t_params):
        with torch._C._DisableFuncTorch():
            return _InverseDynamics._jvp(ctx, _plain(t_q), _plain(t_qd), _plain(t_qdd), _plain(t_params))

    @staticmethod
    def _jvp(ctx, t_q, t_qd, t_qdd, t_params):
        sim = ctx.sim
        has_qd, has_qdd, has_par = ctx.has
        qs, qds, qdds, par = (_plain(t) for t in ctx.jvp_inputs)
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        tq = _soa_opt(t_q, ns, torch.float64)
        tqd = _soa_opt(t_qd if has_qd else None, ns, torch.float64)
        tqdd = _soa_opt(t_qdd if has_qdd else None, ns, torch.float64)
        tp = _soa_opt(t_params if has_par else None, ns, torch.float64)
        t_tau = torch.zeros((max(nd, 1), ns), dtype=torch.float64, device=qs.device)
        if any(t is not None for t in (tq, tqd, tqdd, tp)):
            if has_par:
                sim.set_physical_params(sim.param_ids, par)   # the values of this call
            _on_side_stream(qs.device, lambda st: sim.inverse_dynamics_jvp_device(qs, qds, qdds, 1, tq, tqd, tqdd, tp, t_tau, stream=st),
                            (qs, qds, qdds, tq, tqd, tqdd, tp, t_tau))
        return t_tau[:nd, :n].t().contiguous()


def _soa_opt(x, n_stride, dtype):
    return None if x is None else _soa(x, n_stride, dtype)


def inverse_dynamics(sim, q, qd, qdd=None, params=None):
    """Inverse dynamics of every environment of `sim` (a BatchSim): tau [n_envs, n_qd] float64, the joint forces for which the
    multibodies have the accelerations qdd at (q, qd) under the simulator's gravity (DESIGN.md section 7.14), by the recursive
    Newton-Euler algorithm in fp64 at the fp32-rounded inputs.  q [n_envs, n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors; qd or
    qdd None: zero (the bias forces h(q, qd) are inverse_dynamics(sim, q, qd)).  Fixed base: the inverse of the MODE_FD step, stiffness
    and damping terms included.  Floating base: rows 0..5 are the wrench on the base in the base frame for the base-frame spatial
    acceleration qdd[0:6], with gravity rotated into the base frame - the textbook RNEA in the coordinates of mass_matrix, not the
    inverse of the reference's floating-base forward dynamics.  params: None, or a float64 CUDA tensor [n_envs, k] of values for the
    parameters installed by sim.set_physical_params (then also differentiated).  Differentiable in reverse and forward mode."""
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    for name, t in (("qd", qd), ("qdd", qdd)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or tuple(t.shape) != (sim.n_envs, sim.n_qd)):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, n_qd] is expected")
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
    return _InverseDynamics.apply(sim, q, qd, qdd, params)


_SYM = [0, 1, 2, 1, 3, 4, 2, 4, 5]   # [3, 3] from the components xx, xy, xz, yy, yz, zz


def _cen_outputs(sim, com, A, bias):
    """Device outputs [rows, n_stride] of the centroidal entries -> (m [n], c [n, 3], I_G [n, 3, 3], A [n, 6, n_qd], bias [n, 6])."""
    n, nd = sim.n_envs, sim.n_qd
    com = com[:, :n].t()
    return (com[:, 0].contiguous(), com[:, 1:4].contiguous(), com[:, 4:10][:, _SYM].reshape(n, 3, 3).contiguous(),
            A[:6 * nd, :n].t().reshape(n, 6, nd).contiguous(), bias[:, :n].t().contiguous())


def _cen_buffers(sim, device):
    z = lambda rows: torch.zeros((max(rows, 1), sim.n_stride), dtype=torch.float64, device=device)
    return z(10), z(6 * sim.n_qd), z(6)


class _Centroidal(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, qd, params):
        ns = sim.n_stride
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32)
        com, A, bias = _cen_buffers(sim, q.device)
        _on_side_stream(q.device, lambda st: sim.centroidal_device(qs, qds, com, A, bias, stream=st), (qs, qds, com, A, bias))
        return _cen_outputs(sim, com, A, bias)

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, qd, params = inputs
        ns = sim.n_stride
        qs, qds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32)
        par = params.detach() if params is not None else None
        ctx.sim, ctx.has = sim, (qd is not None, params is not None)
        ctx.save_for_backward(qs, *(t if t is not None else qs for t in (qds, par)))
        ctx.jvp_inputs = (qs, qds, par)

    @staticmethod
    def backward(ctx, g_m, g_c, g_I, g_A, g_bias):
        sim = ctx.sim
        has_qd, has_par = ctx.has
        qs, qds, par = ctx.saved_tensors
        qds = qds if has_qd else None
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        # I_G's symmetric entries are read from the six components: an off-diagonal component collects both of its entries
        gI = g_I.reshape(n, 9).to(torch.float64)
        gIc = torch.stack([gI[:, 0], gI[:, 1] + gI[:, 3], gI[:, 2] + gI[:, 6], gI[:, 4], gI[:, 5] + gI[:, 7], gI[:, 8]], dim=1)
        G_com = _soa(torch.cat([g_m.reshape(n, 1).to(torch.float64), g_c.to(torch.float64), gIc], dim=1), ns, torch.float64)
        G_A = _soa(g_A.reshape(n, 6 * nd), ns, torch.float64)
        G_bias = _soa(g_bias, ns, torch.float64)
        z = lambda rows: torch.zeros((max(rows, 1), ns), dtype=torch.float64, device=qs.device)
        g_q, g_qd = z(sim.n_q), (z(nd) if has_qd else None)
        g_par = z(par.shape[1]) if has_par else None
        if has_par:
            sim.set_physical_params(sim.param_ids, par)   # the values of this call
        _on_side_stream(qs.device, lambda st: sim.centroidal_vjp_device(qs, qds, G_com, G_A, G_bias, g_q, g_qd, g_par, stream=st),
                        (qs, qds, G_com, G_A, G_bias, g_q, g_qd, g_par))
        out = lambda t, rows, dt: None if t is None else t[:rows, :n].t().to(dt).contiguous()
        return None, out(g_q, sim.n_q, torch.float32), out(g_qd, nd, torch.float32), out(g_par, par.shape[1], torch.float64)

    @staticmethod
    def jvp(ctx, _sim, t_q, t_qd, t_params):
        with torch._C._DisableFuncTorch():
            return _Centroidal._jvp(ctx, _plain(t_q), _plain(t_qd), _plain(t_params))

    @staticmethod
    def _jvp(ctx, t_q, t_qd, t_params):
        sim = ctx.sim
        has_qd, has_par = ctx.has
        qs, qds, par = (_plain(t) for t in ctx.jvp_inputs)
        ns = sim.n_stride
        tq = _soa_opt(t_q, ns, torch.float64)
        tqd = _soa_opt(t_qd if has_qd else None, ns, torch.float64)
        tp = _soa_opt(t_params if has_par else None, ns, torch.float64)
        t_com, t_A, t_bias = _cen_buffers(sim, qs.device)
        if any(t is not None for t in (tq, tqd, tp)):
            if has_par:
                sim.set_physical_params(sim.param_ids, par)   # the values of this call
            _on_side_stream(qs.device, lambda st: sim.centroidal_jvp_device(qs, qds, 1, tq, tqd, tp, t_com, t_A, t_bias, stream=st),
                            (qs, qds, tq, tqd, tp, t_com, t_A, t_bias))
        return _cen_outputs(sim, t_com, t_A, t_bias)


def centroidal(sim, q, qd=None, params=None):
    """The centroidal quantities of every environment of `sim` (a BatchSim), DESIGN.md section 7.16, in fp64 at the fp32-rounded inputs:
    (m [n_envs], c [n_envs, 3], I_G [n_envs, 3, 3], A [n_envs, 6, n_qd], bias [n_envs, 6]) float64 - the total mass of the links and a
    floating base, their centre of mass in world coordinates, the rotational inertia about it in world axes, the centroidal momentum
    matrix (h_G = A qd, rows [angular about c; linear] in world axes, columns in the coordinates of mass_matrix) and its bias A' qd (the
    rate of h_G at qdd = 0, without gravity).  q [n_envs, n_q], qd [n_envs, n_qd] float32 CUDA tensors (qd None: zero).  params: None, or
    a float64 CUDA tensor [n_envs, k] of values for the parameters installed by sim.set_physical_params (then also differentiated).
    Differentiable in reverse and forward mode."""
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    if qd is not None and (qd.dtype != torch.float32 or not qd.is_cuda or qd.dim() != 2 or tuple(qd.shape) != (sim.n_envs, sim.n_qd)):
        raise ValueError("qd: a float32 CUDA tensor [n_envs, n_qd] is expected")
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
    return _Centroidal.apply(sim, q, qd, params)


def _kin_outputs(sim, K, xf, x, J):
    """Device outputs [rows, n_stride] of the kinematics entries -> (R [n, n_links, 3, 3], p [n, n_links, 3], x [n, K, 3],
    J [n, K, 3, n_qd])."""
    n, nl, nd = sim.n_envs, sim.n_links, sim.n_qd
    xf = xf[:nl * 12, :n].t().reshape(n, nl, 12)
    return (xf[..., :9].reshape(n, nl, 3, 3).contiguous(), xf[..., 9:].contiguous(), x[:3 * K, :n].t().reshape(n, K, 3).contiguous(),
            J[:3 * K * nd, :n].t().reshape(n, K, 3, nd).contiguous())


def _kin_buffers(sim, K, device):
    ns, nl, nd = sim.n_stride, sim.n_links, sim.n_qd
    z = dict(dtype=torch.float64, device=device)
    return torch.zeros((max(nl * 12, 1), ns), **z), torch.zeros((max(3 * K, 1), ns), **z), torch.zeros((max(3 * K * nd, 1), ns), **z)


class _ForwardKinematics(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, links, local):
        lk, lc, K = sim._points(links, local)
        qs = _soa(q, sim.n_stride, torch.float32)
        xf, x, J = _kin_buffers(sim, K, q.device)
        xo, Jo = (x, J) if K else (None, None)
        _on_side_stream(q.device, lambda st: sim.kinematics_device(qs, lk, lc, xf, xo, Jo, stream=st), (qs, xf, x, J))
        return _kin_outputs(sim, K, xf, x, J)

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, links, local = inputs
        lk, lc, K = sim._points(links, local)
        qs = _soa(q, sim.n_stride, torch.float32)
        ctx.sim, ctx.points = sim, (lk, lc, K)
        ctx.save_for_backward(qs)
        ctx.jvp_q = qs

    @staticmethod
    def backward(ctx, gR, gp, gx, gJ):
        sim = ctx.sim
        (qs,) = ctx.saved_tensors
        lk, lc, K = ctx.points
        n, ns, nl, nd = sim.n_envs, sim.n_stride, sim.n_links, sim.n_qd
        dev = qs.device

        def zero_if_none(g, shape):
            return torch.zeros(shape, dtype=torch.float64, device=dev) if g is None else g.to(torch.float64)
        gxf = torch.cat([zero_if_none(gR, (n, nl, 3, 3)).reshape(n, nl, 9), zero_if_none(gp, (n, nl, 3))], dim=2).reshape(n, nl * 12)
        G_xf = _soa(gxf, ns, torch.float64)
        G_x = _soa(zero_if_none(gx, (n, K, 3)).reshape(n, 3 * K), ns, torch.float64) if K else None
        G_J = _soa(zero_if_none(gJ, (n, K, 3, nd)).reshape(n, 3 * K * nd), ns, torch.float64) if K and nd else None
        g_q = torch.zeros((max(sim.n_q, 1), ns), dtype=torch.float64, device=dev)
        _on_side_stream(dev, lambda st: sim.kinematics_vjp_device(qs, lk, lc, G_xf, G_x, G_J, g_q, stream=st), (qs, G_xf, G_x, G_J, g_q))
        return None, g_q[:sim.n_q, :n].t().to(torch.float32), None, None

    @staticmethod
    def jvp(ctx, _sim, t_q, _links, _local):
        with torch._C._DisableFuncTorch():
            return _ForwardKinematics._jvp(ctx, _plain(t_q))

    @staticmethod
    def _jvp(ctx, t_q):
        sim = ctx.sim
        qs = _plain(ctx.jvp_q)
        lk, lc, K = ctx.points
        t_xf, t_x, t_J = _kin_buffers(sim, K, qs.device)
        if t_q is not None:
            tq = _soa(t_q, sim.n_stride, torch.float64)
            xo, Jo = (t_x, t_J) if K else (None, None)
            _on_side_stream(qs.device, lambda st: sim.kinematics_jvp_device(qs, lk, lc, 1, tq, t_xf, xo, Jo, stream=st), (qs, tq, t_xf, t_x, t_J))
        return _kin_outputs(sim, K, t_xf, t_x, t_J)


def forward_kinematics(sim, q, links, local):
    """Forward kinematics and linear point Jacobians of every environment of `sim` (a BatchSim) at q [n_envs, n_q] float32 CUDA tensor
    (fp64 at the fp32-rounded q), for the point table links [K] (-1: the base) / local [K, 3] (coordinates in the link's frame; both
    constants of the call): (R [n_envs, n_links, 3, 3], p [n_envs, n_links, 3], x [n_envs, K, 3], J [n_envs, K, 3, n_qd]), float64 world
    coordinates.  Differentiable along q in reverse mode (float32 q.grad from the cotangents of all four outputs) and forward mode."""
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    return _ForwardKinematics.apply(sim, q, links, local)


def _mot_outputs(sim, K, J, vel, acc):
    """Device outputs [rows, n_stride] of the point-motion entries -> (J [n, K, 6, n_qd], vel [n, K, 6], acc [n, K, 6])."""
    n, nd = sim.n_envs, sim.n_qd
    return (J[:6 * K * nd, :n].t().reshape(n, K, 6, nd).contiguous(), vel[:6 * K, :n].t().reshape(n, K, 6).contiguous(),
            acc[:6 * K, :n].t().reshape(n, K, 6).contiguous())


def _mot_buffers(sim, K, device):
    z = lambda rows: torch.zeros((max(rows, 1), sim.n_stride), dtype=torch.float64, device=device)
    return z(6 * K * sim.n_qd), z(6 * K), z(6 * K)


class _PointMotion(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, qd, qdd, links, local):
        lk, lc, K = sim._points(links, local)
        ns = sim.n_stride
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        J, vel, acc = _mot_buffers(sim, K, q.device)
        _on_side_stream(q.device, lambda st: sim.point_motion_device(qs, qds, qdds, lk, lc, J, vel, acc, stream=st), (qs, qds, qdds, J, vel, acc))
        return _mot_outputs(sim, K, J, vel, acc)

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, qd, qdd, links, local = inputs
        ns = sim.n_stride
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        ctx.sim, ctx.points, ctx.has = sim, sim._points(links, local), (qd is not None, qdd is not None)
        ctx.save_for_backward(qs, *(t if t is not None else qs for t in (qds, qdds)))
        ctx.jvp_inputs = (qs, qds, qdds)

    @staticmethod
    def backward(ctx, gJ, gvel, gacc):
        sim = ctx.sim
        has_qd, has_qdd = ctx.has
        qs, qds, qdds = ctx.saved_tensors
        qds, qdds = (qds if has_qd else None), (qdds if has_qdd else None)
        lk, lc, K = ctx.points
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        dev = qs.device

        def cot(g, rows):
            return _soa(torch.zeros((n, rows), dtype=torch.float64, device=dev) if g is None else g.reshape(n, rows), ns, torch.float64)
        G_J, G_vel, G_acc = cot(gJ, 6 * K * nd), cot(gvel, 6 * K), cot(gacc, 6 * K)
        z = lambda rows: torch.zeros((max(rows, 1), ns), dtype=torch.float64, device=dev)
        g_q, g_qd, g_qdd = z(sim.n_q), (z(nd) if has_qd else None), (z(nd) if has_qdd else None)
        _on_side_stream(dev, lambda st: sim.point_motion_vjp_device(qs, qds, qdds, lk, lc, G_J, G_vel, G_acc, g_q, g_qd, g_qdd, stream=st),
                        (qs, qds, qdds, G_J, G_vel, G_acc, g_q, g_qd, g_qdd))
        out = lambda t, rows: None if t is None else t[:rows, :n].t().to(torch.float32).contiguous()
        return None, out(g_q, sim.n_q), out(g_qd, nd), out(g_qdd, nd), None, None

    @staticmethod
    def jvp(ctx, _sim, t_q, t_qd, t_qdd, _links, _local):
        with torch._C._DisableFuncTorch():
            return _PointMotion._jvp(ctx, _plain(t_q), _plain(t_qd), _plain(t_qdd))

    @staticmethod
    def _jvp(ctx, t_q, t_qd, t_qdd):
        sim = ctx.sim
        has_qd, has_qdd = ctx.has
        qs, qds, qdds = (_plain(t) for t in ctx.jvp_inputs)
        lk, lc, K = ctx.points
        ns = sim.n_stride
        tq = _soa_opt(t_q, ns, torch.float64)
        tqd = _soa_opt(t_qd if has_qd else None, ns, torch.float64)
        tqdd = _soa_opt(t_qdd if has_qdd else None, ns, torch.float64)
        t_J, t_vel, t_acc = _mot_buffers(sim, K, qs.device)
        if any(t is not None for t in (tq, tqd, tqdd)):
            _on_side_stream(qs.device, lambda st: sim.point_motion_jvp_device(qs, qds, qdds, lk, lc, 1, tq, tqd, tqdd, t_J, t_vel, t_acc,
                                                                              stream=st), (qs, qds, qdds, tq, tqd, tqdd, t_J, t_vel, t_acc))
        return _mot_outputs(sim, K, t_J, t_vel, t_acc)


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
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    for name, t in (("qd", qd), ("qdd", qdd)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or tuple(t.shape) != (sim.n_envs, sim.n_qd)):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, n_qd] is expected")
    return _PointMotion.apply(sim, q, qd, qdd, links, local)


class _StepContacts(torch.autograd.Function):
    @staticmethod
    def forward(sim, mode, use_pd, q, qd, tau, params):
        n, ns, npts = sim.n_envs, sim.n_stride, sim.n_contact_points
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), _soa_opt(tau, ns, torch.float32)
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
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), _soa_opt(tau, ns, torch.float32)
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
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
    return _StepContacts.apply(sim, int(mode), bool(use_pd), q, qd, tau_or_action, params)


class _StepWrench(torch.autograd.Function):
    @staticmethod
    def forward(sim, mode, use_pd, links, local, q, qd, tau, W, params):
        n, ns = sim.n_envs, sim.n_stride
        if params is not None:
            sim.set_physical_params(sim.param_ids, params.detach())
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), _soa_opt(tau, ns, torch.float32)
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
        qs, qds, ts = _soa(q, ns, torch.float32), _soa(qd, ns, torch.float32), _soa_opt(tau, ns, torch.float32)
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
    if params is not None and (params.dtype != torch.float64 or not params.is_cuda or
                               tuple(params.shape) != (sim.n_envs, len(sim.param_ids)) or not sim.param_ids):
        raise ValueError("params: a float64 CUDA tensor [n_envs, k] for the k parameters installed by set_physical_params is expected")
    return _StepWrench.apply(sim, int(mode), bool(use_pd), lk, lc, q, qd, tau_or_action, W, params)


def _reg_outputs(sim, Y, yT, yV):
    """Device outputs [rows, n_stride] of the regressors -> (Y [n, n_qd, n_pi], yT [n, n_pi], yV [n, n_pi])."""
    n, nd, npi = sim.n_envs, sim.n_qd, sim.n_pi
    return (Y[:nd * npi, :n].t().reshape(n, nd, npi).contiguous(), yT[:npi, :n].t().contiguous(), yV[:npi, :n].t().contiguous())


def _reg_buffers(sim, device):
    z = lambda rows: torch.zeros((max(rows, 1), sim.n_stride), dtype=torch.float64, device=device)
    return z(sim.n_qd * sim.n_pi), z(sim.n_pi), z(sim.n_pi)


class _Regressor(torch.autograd.Function):
    @staticmethod
    def forward(sim, q, qd, qdd):
        ns = sim.n_stride
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        Y, yT, yV = _reg_buffers(sim, q.device)
        _on_side_stream(q.device, lambda st: sim.regressor_device(qs, qds, qdds, Y, yT, yV, stream=st), (qs, qds, qdds, Y, yT, yV))
        return _reg_outputs(sim, Y, yT, yV)

    @staticmethod
    def setup_context(ctx, inputs, output):
        sim, q, qd, qdd = inputs
        ns = sim.n_stride
        qs, qds, qdds = _soa(q, ns, torch.float32), _soa_opt(qd, ns, torch.float32), _soa_opt(qdd, ns, torch.float32)
        ctx.sim, ctx.has = sim, (qd is not None, qdd is not None)
        ctx.save_for_backward(qs, *(t if t is not None else qs for t in (qds, qdds)))
        ctx.jvp_inputs = (qs, qds, qdds)

    @staticmethod
    def backward(ctx, gY, gT, gV):
        sim = ctx.sim
        has_qd, has_qdd = ctx.has
        qs, qds, qdds = ctx.saved_tensors
        qds, qdds = (qds if has_qd else None), (qdds if has_qdd else None)
        n, ns, nd = sim.n_envs, sim.n_stride, sim.n_qd
        dev = qs.device

        def cot(g, rows):
            return _soa(torch.zeros((n, rows), dtype=torch.float64, device=dev) if g is None else g.reshape(n, rows), ns, torch.float64)
        G_Y, G_yT, G_yV = cot(gY, nd * sim.n_pi), cot(gT, sim.n_pi), cot(gV, sim.n_pi)
        z = lambda rows: torch.zeros((max(rows, 1), ns), dtype=torch.float64, device=dev)
        g_q, g_qd, g_qdd = z(sim.n_q), (z(nd) if has_qd else None), (z(nd) if has_qdd else None)
        _on_side_stream(dev, lambda st: sim.regressor_vjp_device(qs, qds, qdds, G_Y, G_yT, G_yV, g_q, g_qd, g_qdd, stream=st),
                        (qs, qds, qdds, G_Y, G_yT, G_yV, g_q, g_qd, g_qdd))
        out = lambda t, rows: None if t is None else t[:rows, :n].t().to(torch.float32).contiguous()
        return None, out(g_q, sim.n_q), out(g_qd, nd), out(g_qdd, nd)

    @staticmethod
    def jvp(ctx, _sim, t_q, t_qd, t_qdd):
        with torch._C._DisableFuncTorch():
            return _Regressor._jvp(ctx, _plain(t_q), _plain(t_qd), _plain(t_qdd))

    @staticmethod
    def _jvp(ctx, t_q, t_qd, t_qdd):
        sim = ctx.sim
        has_qd, has_qdd = ctx.has
        qs, qds, qdds = (_plain(t) for t in ctx.jvp_inputs)
        ns = sim.n_stride
        tq = _soa_opt(t_q, ns, torch.float64)
        tqd = _soa_opt(t_qd if has_qd else None, ns, torch.float64)
        tqdd = _soa_opt(t_qdd if has_qdd else None, ns, torch.float64)
        t_Y, t_yT, t_yV = _reg_buffers(sim, qs.device)
        if any(t is not None for t in (tq, tqd, tqdd)):
            _on_side_stream(qs.device, lambda st: sim.regressor_jvp_device(qs, qds, qdds, 1, tq, tqd, tqdd, t_Y, t_yT, t_yV, stream=st),
                            (qs, qds, qdds, tq, tqd, tqdd, t_Y, t_yT, t_yV))
        return _reg_outputs(sim, t_Y, t_yT, t_yV)


def regressor(sim, q, qd=None, qdd=None):
    """The regressors of the inertial parameters of every environment of `sim` (a BatchSim), DESIGN.md section 7.19, in fp64 at the
    fp32-rounded inputs: (Y [n_envs, n_qd, n_pi], yT [n_envs, n_pi], yV [n_envs, n_pi]) float64 with inverse_dynamics(sim, q, qd, qdd) =
    Y @ pi, the kinetic energy 1/2 qd^T M qd = yT . pi and the potential energy yV . pi, for pi of tds_b200.model.inertial_parameters
    (per body: mass, first moment m c and inertia about the body-frame origin; per joint: stiffness and damping; column names from
    tds_b200.model.regressor_names).  q [n_envs, n_q], qd and qdd [n_envs, n_qd] float32 CUDA tensors (qd or qdd None: zero).  Installed
    physical parameters do not enter.  Differentiable along q, qd and qdd in reverse mode (float32 gradients from the cotangents of all
    three outputs) and forward mode."""
    if q.dtype != torch.float32 or not q.is_cuda or q.dim() != 2 or tuple(q.shape) != (sim.n_envs, sim.n_q):
        raise ValueError("q: a float32 CUDA tensor [n_envs, n_q] is expected")
    for name, t in (("qd", qd), ("qdd", qdd)):
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2 or tuple(t.shape) != (sim.n_envs, sim.n_qd)):
            raise ValueError(f"{name}: a float32 CUDA tensor [n_envs, n_qd] is expected")
    return _Regressor.apply(sim, q, qd, qdd)
