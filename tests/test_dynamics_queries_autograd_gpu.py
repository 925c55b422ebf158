"""The torch.autograd binding of the six dynamics queries on the H100 (tds_b200.autograd, DESIGN.md section 7.12): mass_matrix,
inverse_dynamics, centroidal, forward_kinematics, point_motion and regressor share one Function, and on every combination of the inputs
each query takes they match the host entries - values bit for bit, gradients and tangents within 1e-12.  The per-query tests
(tests/test_*_gpu.py) cover each query with all of its inputs given."""
import itertools

import numpy as np
import pytest

import tds_b200
from test_dynamics_queries_gpu import _ids, _setup
from test_mass_matrix_on_host import f32, rel
from test_params_on_host import perturbed

pytestmark = pytest.mark.gpu

_SYM = [0, 1, 2, 1, 3, 4, 2, 4, 5]
# the inputs each query takes beyond q; "points": a table of three points, or none (K = 0)
_OPTIONAL = {"mass_matrix": ("params",), "inverse_dynamics": ("qd", "qdd", "params"), "centroidal": ("qd", "params"),
             "forward_kinematics": ("points",), "point_motion": ("qd", "qdd", "points"), "regressor": ("qd", "qdd")}
_COMBOS = [(query, tuple(o for o, on in zip(opts, mask) if on)) for query, opts in _OPTIONAL.items()
           for mask in itertools.product((False, True), repeat=len(opts))]


def _host_query(query, sim, q, qd, qdd, pts):
    """The host entries in the layout of tds_b200.autograd: (value, jvp(tq, tqd, tqdd, tp), vjp(*G) -> (g_q, g_qd, g_qdd, g_par))."""
    n = sim.n_envs
    if query == "mass_matrix":
        return ((sim.mass_matrix_host(q),), lambda tq, tqd, tqdd, tp: (sim.mass_matrix_jvp_host(q, tq, tp)[1],),
                lambda G: (lambda g_q, g_par: (g_q, None, None, g_par))(*sim.mass_matrix_vjp_host(q, G)))
    if query == "inverse_dynamics":
        return ((sim.inverse_dynamics_host(q, qd, qdd),), lambda *t: (sim.inverse_dynamics_jvp_host(q, qd, qdd, *t)[1],),
                lambda G: sim.inverse_dynamics_vjp_host(q, qd, qdd, G))
    if query == "centroidal":
        def jvp(tq, tqd, tqdd, tp):
            dcom, dA, db = sim.centroidal_jvp_host(q, qd, tq, tqd, tp)
            return dcom[:, 0], dcom[:, 1:4], dcom[:, 4:10][:, _SYM].reshape(n, 3, 3), dA, db

        def vjp(Gm, Gc, GI, GA, Gb):
            Gcom = np.concatenate([Gm[:, None], Gc, (GI + GI.transpose(0, 2, 1)).reshape(n, 9)[:, [0, 1, 2, 4, 5, 8]]], axis=1)
            Gcom[:, [4, 7, 9]] *= 0.5   # the diagonal is read once
            g_q, g_qd, g_par = sim.centroidal_vjp_host(q, qd, Gcom, GA, Gb)
            return g_q, g_qd, None, g_par
        return sim.centroidal_host(q, qd), jvp, vjp
    lk, lc = pts
    if query == "forward_kinematics":
        def jvp(tq, tqd, tqdd, tp):
            dxf, dx, dJ = sim.kinematics_jvp_host(q, lk, lc, tq)
            return dxf[..., :9].reshape(n, sim.n_links, 3, 3), dxf[..., 9:], dx, dJ
        return (sim.kinematics_host(q, lk, lc), jvp, lambda GR, Gp, Gx, GJ: (
            sim.kinematics_vjp_host(q, lk, lc, np.concatenate([GR.reshape(n, -1, 9), Gp], axis=2), Gx, GJ), None, None, None))
    if query == "point_motion":
        return (sim.point_motion_host(q, qd, lk, lc, qdd),
                lambda tq, tqd, tqdd, tp: sim.point_motion_jvp_host(q, qd, lk, lc, qdd, tq, tqd, tqdd),
                lambda *G: sim.point_motion_vjp_host(q, qd, lk, lc, qdd, *G) + (None,))
    return (sim.regressor_host(q, qd, qdd), lambda tq, tqd, tqdd, tp: sim.regressor_jvp_host(q, qd, qdd, tq, tqd, tqdd),
            lambda *G: sim.regressor_vjp_host(q, qd, qdd, *G) + (None,))


@pytest.mark.parametrize("query,given", _COMBOS, ids=[f"{q}-{'+'.join(('q',) + g)}" for q, g in _COMBOS])
def test_autograd_binding_on_every_input_combination(query, given):
    """tds_b200.autograd's six queries on the humanoid with qd and qdd given or None, with and without params, with a point table and
    without points (K = 0): values bit for bit against the host entries; a loss on every output and on the last output only, against
    the host VJP (absent inputs get no gradient); forward mode with tangents on every given input, on the last one only (absent inputs
    and those without a tangent are ignored) and zero tangents on every input (exactly zero), against the host JVP."""
    import torch
    import torch.autograd.forward_ad as fwAD
    n = 64
    model, sim, q, qd, qdd = _setup("humanoid", "params" in given, n)
    qd, qdd = (qd if "qd" in given else None), (qdd if "qdd" in given else None)
    vals = perturbed(model, _ids(model), n, 5, 0.5, 0.0) if "params" in given else None
    K = 3 if "points" in given else 0
    pts = (np.array([-1, 0, sim.n_links - 1])[:K], np.random.default_rng(11).normal(size=(3, 3))[:K] * 0.1)
    host, host_jvp, host_vjp = _host_query(query, sim, q, qd, qdd, pts)
    cu = lambda x, dt=torch.float32: None if x is None else torch.tensor(x, dtype=dt, device="cuda")
    xs = {"q": cu(q), "qd": cu(qd), "qdd": cu(qdd), "params": cu(vals, torch.float64)}

    def call(x):
        f = getattr(tds_b200.autograd, query)
        if query == "mass_matrix":
            out = f(sim, x["q"], x["params"])
        elif query in ("inverse_dynamics", "centroidal"):
            out = f(sim, x["q"], x["qd"], *([x["qdd"]] if query == "inverse_dynamics" else []), params=x["params"])
        elif query == "forward_kinematics":
            out = f(sim, x["q"], *pts)
        elif query == "point_motion":
            out = f(sim, x["q"], x["qd"], *pts, qdd=x["qdd"])
        else:
            out = f(sim, x["q"], x["qd"], x["qdd"])
        return (out,) if isinstance(out, torch.Tensor) else out

    outs = call(xs)
    assert len(outs) == len(host)
    for o, h in zip(outs, host):
        assert o.dtype == torch.float64 and o.is_contiguous() and np.array_equal(o.cpu().numpy(), h)
    rng = np.random.default_rng(12)
    G = [rng.normal(size=h.shape) for h in host]
    for on in [None, len(host) - 1] if len(host) > 1 else [None]:
        Gs = [g if on is None or i == on else np.zeros_like(g) for i, g in enumerate(G)]
        xr = {k: None if v is None else v.clone().requires_grad_(True) for k, v in xs.items()}
        sum((o * cu(g, torch.float64)).sum() for i, (o, g) in enumerate(zip(call(xr), Gs)) if on is None or i == on).backward()
        want = host_vjp(*Gs) if K or query != "point_motion" else (np.zeros((n, sim.n_q)), np.zeros((n, sim.n_qd)),
                                                                    np.zeros((n, sim.n_qd)), None)
        for k, w in zip(("q", "qd", "qdd", "params"), want):
            x = xr[k]
            if x is None:
                continue
            dt = torch.float64 if k == "params" else torch.float32
            assert x.grad is not None and x.grad.dtype == dt and x.grad.is_contiguous(), (k, on)
            ref = w if k == "params" else f32(w)
            assert rel(x.grad.cpu().numpy().astype(np.float64), ref) <= 1e-12, (k, on)
    present = [k for k, v in xs.items() if v is not None]
    for tangent_on in sorted({tuple(present), (present[-1],)}, key=len):
        v = {k: f32(rng.normal(size=xs[k].shape)) if k != "params" else rng.normal(size=xs[k].shape) for k in tangent_on}
        with fwAD.dual_level():
            duals = {k: x if k not in v else fwAD.make_dual(x, cu(v[k], x.dtype)) for k, x in xs.items()}
            tans = [fwAD.unpack_dual(o).tangent for o in call(duals)]
            tans = [t.cpu().numpy() for t in tans]
        want = host_jvp(*(v.get(k) for k in ("q", "qd", "qdd", "params"))) if K or query != "point_motion" else host
        for t, w in zip(tans, want):
            assert t.shape == w.shape and rel(t, w) <= 1e-12, tangent_on
    with fwAD.dual_level():
        duals = {k: x if x is None else fwAD.make_dual(x, torch.zeros_like(x)) for k, x in xs.items()}
        for o, h in zip(call(duals), host):
            t = fwAD.unpack_dual(o).tangent
            assert t.shape == h.shape and not t.cpu().numpy().any()
