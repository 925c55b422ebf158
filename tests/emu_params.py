"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/stepw_param_host.cpp - the instances of the product's generic step kernel
(csrc/tds_stepw.cu) that read per-environment physical parameters, compiled for the host: float / double forward, dual numbers
over the parameters (or over the inputs) and the taping scalar.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu_vjp import _load
from emu import _dp

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib():
    L = _load("stepw_param_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci = ctypes.c_int
    L.tdsemu_param_count.restype = ci
    L.tdsemu_param_count.argtypes = [dp, ci]
    L.tdsemu_stepw_par.restype = ci
    L.tdsemu_stepw_par.argtypes = [dp, ci, dp, dp, ci, ci, ci, ci, ci, dp, dp, dp, ci, ctypes.c_void_p, dp] + [dp] * 7 + [ci, dp]
    return L


def param_count(model):
    m = np.ascontiguousarray(model, dtype=np.float64)
    return lib().tdsemu_param_count(_dp(m), m.size)


def _params(dt=1e-3, gravity=(0.0, 0.0, -9.81), friction=0.5, restitution=0.0, erp=0.2, cfm=1e-5, pgs_iterations=1, keep_all_points=False,
            contact_model=0, spring_k=50000.0, damper_d=5000.0, exponent_n=1.5, v_transition=0.01, hard_contact_condition=True):
    return np.array([dt, *gravity, friction, restitution, erp, cfm, pgs_iterations, int(keep_all_points), contact_model, spring_k,
                     damper_d, exponent_n, v_transition, int(hard_contact_condition)], dtype=np.float64)


def step(model, mode, q, qd, tau=None, ids=(), values=None, what="forward", precision=1, use_pd=False, env=None, g_out=None, want_g_in=True,
         tape_cap=1 << 16, **kw):
    """One step of every environment with the parameters `ids` installed at `values` [n, k] (or [k] for all environments).
    what: "forward" -> dict(q, qd, qdd) at `precision` (0 mixed, 1 fp64, 2 fp32); "param_jacobian" -> dict(jac [n, rows, k]);
    "jacobian" -> dict(jac [n, rows, cols]) over the inputs; "vjp" -> dict(g_in [n, cols] (None unless want_g_in), g_par [n, k],
    nodes, cap, reruns) from g_out [n, rows].  Other arguments as tests/emu.py step."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64); qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd = q.shape[0], int(m[3]), int(m[4])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    n_tau = n_qd - (6 if int(m[2]) else 0)
    rows = n_qd if mode == 0 else n_q + n_qd
    cols = n_q + n_qd + ((int(e[0]) + 3) if use_pd else n_tau)
    code = {"forward": 0, "param_jacobian": 1, "jacobian": 2, "vjp": 3}[what]
    out = {}
    qo, qdo, qddo = np.zeros((n, n_q)), np.zeros((n, n_qd)), np.zeros((n, n_qd))
    jac = g = g_in = g_par = stats = None
    if code == 1:
        jac = np.zeros((n, rows, k))
    elif code == 2:
        jac = np.zeros((n, rows, cols))
    elif code == 3:
        g = np.ascontiguousarray(g_out, dtype=np.float64)
        assert g.shape == (n, rows), (g.shape, rows)
        g_in = np.zeros((n, cols)) if want_g_in else None
        g_par = np.zeros((n, max(k, 1)))
        stats = np.zeros(n + 2)
    rc = lib().tdsemu_stepw_par(_dp(m), m.size, _dp(_params(**kw)), _dp(e), code, precision, mode, int(use_pd), n, _dp(q), _dp(qd), _dp(t), k,
                                idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(qo), _dp(qdo), _dp(qddo), _dp(jac), _dp(g), _dp(g_in),
                                _dp(g_par), int(tape_cap), _dp(stats))
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"tdsemu_stepw_par rc={rc}")
    if code == 0:
        out.update(q=qo, qd=qdo, qdd=qddo)
    elif code in (1, 2):
        out["jac"] = jac
    else:
        out.update(g_in=g_in, g_par=g_par[:, :k], nodes=stats[:n].astype(np.int64), cap=int(stats[n]), reruns=int(stats[n + 1]))
    return out
