"""TEST INFRASTRUCTURE: ctypes binding of the Jacobian-vector product instances of the product's kernels compiled for the host -
tests/cpp/stepw_jvp_host.cpp (csrc/tds_stepw.cu, with and without installed parameters) and tests/cpp/rigid_jvp_host.cpp
(csrc/tds_rigid.cu).  Used only by the CPU test-suite; the package never loads them."""
import ctypes

import numpy as np

from emu import _dp
from emu_params import _params
from emu_vjp import _load

STEPW_DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib_stepw():
    L = _load("stepw_jvp_host", STEPW_DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci = ctypes.c_int
    L.tdsemu_stepw_jvp.restype = ci
    L.tdsemu_stepw_jvp.argtypes = [dp, ci, dp, dp, ci, ci, ci, dp, dp, dp, ci, ctypes.c_void_p, dp, ci, dp, dp, dp]
    return L


def lib_rigid():
    L = _load("rigid_jvp_host", ("tds_rigid.cu", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh"))
    dp = ctypes.POINTER(ctypes.c_double)
    ci = ctypes.c_int
    L.tdsemu_rigid_jvp.restype = ci
    L.tdsemu_rigid_jvp.argtypes = [dp, ci, dp, ci, dp, dp, ci, ci, dp, dp, dp, dp]
    return L


def step_jvp(model, mode, q, qd, t_in=None, t_par=None, tau=None, ids=(), values=None, use_pd=False, env=None, **kw):
    """t_out [n, rows, m] = J V of one step of every environment by the tangent-seeded dual instance of the host-compiled kernel.
    t_in [n, cols, m] (input tangents, columns as emu.step(..., jacobian=True)), t_par [n, k, m] (tangents of the parameters `ids`
    installed at `values` [n, k] or [k]); either may be None.  Other arguments as tests/emu_params.py step."""
    m_ = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64); qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd = q.shape[0], int(m_[3]), int(m_[4])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    n_tau = n_qd - (6 if int(m_[2]) else 0)
    rows = n_qd if mode == 0 else n_q + n_qd
    cols = n_q + n_qd + ((int(e[0]) + 3) if use_pd else n_tau)
    ti = None if t_in is None else np.ascontiguousarray(t_in, dtype=np.float64)
    tp = None if t_par is None else np.ascontiguousarray(t_par, dtype=np.float64)
    m = (ti if ti is not None else tp).shape[2]
    if ti is not None:
        assert ti.shape == (n, cols, m), (ti.shape, cols, m)
    if tp is not None:
        assert tp.shape == (n, k, m), (tp.shape, k, m)
    out = np.zeros((n, rows, m))
    rc = lib_stepw().tdsemu_stepw_jvp(_dp(m_), m_.size, _dp(_params(**kw)), _dp(e), mode, int(use_pd), n, _dp(q), _dp(qd), _dp(t), k,
                                      idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, _dp(ti), _dp(tp), _dp(out))
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"tdsemu_stepw_jvp rc={rc}")
    return out


def rigid_jvp(desc, state, t_state=None, t_force=None, force=None, steps=1, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81), friction=0.5,
              restitution=0.0, erp=0.1, num_solver_iterations=1):
    """(state_out [n][nb][13], t_out [n][nb][13][m]) of `steps` World::step calls along the tangents t_state [n][nb][13][m] and
    t_force [n][nb][3][m] (either may be None) by the tangent-seeded dual instance of the host-compiled rigid-body kernel."""
    d = np.ascontiguousarray(desc, dtype=np.float64)
    s = np.ascontiguousarray(state, dtype=np.float64)
    n, nb = s.shape[0], d.shape[0]
    f = None if force is None else np.ascontiguousarray(force, dtype=np.float64)
    ts = None if t_state is None else np.ascontiguousarray(t_state, dtype=np.float64)
    tf = None if t_force is None else np.ascontiguousarray(t_force, dtype=np.float64)
    m = (ts if ts is not None else tf).shape[-1]
    params = np.array([dt, *gravity, friction, restitution, erp, num_solver_iterations], dtype=np.float64)
    so, to = np.zeros_like(s), np.zeros((n, nb, 13, m))
    rc = lib_rigid().tdsemu_rigid_jvp(_dp(d), nb, _dp(params), n, _dp(s), _dp(f), steps, m, _dp(ts), _dp(tf), _dp(so), _dp(to))
    if rc:
        raise RuntimeError(f"tdsemu_rigid_jvp rc={rc}")
    return so, to
