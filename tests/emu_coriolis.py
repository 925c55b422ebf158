"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/coriolis_host.cpp - the Coriolis-matrix instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag COR) compiled for the host: C(q, qd) in fp64, its Jacobian-vector products and its vector-Jacobian
product, with and without installed physical parameters.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib():
    L = _load("coriolis_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_coriolis.restype = ci
    L.tdsemu_coriolis.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, dp]
    L.tdsemu_coriolis_jvp.restype = ci
    L.tdsemu_coriolis_jvp.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, ci, dp, dp, dp, dp]
    L.tdsemu_coriolis_vjp.restype = ci
    L.tdsemu_coriolis_vjp.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, dp, dp]
    return L


def _args(model, q, qd, ids, values):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    qd = None if qd is None else np.ascontiguousarray(np.atleast_2d(qd), dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    n = q.shape[0]
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    return m, q, qd, idv, k, n, v


def _check(rc, what):
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def coriolis(model, q, qd=None, ids=(), values=None):
    """C [n, n_qd, n_qd] at q [n, n_q] and qd [n, n_qd] (rounded to fp32; None: zero) with the parameters `ids` installed at `values`
    [n, k] or [k]."""
    m, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    nd = int(m[4])
    out = np.zeros((n, nd, nd))
    _check(lib().tdsemu_coriolis(_dp(m), m.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(out)),
           "tdsemu_coriolis")
    return out


def coriolis_jvp(model, q, qd=None, t_q=None, t_qd=None, t_par=None, ids=(), values=None):
    """dC [n, n_qd, n_qd, m] along t_q [n, n_q, m], t_qd [n, n_qd, m] and t_par [n, k, m] (each may be None)."""
    m_, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    nd = int(m_[4])
    ts = [None if t is None else np.ascontiguousarray(t, dtype=np.float64) for t in (t_q, t_qd, t_par)]
    m = next(t for t in ts if t is not None).shape[2]
    out = np.zeros((n, nd, nd, m))
    _check(lib().tdsemu_coriolis_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m,
                                     *(_dp(t) for t in ts), _dp(out)), "tdsemu_coriolis_jvp")
    return out


def coriolis_vjp(model, q, qd, G, ids=(), values=None):
    """(g_q [n, n_q], g_qd [n, n_qd], g_par [n, k]) = sum G * dC / d(q, qd, installed parameters) for the cotangent G [n, n_qd, n_qd]."""
    m, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    n_q, nd = int(m[3]), int(m[4])
    G = np.ascontiguousarray(G, dtype=np.float64)
    g = np.zeros((n, n_q + nd + k))
    _check(lib().tdsemu_coriolis_vjp(_dp(m), m.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(G), _dp(g)),
           "tdsemu_coriolis_vjp")
    return g[:, :n_q], g[:, n_q:n_q + nd], g[:, n_q + nd:]
