"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/mass_host.cpp - the mass-matrix instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag MASS) compiled for the host: M(q) in fp64, its Jacobian-vector products and its vector-Jacobian
product, with and without installed physical parameters.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib():
    L = _load("mass_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_mass.restype = ci
    L.tdsemu_mass.argtypes = [dp, ci, ci, dp, ci, vp, dp, dp]
    L.tdsemu_mass_jvp.restype = ci
    L.tdsemu_mass_jvp.argtypes = [dp, ci, ci, dp, ci, vp, dp, ci, dp, dp, dp]
    L.tdsemu_mass_vjp.restype = ci
    L.tdsemu_mass_vjp.argtypes = [dp, ci, ci, dp, ci, vp, dp, dp, dp]
    return L


def _args(model, q, ids, values):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    n = q.shape[0]
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    return m, q, idv, k, n, v


def _check(rc, what):
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def mass(model, q, ids=(), values=None):
    """M [n, n_qd, n_qd] at q [n, n_q] (rounded to fp32) with the parameters `ids` installed at `values` [n, k] or [k]."""
    m, q, idv, k, n, v = _args(model, q, ids, values)
    nd = int(m[4])
    out = np.zeros((n, nd, nd))
    _check(lib().tdsemu_mass(_dp(m), m.size, n, _dp(q), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(out)), "tdsemu_mass")
    return out


def mass_jvp(model, q, t_q=None, t_par=None, ids=(), values=None):
    """dM [n, n_qd, n_qd, m] along t_q [n, n_q, m] and t_par [n, k, m] (either may be None)."""
    m_, q, idv, k, n, v = _args(model, q, ids, values)
    nd = int(m_[4])
    tq = None if t_q is None else np.ascontiguousarray(t_q, dtype=np.float64)
    tp = None if t_par is None else np.ascontiguousarray(t_par, dtype=np.float64)
    m = (tq if tq is not None else tp).shape[2]
    out = np.zeros((n, nd, nd, m))
    _check(lib().tdsemu_mass_jvp(_dp(m_), m_.size, n, _dp(q), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, _dp(tq), _dp(tp), _dp(out)),
           "tdsemu_mass_jvp")
    return out


def mass_vjp(model, q, G, ids=(), values=None):
    """(g_q [n, n_q], g_par [n, k]) = sum G * dM / d(q, installed parameters) for the cotangent G [n, n_qd, n_qd]."""
    m, q, idv, k, n, v = _args(model, q, ids, values)
    n_q = int(m[3])
    G = np.ascontiguousarray(G, dtype=np.float64)
    g = np.zeros((n, n_q + k))
    _check(lib().tdsemu_mass_vjp(_dp(m), m.size, n, _dp(q), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(G), _dp(g)), "tdsemu_mass_vjp")
    return g[:, :n_q], g[:, n_q:]
