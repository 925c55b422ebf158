"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/mass_inverse_host.cpp - the inverse-mass-matrix instances of the product's generic
step kernel (csrc/tds_stepw.cu, template flags MASS and MINV) and the contraction kernel of J M^-1 J^T (csrc/tds_mass_inverse.cu)
compiled for the host: M^-1(q) in fp64 and its Jacobian-vector products, with and without installed physical parameters, and the
operational-space inverse inertia with its tangents.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_mass_inverse.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h",
        "tds_types.h")


def lib():
    L = _load("mass_inverse_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_mass_inverse.restype = ci
    L.tdsemu_mass_inverse.argtypes = [dp, ci, ci, dp, ci, vp, dp, dp]
    L.tdsemu_mass_inverse_jvp.restype = ci
    L.tdsemu_mass_inverse_jvp.argtypes = [dp, ci, ci, dp, ci, vp, dp, ci, dp, dp, dp]
    L.tdsemu_osim.restype = ci
    L.tdsemu_osim.argtypes = [ci, ci, ci, dp, dp, ci, dp, dp, dp]
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


def mass_inverse(model, q, ids=(), values=None):
    """M^-1 [n, n_qd, n_qd] at q [n, n_q] (rounded to fp32) with the parameters `ids` installed at `values` [n, k] or [k]."""
    m, q, idv, k, n, v = _args(model, q, ids, values)
    nd = int(m[4])
    out = np.zeros((n, nd, nd))
    _check(lib().tdsemu_mass_inverse(_dp(m), m.size, n, _dp(q), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(out)),
           "tdsemu_mass_inverse")
    return out


def mass_inverse_jvp(model, q, t_q=None, t_par=None, ids=(), values=None):
    """dM^-1 [n, n_qd, n_qd, m] along t_q [n, n_q, m] and t_par [n, k, m] (either may be None)."""
    m_, q, idv, k, n, v = _args(model, q, ids, values)
    nd = int(m_[4])
    tq = None if t_q is None else np.ascontiguousarray(t_q, dtype=np.float64)
    tp = None if t_par is None else np.ascontiguousarray(t_par, dtype=np.float64)
    m = (tq if tq is not None else tp).shape[2]
    out = np.zeros((n, nd, nd, m))
    _check(lib().tdsemu_mass_inverse_jvp(_dp(m_), m_.size, n, _dp(q), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, _dp(tq), _dp(tp),
                                         _dp(out)), "tdsemu_mass_inverse_jvp")
    return out


def osim(J, Minv, dJ=None, dMinv=None):
    """L = J Minv J^T [n, 6K, 6K] from J [n, K, 6, n_qd] (or [n, 6K, n_qd]) and Minv [n, n_qd, n_qd] by the contraction kernel; with dMinv
    [n, n_qd, n_qd, m] (and dJ [n, 6K, n_qd, m] or None: zero) its tangents [n, 6K, 6K, m]."""
    Minv = np.ascontiguousarray(Minv, dtype=np.float64)
    n, nd = Minv.shape[0], Minv.shape[1]
    J = np.ascontiguousarray(np.reshape(J, (n, -1, nd)), dtype=np.float64)
    R = J.shape[1]
    m = 0 if dMinv is None else dMinv.shape[-1]
    dJ = None if dJ is None else np.ascontiguousarray(np.reshape(dJ, (n, R, nd, m)), dtype=np.float64)
    dMinv = None if dMinv is None else np.ascontiguousarray(dMinv, dtype=np.float64)
    out = np.zeros((n, R, R) + ((m,) if m else ()))
    _check(lib().tdsemu_osim(n, R // 6, nd, _dp(J), _dp(Minv), m, _dp(dJ), _dp(dMinv), _dp(out)), "tdsemu_osim")
    return out
