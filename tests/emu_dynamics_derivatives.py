"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/dynamics_derivatives_host.cpp - the dynamics-derivative instances of the product's
generic step kernel (csrc/tds_stepw.cu, template flag DER) compiled for the host: d tau / dq and d tau / dqd of the inverse dynamics in fp64
and their Jacobian-vector products, with and without installed physical parameters.  Used only by the CPU test-suite; the package never
loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_invdyn import GRAVITY, _args, _check, _vec
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib():
    L = _load("dynamics_derivatives_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_dynamics_derivatives.restype = ci
    L.tdsemu_dynamics_derivatives.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, dp, dp]
    L.tdsemu_dynamics_derivatives_jvp.restype = ci
    L.tdsemu_dynamics_derivatives_jvp.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, ci, dp, dp, dp, dp, dp, dp]
    return L


def inverse_dynamics_derivatives(model, q, qd=None, qdd=None, ids=(), values=None, gravity=GRAVITY):
    """(d tau / dq, d tau / dqd) [n, n_qd, n_qd] at q [n, n_q], qd, qdd [n, n_qd] (None: zero; rounded to fp32) with the parameters `ids`
    installed at `values`."""
    m, q, qd, qdd, idv, k, n, v = _args(model, q, qd, qdd, ids, values)
    nd = int(m[4])
    dq, dqd = np.zeros((n, nd, nd)), np.zeros((n, nd, nd))
    _check(lib().tdsemu_dynamics_derivatives(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k,
                                             idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(dq), _dp(dqd)),
           "tdsemu_dynamics_derivatives")
    return dq, dqd


def inverse_dynamics_derivatives_jvp(model, q, qd=None, qdd=None, t_q=None, t_qd=None, t_qdd=None, t_par=None, ids=(), values=None,
                                     gravity=GRAVITY):
    """Tangents [n, n_qd, n_qd, m] of (d tau / dq, d tau / dqd) along t_q [n, n_q, m], t_qd, t_qdd [n, n_qd, m] and t_par [n, k, m]
    (each may be None)."""
    m_, q, qd, qdd, idv, k, n, v = _args(model, q, qd, qdd, ids, values)
    nd = int(m_[4])
    ts = [_vec(t) for t in (t_q, t_qd, t_qdd, t_par)]
    m = next(t for t in ts if t is not None).shape[2]
    a, b = np.zeros((n, nd, nd, m)), np.zeros((n, nd, nd, m))
    _check(lib().tdsemu_dynamics_derivatives_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k,
                                                 idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, *(_dp(t) for t in ts), _dp(a), _dp(b)),
           "tdsemu_dynamics_derivatives_jvp")
    return a, b
