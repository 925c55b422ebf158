"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/fd_derivatives_host.cpp - the product kernel of the forward dynamics' derivatives
(csrc/tds_fd_derivatives.cu) and the DER instances of csrc/tds_stepw.cu reading qdd in fp64, compiled for the host - composed with the host
builds of the inverse dynamics, the inverse mass matrix and the constrained dynamics' solve (tests/emu_constrained_dynamics.py) as the
C-ABI composes their device launches: qdd, d qdd / dq, d qdd / dqd and d qdd / dtau in fp64 and their Jacobian-vector products, with and
without installed physical parameters.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_invdyn import GRAVITY, _args, _check, _vec
from emu_vjp import _load
import emu_constrained_dynamics as ecd
import emu_mass_inverse as emi

DEPS = ("tds_fd_derivatives.cu", "tds_soa.cuh", "tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh",
        "tds_model.h", "tds_types.h", "../../tests/cpp/dynamics_derivatives_host.cpp")


def lib():
    L = _load("fd_derivatives_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_der_qdd64.restype = ci
    L.tdsemu_der_qdd64.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, ci, dp, dp, dp, dp, dp, dp]
    L.tdsemu_fdd.restype = ci
    L.tdsemu_fdd.argtypes = [ci, ci, dp, dp, dp, ci, dp, dp, dp, dp, dp, dp]
    return L


def der_qdd64(model, q, qd, qdd, ids=(), values=None, t_q=None, t_qd=None, t_qdd=None, t_par=None, gravity=GRAVITY):
    """(d tau / dq, d tau / dqd) [n, n_qd, n_qd] of the DER instances at q, qd (rounded to fp32) and qdd read in fp64; with any tangent t_q
    [n, n_q, m], t_qd, t_qdd [n, n_qd, m], t_par [n, k, m] instead their tangents [n, n_qd, n_qd, m]."""
    m_, q, qd, _, idv, k, n, v = _args(model, q, qd, None, ids, values)
    nd = int(m_[4])
    qdd = np.ascontiguousarray(np.atleast_2d(qdd), dtype=np.float64)
    ts = [_vec(t) for t in (t_q, t_qd, t_qdd, t_par)]
    m = next((t.shape[2] for t in ts if t is not None), 0)
    tail = (m,) if m else ()
    a, b = np.zeros((n, nd, nd) + tail), np.zeros((n, nd, nd) + tail)
    _check(lib().tdsemu_der_qdd64(_dp(m_), m_.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k, idv.ctypes.data_as(ctypes.c_void_p),
                                  _dp(v), m, *(_dp(t) for t in ts), _dp(a), _dp(b)), "tdsemu_der_qdd64")
    return a, b


def product(Mi, Aq, Aqd, dMi=None, dAq=None, dAqd=None, m=0):
    """The product kernel alone: (-Mi Aq, -Mi Aqd, Mi) [n, n_qd, n_qd]; with m >= 1 instead their tangents [n, n_qd, n_qd, m] from the
    tangents [n, n_qd, n_qd, m] of the inputs (each may be None: zero)."""
    c = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float64)
    Mi, Aq, Aqd = c(Mi), c(Aq), c(Aqd)
    n, nd = Mi.shape[0], Mi.shape[1]
    tail = (m,) if m else ()
    out = [np.zeros((n, nd, nd) + tail) for _ in range(3)]
    rc = lib().tdsemu_fdd(n, nd, _dp(Mi), _dp(Aq), _dp(Aqd), m, _dp(c(dMi)), _dp(c(dAq)), _dp(c(dAqd)), *(_dp(o) for o in out))
    if rc:
        raise RuntimeError(f"tdsemu_fdd rc={rc}")
    return tuple(out)


def forward_dynamics_derivatives(model, q, qd=None, tau=None, ids=(), values=None):
    """(qdd [n, n_qd], d qdd / dq, d qdd / dqd, d qdd / dtau [n, n_qd, n_qd]) at q [n, n_q], qd and tau [n, n_qd] (None: zero; rounded to
    fp32) with the parameters `ids` installed at `values`."""
    qdd, _ = ecd.constrained_dynamics(model, q, qd, tau, ids=ids, values=values)
    Mi = emi.mass_inverse(model, q, ids=ids, values=values)
    Aq, Aqd = der_qdd64(model, q, qd, qdd, ids, values)
    return (qdd,) + product(Mi, Aq, Aqd)


def forward_dynamics_derivatives_jvp(model, q, qd=None, tau=None, t_q=None, t_qd=None, t_tau=None, t_par=None, ids=(), values=None):
    """Tangents (dqdd [n, n_qd, m], d(d qdd / dq), d(d qdd / dqd), d(d qdd / dtau) [n, n_qd, n_qd, m]) along t_q [n, n_q, m], t_qd and
    t_tau [n, n_qd, m] and t_par [n, k, m] (each may be None, not all)."""
    qdd, _ = ecd.constrained_dynamics(model, q, qd, tau, ids=ids, values=values)
    Mi = emi.mass_inverse(model, q, ids=ids, values=values)
    Aq, Aqd = der_qdd64(model, q, qd, qdd, ids, values)
    dqdd, _ = ecd.constrained_dynamics_jvp(model, q, qd, tau, t_q=t_q, t_qd=t_qd, t_tau=t_tau, t_par=t_par, ids=ids, values=values)
    n, nd, m = qdd.shape[0], qdd.shape[1], dqdd.shape[2]
    dMi = None
    if t_q is not None or t_par is not None:
        dMi = emi.mass_inverse_jvp(model, q, t_q, t_par, ids=ids, values=values).reshape(n, nd, nd, m)
    dAq, dAqd = der_qdd64(model, q, qd, qdd, ids, values, t_q, t_qd, dqdd, t_par)
    return (dqdd,) + product(Mi, Aq, Aqd, dMi, dAq, dAqd, m)
