"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/constrained_dynamics_host.cpp - the constraint-row and solve kernels of the
point-constrained forward dynamics (csrc/tds_constrained.cu) compiled for the host - composed with the host builds of the inverse dynamics,
the inverse mass matrix and the point motion as the C-ABI composes their device launches: qdd and f in fp64 and their Jacobian-vector
products, with and without installed physical parameters.  Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load
import emu_invdyn
import emu_mass_inverse as emi
import emu_point_motion as ep

DEPS = ("tds_constrained.cu", "tds_soa.cuh", "tds_types.h", "tds_dual.cuh", "tds_math.cuh")


def lib():
    L = _load("constrained_dynamics_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci = ctypes.c_int
    L.tdsemu_cdyn.restype = ci
    L.tdsemu_cdyn.argtypes = [ci, ci, ci, ci, ctypes.c_double] + [dp] * 5 + [ci] + [dp] * 9
    return L


def _c(x):
    return None if x is None else np.ascontiguousarray(x, dtype=np.float64)


def kernels(K, dims, eps, tau, h, Mi, J, acc, dtau=None, dh=None, dMi=None, dJ=None, dacc=None, m=0):
    """The rows and solve kernels alone: (qdd [n, n_qd], f [n, K * dims]) from tau, h [n, n_qd], Mi [n, n_qd, n_qd], J [n, 6K, n_qd] and
    acc [n, 6K]; with m >= 1 their tangents [n, n_qd, m] and [n, K * dims, m] from the inputs' tangents (each may be None: zero)."""
    h, Mi = _c(h), _c(Mi)
    n, nd = h.shape
    J = _c(np.zeros((n, 0)) if J is None else J)
    acc = _c(np.zeros((n, 0)) if acc is None else acc)
    R = dims * K
    tail = (m,) if m else ()
    qdd, f = np.zeros((n, nd) + tail), np.zeros((n, R) + tail)
    out = (None, None, _dp(qdd), _dp(f)) if m else (_dp(qdd), _dp(f), None, None)
    rc = lib().tdsemu_cdyn(n, K, dims, nd, float(eps), _dp(_c(tau)), _dp(h), _dp(Mi), _dp(J), _dp(acc), m, _dp(_c(dtau)), _dp(_c(dh)),
                           _dp(_c(dMi)), _dp(_c(dJ)), _dp(_c(dacc)), *out)
    if rc:
        raise RuntimeError(f"tdsemu_cdyn rc={rc}")
    return qdd, f


def _table(links, local):
    lk = np.asarray([] if links is None else links, dtype=np.int64).ravel()
    lc = np.asarray(np.zeros((0, 3)) if local is None else local, dtype=np.float64).reshape(-1, 3)
    return lk, lc, lk.size


def constrained_dynamics(model, q, qd=None, tau=None, links=None, local=None, dims=3, eps=0.0, ids=(), values=None):
    """(qdd [n, n_qd], f [n, K, dims]) at q [n, n_q], qd and tau [n, n_qd] (None: zero; all rounded to fp32) with the parameters `ids`
    installed at `values`."""
    f32 = lambda x: None if x is None else np.asarray(x, dtype=np.float32).astype(np.float64)
    q, qd, tau = f32(np.atleast_2d(q)), f32(qd), f32(tau)
    lk, lc, K = _table(links, local)
    n, nd = q.shape[0], int(model[4])
    h = emu_invdyn.inverse_dynamics(model, q, qd, ids=ids, values=values)
    Mi = emi.mass_inverse(model, q, ids=ids, values=values)
    J = acc = None
    if K:
        J, _, acc = ep.point_motion(model, q, lk, lc, qd)
        J, acc = J.reshape(n, 6 * K, nd), acc.reshape(n, 6 * K)
    qdd, f = kernels(K, dims, eps, tau, h, Mi, J, acc)
    return qdd, f.reshape(n, K, dims)


def constrained_dynamics_jvp(model, q, qd=None, tau=None, links=None, local=None, dims=3, eps=0.0, t_q=None, t_qd=None, t_tau=None,
                             t_par=None, ids=(), values=None):
    """(dqdd [n, n_qd, m], df [n, K, dims, m]) along t_q [n, n_q, m], t_qd and t_tau [n, n_qd, m] and t_par [n, k, m] (each may be None)."""
    f32 = lambda x: None if x is None else np.asarray(x, dtype=np.float32).astype(np.float64)
    q, qd, tau = f32(np.atleast_2d(q)), f32(qd), f32(tau)
    lk, lc, K = _table(links, local)
    n, n_q, nd = q.shape[0], int(model[3]), int(model[4])
    m = next(t.shape[2] for t in (t_q, t_qd, t_tau, t_par) if t is not None)
    z = lambda d: np.zeros((n, d, m))
    t_in = np.concatenate([z(n_q) if t_q is None else t_q, z(nd) if t_qd is None else t_qd, z(nd)], axis=1)
    h = emu_invdyn.inverse_dynamics(model, q, qd, ids=ids, values=values)
    Mi = emi.mass_inverse(model, q, ids=ids, values=values)
    dh = dMi = J = acc = dJ = dacc = None
    if t_q is not None or t_qd is not None or t_par is not None:
        dh = emu_invdyn.inverse_dynamics_jvp(model, q, qd, None, t_in, t_par, ids=ids, values=values)
    if t_q is not None or t_par is not None:
        dMi = emi.mass_inverse_jvp(model, q, t_q, t_par, ids=ids, values=values)
    if K:
        J, _, acc = ep.point_motion(model, q, lk, lc, qd)
        J, acc = J.reshape(n, 6 * K, nd), acc.reshape(n, 6 * K)
        if t_q is not None or t_qd is not None:
            dJ, _, dacc = ep.split(ep.point_motion_jvp(model, q, lk, lc, t_in, qd), model, K)
            dJ, dacc = dJ.reshape(n, 6 * K * nd, m), dacc.reshape(n, 6 * K, m)
    dqdd, df = kernels(K, dims, eps, tau, h, Mi, J, acc, t_tau, dh, None if dMi is None else dMi.reshape(n, nd * nd, m), dJ, dacc, m)
    return dqdd, df.reshape(n, K, dims, m)
