"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/invdyn_host.cpp - the inverse-dynamics instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag INV) compiled for the host: tau = ID(q, qd, qdd) in fp64, its Jacobian-vector products and its
vector-Jacobian product, with and without installed physical parameters - and of tests/cpp/oracle_invdyn.c, the C oracle's inverse
dynamics restated in link frames.  Used only by the CPU test-suite; the package never loads them."""
import ctypes
import os
import subprocess

import numpy as np

from emu import HERE, ROOT, _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")
GRAVITY = (0.0, 0.0, -9.81)
_oracle = None


def lib():
    L = _load("invdyn_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_invdyn.restype = ci
    L.tdsemu_invdyn.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, dp]
    L.tdsemu_invdyn_jvp.restype = ci
    L.tdsemu_invdyn_jvp.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, ci, dp, dp, dp]
    L.tdsemu_invdyn_vjp.restype = ci
    L.tdsemu_invdyn_vjp.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, vp, dp, dp, dp]
    return L


def oracle_lib():
    """tests/cpp/oracle_invdyn.c built next to it (rebuilt when it or the oracle source is newer)."""
    global _oracle
    if _oracle is None:
        src = os.path.join(HERE, "cpp", "oracle_invdyn.c")
        so = os.path.join(HERE, "cpp", "_oracle_invdyn.so")
        deps = [src, os.path.join(ROOT, "oracle", "tds_oracle.c"), os.path.join(ROOT, "oracle", "tds_oracle.h")]
        if not (os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"),
                                   "-I" + os.path.join(ROOT, "oracle"), src, "-o", so + ".tmp", "-lm"])
            os.replace(so + ".tmp", so)
        L = ctypes.CDLL(so)
        dp = ctypes.POINTER(ctypes.c_double)
        L.tdso_inverse_dynamics.restype = ctypes.c_int
        L.tdso_inverse_dynamics.argtypes = [dp, dp, dp, dp, dp, dp]
        _oracle = L
    return _oracle


def _vec(x):
    return None if x is None else np.ascontiguousarray(x, dtype=np.float64)


def oracle(model, q, qd=None, qdd=None, gravity=GRAVITY):
    """The C oracle's tau [n_qd] at one q, qd, qdd (fp64, as given; None: zero)."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    tau = np.zeros(int(m[4]))
    rc = oracle_lib().tdso_inverse_dynamics(_dp(m), _dp(_vec(q)), _dp(_vec(qd)), _dp(_vec(qdd)), _dp(_vec(gravity)), _dp(tau))
    if rc:
        raise RuntimeError(f"tdso_inverse_dynamics rc={rc}")
    return tau


def _args(model, q, qd, qdd, ids, values):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    n = q.shape[0]
    qd = None if qd is None else np.ascontiguousarray(np.atleast_2d(qd), dtype=np.float64)
    qdd = None if qdd is None else np.ascontiguousarray(np.atleast_2d(qdd), dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    return m, q, qd, qdd, idv, k, n, v


def _check(rc, what):
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def inverse_dynamics(model, q, qd=None, qdd=None, ids=(), values=None, gravity=GRAVITY):
    """tau [n, n_qd] at q [n, n_q], qd, qdd [n, n_qd] (None: zero; rounded to fp32) with the parameters `ids` installed at `values`."""
    m, q, qd, qdd, idv, k, n, v = _args(model, q, qd, qdd, ids, values)
    out = np.zeros((n, int(m[4])))
    _check(lib().tdsemu_invdyn(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k, idv.ctypes.data_as(ctypes.c_void_p),
                               _dp(v), _dp(out)), "tdsemu_invdyn")
    return out


def inverse_dynamics_jvp(model, q, qd=None, qdd=None, t_in=None, t_par=None, ids=(), values=None, gravity=GRAVITY):
    """dtau [n, n_qd, m] along t_in [n, n_q + 2 n_qd, m] (q | qd | qdd tangents) and t_par [n, k, m] (either may be None)."""
    m_, q, qd, qdd, idv, k, n, v = _args(model, q, qd, qdd, ids, values)
    ti, tp = _vec(t_in), _vec(t_par)
    m = (ti if ti is not None else tp).shape[2]
    out = np.zeros((n, int(m_[4]), m))
    _check(lib().tdsemu_invdyn_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k,
                                   idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, _dp(ti), _dp(tp), _dp(out)), "tdsemu_invdyn_jvp")
    return out


def inverse_dynamics_vjp(model, q, qd, qdd, G, ids=(), values=None, gravity=GRAVITY):
    """(g_in [n, n_q + 2 n_qd], g_par [n, k]) = sum_r G[r] dtau[r] / d(q | qd | qdd, installed parameters) for G [n, n_qd]."""
    m, q, qd, qdd, idv, k, n, v = _args(model, q, qd, qdd, ids, values)
    n_in = int(m[3]) + 2 * int(m[4])
    G = np.ascontiguousarray(G, dtype=np.float64)
    g = np.zeros((n, n_in + k))
    _check(lib().tdsemu_invdyn_vjp(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(_vec(gravity)), k, idv.ctypes.data_as(ctypes.c_void_p),
                                   _dp(v), _dp(G), _dp(g)), "tdsemu_invdyn_vjp")
    return g[:, :n_in], g[:, n_in:]
