"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/point_motion_host.cpp - the point-motion instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag MOT) compiled for the host: spatial point Jacobians J [K, 6, n_qd], point velocities vel [K, 6] and
accelerations acc [K, 6] in fp64, their Jacobian-vector products and their vector-Jacobian product - and of tests/cpp/oracle_motion.c, the
C oracle's link velocities and accelerations.  Used only by the CPU test-suite; the package never loads them."""
import ctypes
import os
import subprocess

import numpy as np

from emu import HERE, ROOT, _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")
_oracle = None


def lib():
    L = _load("point_motion_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_point_motion.restype = ci
    L.tdsemu_point_motion.argtypes = [dp, ci, ci, dp, dp, dp, ci, vp, dp, dp, dp, dp]
    L.tdsemu_point_motion_jvp.restype = ci
    L.tdsemu_point_motion_jvp.argtypes = [dp, ci, ci, dp, dp, dp, ci, vp, dp, ci, dp, dp]
    L.tdsemu_point_motion_vjp.restype = ci
    L.tdsemu_point_motion_vjp.argtypes = [dp, ci, ci, dp, dp, dp, ci, vp, dp, dp, dp]
    return L


def oracle_lib():
    """tests/cpp/oracle_motion.c built next to it (rebuilt when it or the oracle source is newer)."""
    global _oracle
    if _oracle is None:
        src = os.path.join(HERE, "cpp", "oracle_motion.c")
        so = os.path.join(HERE, "cpp", "_oracle_motion.so")
        deps = [src, os.path.join(ROOT, "oracle", "tds_oracle.c"), os.path.join(ROOT, "oracle", "tds_oracle.h")]
        if not (os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"),
                                   "-I" + os.path.join(ROOT, "oracle"), src, "-o", so + ".tmp", "-lm"])
            os.replace(so + ".tmp", so)
        L = ctypes.CDLL(so)
        dp = ctypes.POINTER(ctypes.c_double)
        L.tdso_motion.restype = ctypes.c_int
        L.tdso_motion.argtypes = [dp, dp, dp, dp, dp]
        _oracle = L
    return _oracle


def oracle_motion(model, q, qd, qdd):
    """The C oracle's (R [n_links + 1, 3, 3], origin [n_links + 1, 3], v [n_links + 1, 6], a [n_links + 1, 6]) of the base (index 0) and
    every link (index i + 1) at q, qd, qdd (fp64, as given; qdd None: zero): v and a in link axes at the link origin, no gravity."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    nl = int(m[1])
    out = np.zeros((nl + 1, 24))
    c = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float64)
    rc = oracle_lib().tdso_motion(_dp(m), _dp(c(q)), _dp(c(qd)), _dp(c(qdd)), _dp(out))
    if rc:
        raise RuntimeError(f"tdso_motion rc={rc}")
    return out[:, :9].reshape(-1, 3, 3), out[:, 9:12], out[:, 12:18], out[:, 18:24]


def _args(model, q, qd, qdd, links, local):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    c = lambda x: None if x is None else np.ascontiguousarray(np.atleast_2d(x), dtype=np.float64)
    lk = np.ascontiguousarray(links, dtype=np.int32).ravel()
    lc = np.ascontiguousarray(local, dtype=np.float64).reshape(-1)
    assert lc.size == 3 * lk.size
    return m, q, c(qd), c(qdd), lk, lc, lk.size, q.shape[0]


def _check(rc, what):
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def rows(model, K):
    """(rows of J, of vel, of acc) for a model and K points."""
    return 6 * K * int(model[4]), 6 * K, 6 * K


def point_motion(model, q, links, local, qd=None, qdd=None, concat=False):
    """(J [n, K, 6, n_qd], vel [n, K, 6], acc [n, K, 6]) at q [n, n_q], qd and qdd [n, n_qd] (None: zero; all rounded to fp32); or the
    concatenated rows [n, rows]."""
    m, q, qd, qdd, lk, lc, K, n = _args(model, q, qd, qdd, links, local)
    nd = int(m[4])
    J, vel, acc = np.zeros((n, K, 6, nd)), np.zeros((n, K, 6)), np.zeros((n, K, 6))
    _check(lib().tdsemu_point_motion(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), _dp(J),
                                     _dp(vel), _dp(acc)), "tdsemu_point_motion")
    if concat:
        return np.concatenate([J.reshape(n, -1), vel.reshape(n, -1), acc.reshape(n, -1)], axis=1)
    return J, vel, acc


def split(out, model, K):
    """(J [n, K, 6, n_qd, ...], vel [n, K, 6, ...], acc [n, K, 6, ...]) from the concatenated rows [n, rows, ...]."""
    n, tail = out.shape[0], out.shape[2:]
    r_J, r_v, _ = rows(model, K)
    return (out[:, :r_J].reshape((n, K, 6, int(model[4])) + tail), out[:, r_J:r_J + r_v].reshape((n, K, 6) + tail),
            out[:, r_J + r_v:].reshape((n, K, 6) + tail))


def point_motion_jvp(model, q, links, local, t_in, qd=None, qdd=None):
    """The concatenated rows' derivatives [n, rows, m] along t_in [n, n_q + 2 n_qd, m] (q | qd | qdd tangents)."""
    m_, q, qd, qdd, lk, lc, K, n = _args(model, q, qd, qdd, links, local)
    ti = np.ascontiguousarray(t_in, dtype=np.float64)
    m = ti.shape[2]
    out = np.zeros((n, sum(rows(m_, K)), m))
    _check(lib().tdsemu_point_motion_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), _dp(qdd), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), m,
                                         _dp(ti), _dp(out)), "tdsemu_point_motion_jvp")
    return out


def point_motion_vjp(model, q, links, local, G, qd=None, qdd=None):
    """g [n, n_q + 2 n_qd] = <G, d(J | vel | acc) / d(q | qd | qdd)> for the concatenated cotangent G [n, rows]."""
    m, q, qd, qdd, lk, lc, K, n = _args(model, q, qd, qdd, links, local)
    G = np.ascontiguousarray(G, dtype=np.float64)
    assert G.shape == (n, sum(rows(m, K)))
    g = np.zeros((n, int(m[3]) + 2 * int(m[4])))
    _check(lib().tdsemu_point_motion_vjp(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), _dp(G),
                                         _dp(g)), "tdsemu_point_motion_vjp")
    return g
