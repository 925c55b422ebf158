"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/kin_host.cpp - the kinematics instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag KIN) compiled for the host: link world transforms, point positions and linear point Jacobians in fp64,
their Jacobian-vector products and their vector-Jacobian product - and of tests/cpp/oracle_kin.c, the C oracle's point Jacobian.  Used
only by the CPU test-suite; the package never loads them."""
import ctypes
import os
import subprocess

import numpy as np

from emu import HERE, ROOT, _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")
_oracle = None


def lib():
    L = _load("kin_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_kin.restype = ci
    L.tdsemu_kin.argtypes = [dp, ci, ci, dp, ci, vp, dp, dp, dp, dp]
    L.tdsemu_kin_jvp.restype = ci
    L.tdsemu_kin_jvp.argtypes = [dp, ci, ci, dp, ci, vp, dp, ci, dp, dp]
    L.tdsemu_kin_vjp.restype = ci
    L.tdsemu_kin_vjp.argtypes = [dp, ci, ci, dp, ci, vp, dp, dp, dp]
    return L


def oracle_lib():
    """tests/cpp/oracle_kin.c built next to it (rebuilt when it or the oracle source is newer)."""
    global _oracle
    if _oracle is None:
        src = os.path.join(HERE, "cpp", "oracle_kin.c")
        so = os.path.join(HERE, "cpp", "_oracle_kin.so")
        deps = [src, os.path.join(ROOT, "oracle", "tds_oracle.c"), os.path.join(ROOT, "oracle", "tds_oracle.h")]
        if not (os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"),
                                   "-I" + os.path.join(ROOT, "oracle"), src, "-o", so + ".tmp", "-lm"])
            os.replace(so + ".tmp", so)
        L = ctypes.CDLL(so)
        dp = ctypes.POINTER(ctypes.c_double)
        L.tdso_point_jacobian.restype = ctypes.c_int
        L.tdso_point_jacobian.argtypes = [dp, dp, ctypes.c_int, dp, dp]
        _oracle = L
    return _oracle


def oracle_point_jacobian(model, q, link, point_world):
    """The C oracle's J [3, n_qd] of a world point on `link` at q (fp64, q as given)."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64)
    p = np.ascontiguousarray(point_world, dtype=np.float64)
    J = np.zeros((3, int(m[4])))
    rc = oracle_lib().tdso_point_jacobian(_dp(m), _dp(q), int(link), _dp(p), _dp(J))
    if rc:
        raise RuntimeError(f"tdso_point_jacobian rc={rc}")
    return J


def _args(model, q, links, local):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    lk = np.ascontiguousarray(links, dtype=np.int32).ravel()
    lc = np.ascontiguousarray(local, dtype=np.float64).reshape(-1)
    assert lc.size == 3 * lk.size
    return m, q, lk, lc, lk.size, q.shape[0]


def _check(rc, what):
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def rows(model, K):
    """(rows of xf, of x, of J) for a model and K points."""
    return int(model[1]) * 12, 3 * K, 3 * K * int(model[4])


def kinematics(model, q, links, local):
    """(xf [n, n_links, 12], x [n, K, 3], J [n, K, 3, n_qd]) at q [n, n_q] (rounded to fp32)."""
    m, q, lk, lc, K, n = _args(model, q, links, local)
    nl, nd = int(m[1]), int(m[4])
    xf, x, J = np.zeros((n, nl, 12)), np.zeros((n, K, 3)), np.zeros((n, K, 3, nd))
    _check(lib().tdsemu_kin(_dp(m), m.size, n, _dp(q), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), _dp(xf), _dp(x), _dp(J)),
           "tdsemu_kin")
    return xf, x, J


def kinematics_jvp(model, q, links, local, t_q):
    """d(xf | x | J) along t_q [n, n_q, m]: (dxf [n, n_links, 12, m], dx [n, K, 3, m], dJ [n, K, 3, n_qd, m])."""
    m_, q, lk, lc, K, n = _args(model, q, links, local)
    tq = np.ascontiguousarray(t_q, dtype=np.float64)
    m = tq.shape[2]
    r_xf, r_x, r_J = rows(m_, K)
    out = np.zeros((n, r_xf + r_x + r_J, m))
    _check(lib().tdsemu_kin_jvp(_dp(m_), m_.size, n, _dp(q), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), m, _dp(tq), _dp(out)),
           "tdsemu_kin_jvp")
    nl, nd = int(m_[1]), int(m_[4])
    return (out[:, :r_xf].reshape(n, nl, 12, m), out[:, r_xf:r_xf + r_x].reshape(n, K, 3, m),
            out[:, r_xf + r_x:].reshape(n, K, 3, nd, m))


def kinematics_vjp(model, q, links, local, G_xf, G_x, G_J):
    """g_q [n, n_q] = <G, d(xf | x | J) / dq> for the cotangents G_xf [n, n_links, 12], G_x [n, K, 3], G_J [n, K, 3, n_qd]."""
    m, q, lk, lc, K, n = _args(model, q, links, local)
    G = np.ascontiguousarray(np.concatenate([np.reshape(G_xf, (n, -1)), np.reshape(G_x, (n, -1)), np.reshape(G_J, (n, -1))], axis=1))
    assert G.shape[1] == sum(rows(m, K))
    g = np.zeros((n, int(m[3])))
    _check(lib().tdsemu_kin_vjp(_dp(m), m.size, n, _dp(q), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lc), _dp(G), _dp(g)), "tdsemu_kin_vjp")
    return g
