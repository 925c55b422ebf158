"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/wrench_host.cpp - the external-wrench instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag EXT) compiled for the host: the step's q', qd' or qdd with a wrench per point in the three precisions, and
its Jacobian-vector products on dual numbers, with and without installed physical parameters - and of tests/cpp/oracle_wrench.c, the C
oracle's forward dynamics with the reference's f_ext term.  Used only by the CPU test-suite; the package never loads them."""
import ctypes
import os
import subprocess

import numpy as np

from emu import HERE, ROOT, _dp
from emu_contacts import _params
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")
_oracle = None


def lib():
    L = _load("wrench_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_wrench.restype = ci
    L.tdsemu_wrench.argtypes = [dp, ci, dp, dp, ci, ci, ci, ci, dp, dp, dp, ci, vp, dp, ci, vp, dp, dp, dp, dp, dp, ci, dp, dp, dp, dp]
    return L


def oracle_lib():
    """tests/cpp/oracle_wrench.c built next to it (rebuilt when it or the oracle source is newer)."""
    global _oracle
    if _oracle is None:
        src = os.path.join(HERE, "cpp", "oracle_wrench.c")
        so = os.path.join(HERE, "cpp", "_oracle_wrench.so")
        deps = [src, os.path.join(ROOT, "oracle", "tds_oracle.c"), os.path.join(ROOT, "oracle", "tds_oracle.h")]
        if not (os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"),
                                   "-I" + os.path.join(ROOT, "oracle"), src, "-o", so + ".tmp", "-lm"])
            os.replace(so + ".tmp", so)
        L = ctypes.CDLL(so)
        dp = ctypes.POINTER(ctypes.c_double)
        L.tdso_wrench_fd.restype = ctypes.c_int
        L.tdso_wrench_fd.argtypes = [dp, dp, dp, dp, dp, ctypes.c_int, ctypes.c_void_p, dp, dp, dp]
        _oracle = L
    return _oracle


def oracle_fd(model, q, qd, tau, links, local, W, gravity=(0.0, 0.0, -9.81)):
    """The C oracle's qdd [n_qd] of one environment (fp64, as given; tau [n_tau] or None) with wrenches W [K, 6]; None when the oracle
    does not cover the model."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    c = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float64)
    lk = np.ascontiguousarray(links, dtype=np.int32)
    out = np.zeros(int(m[4]))
    rc = oracle_lib().tdso_wrench_fd(_dp(m), _dp(c(q)), _dp(c(qd)), _dp(c(tau)), _dp(c(np.array(gravity))), lk.size,
                                     lk.ctypes.data_as(ctypes.c_void_p), _dp(c(np.reshape(local, -1))), _dp(c(np.reshape(W, -1))), _dp(out))
    return None if rc else out


def _call(model, mode, q, qd, tau, links, local, W, precision, use_pd, env, ids, values, m, t_in, t_W, t_par, kw):
    mo = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64)
    qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd = q.shape[0], int(mo[3]), int(mo[4])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    lk = np.ascontiguousarray(links, dtype=np.int32)
    K = lk.size
    lo = np.ascontiguousarray(np.reshape(local, (K, 3)), dtype=np.float64)
    w = np.ascontiguousarray(np.broadcast_to(np.asarray(W, dtype=np.float64), (n, K, 6))) if K else np.zeros((n, 1, 6))
    qo, qdo, qddo = np.zeros((n, n_q)), np.zeros((n, n_qd)), np.zeros((n, n_qd))
    n_tau = n_qd - (6 if int(mo[2]) else 0)
    cols = n_q + n_qd + ((int(e[0]) + 3) if use_pd else n_tau)
    rows = n_qd if mode == 0 else n_q + n_qd
    ti, tw, tp = (None if x is None else np.ascontiguousarray(x, dtype=np.float64) for x in (t_in, t_W, t_par))
    if ti is not None:
        assert ti.shape == (n, cols, m), (ti.shape, cols, m)
    if tw is not None:
        assert tw.shape == (n, K, 6, m), (tw.shape, K, m)
    tout = np.zeros((n, rows, max(m, 1)))
    rc = lib().tdsemu_wrench(_dp(mo), mo.size, _dp(_params(**kw)), _dp(e), precision, mode, int(use_pd), n, _dp(q), _dp(qd), _dp(t), k,
                             idv.ctypes.data_as(ctypes.c_void_p), _dp(v), K, lk.ctypes.data_as(ctypes.c_void_p), _dp(lo), _dp(w), _dp(qo),
                             _dp(qdo), _dp(qddo), m, _dp(ti), _dp(tw), _dp(tp), _dp(tout))
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"tdsemu_wrench rc={rc}")
    return qo, qdo, qddo, tout


def step_wrench(model, mode, q, qd, tau, links, local, W, precision=1, use_pd=False, env=None, ids=(), values=None, **kw):
    """(q' [n, n_q], qd' [n, n_qd]) in MODE_NOCONTACT / MODE_FULL, or qdd [n, n_qd] in MODE_FD, of one step with the wrenches W [n, K, 6]
    (or [K, 6] for every environment) at the points links [K] / local [K, 3], through the host-compiled EXT value instance of
    `precision` (0 mixed, 1 fp64, 2 fp32); kw: the solver settings of emu.step."""
    qo, qdo, qddo, _ = _call(model, mode, q, qd, tau, links, local, W, precision, use_pd, env, ids, values, 0, None, None, None, kw)
    return qddo if mode == 0 else (qo, qdo)


def step_wrench_jvp(model, mode, q, qd, tau, links, local, W, t_in=None, t_W=None, t_par=None, use_pd=False, env=None, ids=(), values=None,
                    **kw):
    """t_out [n, rows, m] along t_in [n, cols, m], t_W [n, K, 6, m] and t_par [n, k, m] (each may be None) by the dual-number EXT
    instance (rows q' | qd', or qdd in MODE_FD)."""
    m = next(x for x in (t_in, t_W, t_par) if x is not None).shape[-1]
    return _call(model, mode, q, qd, tau, links, local, W, 1, use_pd, env, ids, values, m, t_in, t_W, t_par, kw)[3]
