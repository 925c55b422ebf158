"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/contacts_host.cpp - the contact-reporting instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag CF) compiled for the host: the step's q', qd' and contact records in the three precisions, and their
Jacobian-vector products on dual numbers, with and without installed physical parameters.  Used only by the CPU test-suite; the package
never loads it."""
import ctypes
import os

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib(name="contacts_host"):
    """contacts_host, or contacts_fp64_host: the same instances with the dual-number ones writing the records' value parts."""
    L = _load(name, DEPS + (() if name == "contacts_host" else (os.path.join("..", "..", "tests", "cpp", "contacts_host.cpp"),)))
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_contacts.restype = ci
    L.tdsemu_contacts.argtypes = [dp, ci, dp, dp, ci, ci, ci, ci, dp, dp, dp, ci, vp, dp, dp, dp, dp, ci, dp, dp, dp]
    return L


def _params(dt=1e-3, gravity=(0.0, 0.0, -9.81), friction=0.5, restitution=0.0, erp=0.2, cfm=1e-5, pgs_iterations=1, keep_all_points=False,
            contact_model=0, spring_k=50000.0, damper_d=5000.0, exponent_n=1.5, v_transition=0.01, hard_contact_condition=True):
    return np.array([dt, *gravity, friction, restitution, erp, cfm, pgs_iterations, int(keep_all_points), contact_model, spring_k,
                     damper_d, exponent_n, v_transition, int(hard_contact_condition)], dtype=np.float64)


def _call(model, mode, q, qd, tau, precision, use_pd, env, ids, values, m, t_in, t_par, kw, name="contacts_host"):
    mo = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64)
    qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd = q.shape[0], int(mo[3]), int(mo[4])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    cap = 10 * 128 + 1
    qo, qdo, C = np.zeros((n, n_q)), np.zeros((n, n_qd)), np.zeros(n * cap)
    n_tau = n_qd - (6 if int(mo[2]) else 0)
    cols = n_q + n_qd + ((int(e[0]) + 3) if use_pd else n_tau)
    ti, tp = (None if x is None else np.ascontiguousarray(x, dtype=np.float64) for x in (t_in, t_par))
    tout = np.zeros(n * (n_q + n_qd + cap) * max(m, 1))
    if ti is not None:
        assert ti.shape == (n, cols, m), (ti.shape, cols, m)
    rc = lib(name).tdsemu_contacts(_dp(mo), mo.size, _dp(_params(**kw)), _dp(e), precision, mode, int(use_pd), n, _dp(q), _dp(qd), _dp(t), k,
                               idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(qo), _dp(qdo), _dp(C), m, _dp(ti), _dp(tp), _dp(tout))
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"tdsemu_contacts rc={rc}")
    return rc, qo, qdo, C, tout, n, n_q + n_qd


def step_contacts(model, mode, q, qd, tau=None, precision=1, use_pd=False, env=None, ids=(), values=None, **kw):
    """(q' [n, n_q], qd' [n, n_qd], C [n, n_pts, 10]) of one step through the host-compiled CF value instance of `precision` (0 mixed,
    1 fp64, 2 fp32); kw: the solver settings of emu.step."""
    npts, qo, qdo, C, _, n, _ = _call(model, mode, q, qd, tau, precision, use_pd, env, ids, values, 0, None, None, kw)
    return qo, qdo, C[:n * 10 * npts].reshape(n, npts, 10)


def step_contacts_jvp(model, mode, q, qd, tau=None, t_in=None, t_par=None, use_pd=False, env=None, ids=(), values=None, **kw):
    """t_out [n, n_q + n_qd + 10 n_pts, m] along t_in [n, cols, m] and t_par [n, k, m] (either may be None) by the dual-number CF
    instance (rows q' | qd' | records)."""
    m = (t_in if t_in is not None else t_par).shape[2]
    npts, _, _, _, tout, n, nqq = _call(model, mode, q, qd, tau, 1, use_pd, env, ids, values, m, t_in, t_par, kw)
    rows = nqq + 10 * npts
    return tout[:n * rows * m].reshape(n, rows, m)


def step_contacts_fp64(model, mode, q, qd, tau=None, use_pd=False, env=None, ids=(), values=None, **kw):
    """The records [n, n_pts, 10] in fp64 from the dual-number instance's value parts (inputs rounded to fp32 as loaded, nothing rounded
    after): the function whose derivative step_contacts_jvp computes."""
    mo = np.asarray(model, dtype=np.float64)
    n = np.atleast_2d(q).shape[0]
    n_tau = int(mo[4]) - (6 if int(mo[2]) else 0)
    cols = int(mo[3]) + int(mo[4]) + ((int(env[0]) + 3) if use_pd else n_tau)
    npts, _, _, _, tout, n, nqq = _call(model, mode, q, qd, tau, 1, use_pd, env, ids, values, 1, np.zeros((n, cols, 1)), None, kw,
                                        name="contacts_fp64_host")
    rows = nqq + 10 * npts
    return tout[:n * rows].reshape(n, rows)[:, nqq:].reshape(n, npts, 10)
