"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/centroidal_host.cpp - the centroidal instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flag CEN) compiled for the host: the body record com [10], the centroidal momentum matrix A [6, n_qd] and its
bias [6] in fp64, their Jacobian-vector products and their vector-Jacobian product, with and without installed physical parameters.
Used only by the CPU test-suite; the package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")


def lib():
    L = _load("centroidal_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_centroidal.restype = ci
    L.tdsemu_centroidal.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, dp]
    L.tdsemu_centroidal_jvp.restype = ci
    L.tdsemu_centroidal_jvp.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, ci, dp, dp, dp]
    L.tdsemu_centroidal_vjp.restype = ci
    L.tdsemu_centroidal_vjp.argtypes = [dp, ci, ci, dp, dp, ci, vp, dp, dp, dp]
    return L


def rows(model):
    """Rows of the concatenated outputs com | A | bias."""
    return 16 + 6 * int(model[4])


def split(out, nd):
    """com [n, 10], A [n, 6, n_qd], bias [n, 6] (trailing axes kept) from the concatenated rows [n, rows, ...]."""
    n = out.shape[0]
    return out[:, :10], out[:, 10:10 + 6 * nd].reshape((n, 6, nd) + out.shape[2:]), out[:, 10 + 6 * nd:]


def _args(model, q, qd, ids, values):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    n = q.shape[0]
    qd = None if qd is None else np.ascontiguousarray(np.atleast_2d(qd), dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.zeros((n, max(k, 1))) if values is None else np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (n, k)))
    return m, q, qd, idv, k, n, v


def _check(rc, what):
    if rc == -100:
        raise ValueError("parameter ids rejected")
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def centroidal(model, q, qd=None, ids=(), values=None, concat=False):
    """(com [n, 10], A [n, 6, n_qd], bias [n, 6]) at q [n, n_q], qd [n, n_qd] (None: zero; rounded to fp32) with the parameters `ids`
    installed at `values`; or the concatenated rows [n, rows]."""
    m, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    out = np.zeros((n, rows(m)))
    _check(lib().tdsemu_centroidal(_dp(m), m.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(out)),
           "tdsemu_centroidal")
    return out if concat else split(out, int(m[4]))


def centroidal_jvp(model, q, qd=None, t_in=None, t_par=None, ids=(), values=None):
    """The concatenated rows' derivatives [n, rows, m] along t_in [n, n_q + n_qd, m] (q | qd tangents) and t_par [n, k, m] (either None)."""
    m_, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    ti = None if t_in is None else np.ascontiguousarray(t_in, dtype=np.float64)
    tp = None if t_par is None else np.ascontiguousarray(t_par, dtype=np.float64)
    m = (ti if ti is not None else tp).shape[2]
    out = np.zeros((n, rows(m_), m))
    _check(lib().tdsemu_centroidal_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m, _dp(ti),
                                       _dp(tp), _dp(out)), "tdsemu_centroidal_jvp")
    return out


def centroidal_vjp(model, q, qd, G, ids=(), values=None):
    """(g_in [n, n_q + n_qd], g_par [n, k]) = <G, d(com | A | bias)> for the concatenated cotangent G [n, rows]."""
    m, q, qd, idv, k, n, v = _args(model, q, qd, ids, values)
    n_in = int(m[3]) + int(m[4])
    G = np.ascontiguousarray(G, dtype=np.float64)
    g = np.zeros((n, n_in + k))
    _check(lib().tdsemu_centroidal_vjp(_dp(m), m.size, n, _dp(q), _dp(qd), k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(G), _dp(g)),
           "tdsemu_centroidal_vjp")
    return g[:, :n_in], g[:, n_in:]
