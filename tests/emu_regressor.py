"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/regressor_host.cpp - the regressor instances of the product's generic step kernel
(csrc/tds_stepw.cu, template flags INV and REG) compiled for the host: the joint-torque regressor Y [n_qd, n_pi] and the energy
regressors yT, yV [n_pi] in fp64, their Jacobian-vector products and their vector-Jacobian product.  Used only by the CPU test-suite; the
package never loads it."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h")
GRAVITY = (0.0, 0.0, -9.81)


def lib():
    L = _load("regressor_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci = ctypes.c_int
    L.tdsemu_regressor.restype = ci
    L.tdsemu_regressor.argtypes = [dp, ci, ci, dp, dp, dp, dp, ctypes.c_double, dp, dp, dp]
    L.tdsemu_regressor_jvp.restype = ci
    L.tdsemu_regressor_jvp.argtypes = [dp, ci, ci, dp, dp, dp, dp, ci, dp, dp]
    L.tdsemu_regressor_vjp.restype = ci
    L.tdsemu_regressor_vjp.argtypes = [dp, ci, ci, dp, dp, dp, dp, dp, dp]
    return L


def n_pi(model):
    return 12 * int(model[1]) + 10


def rows(model):
    """(rows of Y, of yT, of yV)."""
    return int(model[4]) * n_pi(model), n_pi(model), n_pi(model)


def _args(model, q, qd, qdd, gravity):
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(np.atleast_2d(q), dtype=np.float64)
    c = lambda x: None if x is None else np.ascontiguousarray(np.atleast_2d(x), dtype=np.float64)
    return m, q, c(qd), c(qdd), np.ascontiguousarray(gravity, dtype=np.float64), q.shape[0]


def _check(rc, what):
    if rc < 0:
        raise RuntimeError(f"{what} rc={rc}")


def regressor(model, q, qd=None, qdd=None, gravity=GRAVITY, fill=0.0, concat=False):
    """(Y [n, n_qd, n_pi], yT [n, n_pi], yV [n, n_pi]) at q [n, n_q], qd and qdd [n, n_qd] (None: zero; all rounded to fp32), the output
    buffers filled with `fill` before the launch; or the concatenated rows [n, rows]."""
    m, q, qd, qdd, g, n = _args(model, q, qd, qdd, gravity)
    nd, npi = int(m[4]), n_pi(m)
    Y, yT, yV = np.zeros((n, nd, npi)), np.zeros((n, npi)), np.zeros((n, npi))
    _check(lib().tdsemu_regressor(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(g), float(fill), _dp(Y), _dp(yT), _dp(yV)),
           "tdsemu_regressor")
    if concat:
        return np.concatenate([Y.reshape(n, -1), yT, yV], axis=1)
    return Y, yT, yV


def split(out, model):
    """(Y [n, n_qd, n_pi, ...], yT [n, n_pi, ...], yV [n, n_pi, ...]) from the concatenated rows [n, rows, ...]."""
    n, tail = out.shape[0], out.shape[2:]
    r_Y, r_pi, _ = rows(model)
    return out[:, :r_Y].reshape((n, int(model[4]), r_pi) + tail), out[:, r_Y:r_Y + r_pi], out[:, r_Y + r_pi:]


def regressor_jvp(model, q, t_in, qd=None, qdd=None, gravity=GRAVITY):
    """The concatenated rows' derivatives [n, rows, m] along t_in [n, n_q + 2 n_qd, m] (q | qd | qdd tangents)."""
    m_, q, qd, qdd, g, n = _args(model, q, qd, qdd, gravity)
    ti = np.ascontiguousarray(t_in, dtype=np.float64)
    m = ti.shape[2]
    out = np.zeros((n, sum(rows(m_)), m))
    _check(lib().tdsemu_regressor_jvp(_dp(m_), m_.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(g), m, _dp(ti), _dp(out)), "tdsemu_regressor_jvp")
    return out


def regressor_vjp(model, q, G, qd=None, qdd=None, gravity=GRAVITY):
    """g [n, n_q + 2 n_qd] = <G, d(Y | yT | yV) / d(q | qd | qdd)> for the concatenated cotangent G [n, rows]."""
    m, q, qd, qdd, g_, n = _args(model, q, qd, qdd, gravity)
    G = np.ascontiguousarray(G, dtype=np.float64)
    assert G.shape == (n, sum(rows(m)))
    g = np.zeros((n, int(m[3]) + 2 * int(m[4])))
    _check(lib().tdsemu_regressor_vjp(_dp(m), m.size, n, _dp(q), _dp(qd), _dp(qdd), _dp(g_), _dp(G), _dp(g)), "tdsemu_regressor_vjp")
    return g
