"""TEST INFRASTRUCTURE: ctypes binding of the rigid-body kernel's instances with per-world physical parameters compiled for the host
(tests/cpp/rigid_param_host.cpp, csrc/tds_rigid.cu with PAR).  Used only by the CPU test-suite; the package never loads them."""
import ctypes

import numpy as np

from emu import _dp
from emu_vjp import _load

DEPS = ("tds_rigid.cu", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh")


class Refused(ValueError):
    def __init__(self, rc, reason):
        super().__init__(f"rc={rc}: {reason}")
        self.rc, self.reason = rc, reason


def lib():
    L = _load("rigid_param_host", DEPS)
    dp = ctypes.POINTER(ctypes.c_double)
    ci, vp = ctypes.c_int, ctypes.c_void_p
    L.tdsemu_rigid_par_check.restype = ci
    L.tdsemu_rigid_par_check.argtypes = [dp, ci, ci, vp, ci, dp, ctypes.c_char_p, ci]
    L.tdsemu_rigid_par.restype = ci
    L.tdsemu_rigid_par.argtypes = [dp, ci, dp, ci, dp, dp, ci, ci, vp, dp, dp, dp, dp]
    L.tdsemu_rigid_par_jvp.restype = ci
    L.tdsemu_rigid_par_jvp.argtypes = [dp, ci, dp, ci, dp, dp, ci, ci, vp, dp, ci, dp, dp, dp, dp, dp]
    L.tdsemu_rigid_par_vjp.restype = ci
    L.tdsemu_rigid_par_vjp.argtypes = [dp, ci, dp, ci, dp, dp, ci, ci, vp, dp, dp, dp, dp, dp, ci, ci, dp]
    return L


def _world(desc, state, force, ids, values, dt, gravity, friction, restitution, erp, num_solver_iterations):
    d = np.ascontiguousarray(desc, dtype=np.float64)
    s = np.ascontiguousarray(state, dtype=np.float64)
    n, nb = s.shape[0], d.shape[0]
    f = None if force is None else np.ascontiguousarray(force, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.ascontiguousarray(np.broadcast_to(np.asarray(values if k else np.zeros(0), dtype=np.float64), (n, k)))
    params = np.array([dt, *gravity, friction, restitution, erp, num_solver_iterations], dtype=np.float64)
    return d, s, f, idv, v, params, n, nb, k


def _rc(rc, what):
    if rc == -100:
        raise Refused(rc, "parameter ids rejected")
    if rc:
        raise RuntimeError(f"{what} rc={rc}")


def check(desc, ids, values=None, n=1):
    """The checks of tds_b200_rigid_set_physical_params_host on the host: raises Refused(-2 | -3, reason)."""
    d = np.ascontiguousarray(desc, dtype=np.float64)
    idv = np.ascontiguousarray(list(ids), dtype=np.int32)
    k = idv.size
    v = np.ascontiguousarray(np.broadcast_to(np.asarray(values if values is not None else np.ones(k), dtype=np.float64), (n, k)))
    err = ctypes.create_string_buffer(256)
    rc = lib().tdsemu_rigid_par_check(_dp(d), d.shape[0], k, idv.ctypes.data_as(ctypes.c_void_p), n, _dp(v), err, 256)
    if rc:
        raise Refused(rc, err.value.decode())


def step(desc, state, ids, values, force=None, steps=1, jac_in=False, jac_par=False, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81),
         friction=0.5, restitution=0.0, erp=0.1, num_solver_iterations=1):
    """`steps` steps with parameters ids installed at values [n, k] (or [k]): dict(state [n][nb][13], jac [n][13 nb][16 nb] with jac_in,
    jac_par [n][13 nb][k] with jac_par)."""
    d, s, f, idv, v, params, n, nb, k = _world(desc, state, force, ids, values, dt, gravity, friction, restitution, erp, num_solver_iterations)
    out = np.zeros_like(s)
    ji = np.zeros((n, 13 * nb, 16 * nb)) if jac_in else None
    jp = np.zeros((n, 13 * nb, k)) if jac_par else None
    _rc(lib().tdsemu_rigid_par(_dp(d), nb, _dp(params), n, _dp(s), _dp(f), steps, k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(out),
                               _dp(ji), _dp(jp)), "tdsemu_rigid_par")
    return dict(state=out, jac=ji, jac_par=jp)


def jvp(desc, state, ids, values, t_state=None, t_force=None, t_par=None, force=None, steps=1, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81),
        friction=0.5, restitution=0.0, erp=0.1, num_solver_iterations=1):
    """(state_out [n][nb][13], t_out [n][nb][13][m]) along t_state [n][nb][13][m], t_force [n][nb][3][m], t_par [n][k][m] (each may be
    None)."""
    d, s, f, idv, v, params, n, nb, k = _world(desc, state, force, ids, values, dt, gravity, friction, restitution, erp, num_solver_iterations)
    prep = lambda x: None if x is None else np.ascontiguousarray(x, dtype=np.float64)
    ts, tf, tp = prep(t_state), prep(t_force), prep(t_par)
    m = next(x for x in (ts, tf, tp) if x is not None).shape[-1]
    so, to = np.zeros_like(s), np.zeros((n, nb, 13, m))
    _rc(lib().tdsemu_rigid_par_jvp(_dp(d), nb, _dp(params), n, _dp(s), _dp(f), steps, k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), m,
                                   _dp(ts), _dp(tf), _dp(tp), _dp(so), _dp(to)), "tdsemu_rigid_par_jvp")
    return so, to


def vjp(desc, state, ids, values, g_state_out, force=None, steps=1, tape_cap=4096, chunk=None, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81),
        friction=0.5, restitution=0.0, erp=0.1, num_solver_iterations=1):
    """(g_state [n][nb][13], g_force [n][nb][3], g_par [n][k], stats) of `steps` steps, checkpointed and chunked (chunk worlds per
    launch; None: all) as the device does it.  tape_cap: starting capacity (regrown on overflow).  stats = dict(nodes, cap, reruns)."""
    d, s, f, idv, v, params, n, nb, k = _world(desc, state, force, ids, values, dt, gravity, friction, restitution, erp, num_solver_iterations)
    g = np.ascontiguousarray(g_state_out, dtype=np.float64).reshape(n, nb, 13)
    gs, gf, gp, st = np.zeros((n, nb, 13)), np.zeros((n, nb, 3)), np.zeros((n, max(k, 1))), np.zeros(3)
    _rc(lib().tdsemu_rigid_par_vjp(_dp(d), nb, _dp(params), n, _dp(s), _dp(f), steps, k, idv.ctypes.data_as(ctypes.c_void_p), _dp(v), _dp(g),
                                   _dp(gs), _dp(gf), _dp(gp), int(tape_cap), int(chunk or n), _dp(st)), "tdsemu_rigid_par_vjp")
    return gs, gf, gp[:, :k], dict(nodes=int(st[0]), cap=int(st[1]), reruns=int(st[2]))
