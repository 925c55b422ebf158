"""TEST INFRASTRUCTURE: ctypes binding of the reverse-mode (taping) instances of the product's kernels compiled for the host -
tests/cpp/stepw_vjp_host.cpp (csrc/tds_stepw.cu) and tests/cpp/rigid_vjp_host.cpp (csrc/tds_rigid.cu).  The companions of tests/emu.py
(the float / double / dual-number instances of the same sources); used only by the CPU test-suite, the package never loads them."""
import ctypes
import os
import subprocess

import numpy as np

from emu import CSRC, HERE, ROOT, _dp

_libs = {}


def _load(name, deps):
    """Compile tests/cpp/<name>.cpp to tests/cpp/_<name>.so when a source is newer, and load it."""
    if name not in _libs:
        src = os.path.join(HERE, "cpp", name + ".cpp")
        so = os.path.join(HERE, "cpp", "_" + name + ".so")
        deps = [src] + [os.path.join(CSRC, f) for f in deps]
        if not (os.path.exists(so) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)):
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-w", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                                   "-I/usr/local/cuda/include", src, "-o", so + ".tmp"])
            os.replace(so + ".tmp", so)
        _libs[name] = ctypes.CDLL(so)
    return _libs[name]


def lib_stepw():
    L = _load("stepw_vjp_host", ("tds_stepw.cu", "tds_wcommon.cuh", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh", "tds_model.h", "tds_types.h"))
    dp = ctypes.POINTER(ctypes.c_double)
    L.tdsemu_stepw_vjp.restype = ctypes.c_int
    L.tdsemu_stepw_vjp.argtypes = [dp, ctypes.c_int, dp, dp, ctypes.c_int, ctypes.c_int, ctypes.c_int] + [dp] * 5 + [ctypes.c_int, dp]
    return L


def lib_rigid():
    L = _load("rigid_vjp_host", ("tds_rigid.cu", "tds_math.cuh", "tds_dual.cuh", "tds_tape.cuh"))
    dp = ctypes.POINTER(ctypes.c_double)
    L.tdsemu_rigid_vjp.restype = ctypes.c_int
    L.tdsemu_rigid_vjp.argtypes = [dp, ctypes.c_int, dp, ctypes.c_int, dp, dp, ctypes.c_int, dp, dp, dp, ctypes.c_int, dp]
    return L


def step_vjp(model, mode, q, qd, g_out, tau=None, use_pd=False, env=None, tape_cap=1 << 16, dt=1e-3, gravity=(0.0, 0.0, -9.81),
             friction=0.5, restitution=0.0, erp=0.2, cfm=1e-5, pgs_iterations=1, keep_all_points=False, contact_model=0,
             spring_k=50000.0, damper_d=5000.0, exponent_n=1.5, v_transition=0.01, hard_contact_condition=True):
    """g_out [n, rows] -> g_in [n, cols] = g_out^T d(step) / d(inputs) by the taping instance of the host-compiled kernel (rows and
    columns as for emu.step(..., jacobian=True)).  tape_cap: starting tape capacity in nodes per lane (the run regrows it).
    Returns (g_in, stats): stats = dict(nodes=[n] recorded nodes per lane, cap=final capacity, reruns=overflow reruns)."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64); qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd = q.shape[0], int(m[3]), int(m[4])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    params = np.array([dt, *gravity, friction, restitution, erp, cfm, pgs_iterations, int(keep_all_points), contact_model, spring_k,
                       damper_d, exponent_n, v_transition, int(hard_contact_condition)], dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    n_tau = n_qd - (6 if int(m[2]) else 0)
    rows = n_qd if mode == 0 else n_q + n_qd
    cols = n_q + n_qd + ((int(e[0]) + 3) if use_pd else n_tau)
    g = np.ascontiguousarray(g_out, dtype=np.float64)
    assert g.shape == (n, rows), (g.shape, rows)
    g_in = np.zeros((n, cols))
    stats = np.zeros(n + 2)
    rc = lib_stepw().tdsemu_stepw_vjp(_dp(m), m.size, _dp(params), _dp(e), mode, int(use_pd), n, _dp(q), _dp(qd), _dp(t), _dp(g),
                                      _dp(g_in), int(tape_cap), _dp(stats))
    if rc < 0:
        raise RuntimeError(f"tdsemu_stepw_vjp rc={rc}")
    return g_in, dict(nodes=stats[:n].astype(np.int64), cap=int(stats[n]), reruns=int(stats[n + 1]))


def rigid_vjp(desc, state, g_state_out, force=None, steps=1, tape_cap=4096, dt=1.0 / 60.0, gravity=(0.0, 0.0, -9.81), friction=0.5,
              restitution=0.0, erp=0.1, num_solver_iterations=1):
    """(g_state [n][n_bodies][13], g_force [n][n_bodies][3], stats) of `steps` World::step calls by the taping instance of the
    host-compiled rigid-body kernel, checkpointed one step at a time.  stats = dict(nodes=longest tape of a step, cap, reruns)."""
    d = np.ascontiguousarray(desc, dtype=np.float64)
    s = np.ascontiguousarray(state, dtype=np.float64)
    n, nb = s.shape[0], d.shape[0]
    f = None if force is None else np.ascontiguousarray(force, dtype=np.float64)
    g = np.ascontiguousarray(g_state_out, dtype=np.float64).reshape(n, nb, 13)
    params = np.array([dt, *gravity, friction, restitution, erp, num_solver_iterations], dtype=np.float64)
    gs, gf, st = np.zeros((n, nb, 13)), np.zeros((n, nb, 3)), np.zeros(3)
    rc = lib_rigid().tdsemu_rigid_vjp(_dp(d), nb, _dp(params), n, _dp(s), _dp(f), steps, _dp(g), _dp(gs), _dp(gf), int(tape_cap), _dp(st))
    if rc:
        raise RuntimeError(f"tdsemu_rigid_vjp rc={rc}")
    return gs, gf, dict(nodes=int(st[0]), cap=int(st[1]), reruns=int(st[2]))
