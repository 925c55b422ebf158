"""TEST INFRASTRUCTURE: ctypes binding of tests/cpp/_team_host.so - the table-driven tree kernels (csrc/tds_team_step.cuh run by
the lane-team mapping of csrc/tds_stept.cu and the role-warp mapping of csrc/tds_stepr.cu) compiled for the host, see
tests/cpp/team_host.cpp.  Used only by the CPU test-suite to execute the kernel SOURCE without a GPU; the package never loads it."""
import ctypes
import os
import subprocess

import numpy as np

from emu import CSRC, HERE, ROOT, _dp

SO = os.path.join(HERE, "cpp", "_team_host.so")
SRC = os.path.join(HERE, "cpp", "team_host.cpp")
DEPS = [SRC] + [os.path.join(CSRC, f) for f in ("tds_team.h", "tds_team_step.cuh", "tds_stept.cu", "tds_stepr.cu", "tds_wcommon.cuh",
                                                 "tds_math.cuh", "tds_model.h", "tds_types.h")]
LANE_TEAM, ROLE_WARPS = 0, 1
MAPS = {"team": LANE_TEAM, "role": ROLE_WARPS}
_lib = None


def build():
    if os.path.exists(SO) and all(os.path.getmtime(d) <= os.path.getmtime(SO) for d in DEPS):
        return
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-w", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           "-I/usr/local/cuda/include", SRC, "-o", SO + ".tmp"])
    os.replace(SO + ".tmp", SO)


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(SO)
        dp = ctypes.POINTER(ctypes.c_double)
        L.tdsemu_team_step.restype = ctypes.c_int
        L.tdsemu_team_step.argtypes = [dp, ctypes.c_int, dp, dp] + [ctypes.c_int] * 7 + [dp] * 10
        L.tdsemu_team_info.restype = ctypes.c_int
        L.tdsemu_team_info.argtypes = [dp, ctypes.c_int, dp, dp]
        _lib = L
    return _lib


def env_vector(model, n_act, start_link, kp, kd, max_force, action_limit, poses, reward_kind=0, auto_reset=False, reset_q=None):
    """The env array of tdsemu_team_step / tdsemu_team_info: action k drives the k-th non-fixed link at or after start_link
    (from link 0 on a floating base), as tds_b200_set_env maps it."""
    n_q = int(model[3])
    rq = np.zeros(n_q) if reset_q is None else np.asarray(reset_q, dtype=np.float64)
    return np.ascontiguousarray(np.concatenate([[n_act, start_link, kp, kd, max_force, action_limit, reward_kind, float(auto_reset)],
                                                np.asarray(poses, dtype=np.float64)[:n_act], rq]), dtype=np.float64)


def step(model, mode, q, qd, tau=None, map="role", precision=1, smem=True, lane_by_lane=False, force_or=False, descending=False,
         use_pd=False, env=None, dt=1e-3, gravity=(0.0, 0.0, -9.81), friction=0.5, restitution=0.0, erp=0.2, cfm=1e-5,
         pgs_iterations=1, keep_all_points=False):
    """One step of every row of q / qd through the host-compiled tree kernel `map` ("team": lane teams, "role": role warps).
    State is carried in fp32 as on the device; tau holds the joint torques (without the base's) or, with use_pd, the actions.
    Returns dict(q, qd, qdd, reward, done, contact_dist [n][n_cand], link_xf [n][n_links][12])."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    q = np.ascontiguousarray(q, dtype=np.float64); qd = np.ascontiguousarray(qd, dtype=np.float64)
    n, n_q, n_qd, n_links = q.shape[0], int(m[3]), int(m[4]), int(m[1])
    t = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    params = np.array([dt, *gravity, friction, restitution, erp, cfm, pgs_iterations, int(keep_all_points)], dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    out = dict(q=np.zeros((n, n_q)), qd=np.zeros((n, n_qd)), qdd=np.zeros((n, n_qd)), reward=np.zeros(n), done=np.zeros(n))
    cd = np.zeros(n * 48)
    xf = np.zeros((n, n_links, 12))
    flags = int(force_or) | (int(lane_by_lane) << 1) | (int(descending) << 2)
    rc = lib().tdsemu_team_step(_dp(m), m.size, _dp(params), _dp(e), MAPS[map], precision, int(smem), mode, int(use_pd), flags, n,
                                _dp(q), _dp(qd), _dp(t), _dp(out["q"]), _dp(out["qd"]), _dp(out["qdd"]), _dp(out["reward"]),
                                _dp(out["done"]), _dp(cd), _dp(xf))
    if rc < 0:
        raise RuntimeError(f"tdsemu_team_step rc={rc}")
    out["contact_dist"] = cd[:n * rc].reshape(n, rc)
    out["link_xf"] = xf
    return out


def info(model, env=None):
    """tds_build_team's verdict on a model and a summary of its partition (tests/cpp/team_host.cpp: tdsemu_team_info)."""
    m = np.ascontiguousarray(model, dtype=np.float64)
    e = None if env is None else np.ascontiguousarray(env, dtype=np.float64)
    o = np.zeros(78)
    rc = lib().tdsemu_team_info(_dp(m), m.size, _dp(e), _dp(o))
    if rc:
        raise RuntimeError(f"tdsemu_team_info: model rejected rc={rc}")
    n_cand = int(o[14])
    return dict(rc=int(o[0]), n_trunk=int(o[1]), n_loc=o[2:6].astype(int), n_od=o[6:10].astype(int), n_att=int(o[10]),
                n_acc=int(o[11]), n_xw_team=int(o[12]), n_xw_lane=int(o[13]), n_cand=n_cand, trunk_internal=int(o[15]),
                own_internal=int(o[16]), kmax=int(o[17]), floating=bool(o[18]), dropped_subtrees=int(o[19]),
                team_tile_bytes=o[20:23].astype(int), role_tile_bytes=o[23:26].astype(int), subtrees=o[26:30].astype(int),
                cand_owner=o[30:30 + n_cand].astype(int))
