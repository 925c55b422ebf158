"""The derivatives of the inverse dynamics on the GPU (DESIGN.md section 7.23): d tau / dq and d tau / dqd in one call
(BatchSim.inverse_dynamics_derivatives_device), their JVP at m = 1 and m = n_q + 2 n_qd (inverse_dynamics_derivatives_jvp_device), their
VJP, the backward of tds_b200.autograd.inverse_dynamics_derivatives, and in the same run the route they replace: inverse_dynamics_jvp_device
at m = n_q + n_qd along the unit tangents of q (in its own coordinates) and qd, then the map of the q columns to velocity coordinates
through dq_dt (a batched product on the device; dq_dt itself is evaluated on the host beforehand, untimed), plus the value tau itself, on Laikago and the humanoid.  CUDA events after a warm-up, median of --reps runs; prints the GPU's name, power
limit and maximum SM clock read in the same run, and the largest difference between the two routes.

    python scripts/bench_dynamics_derivatives.py [--n 4096] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tds_b200  # noqa: E402
from tds_b200.model import fixture_path, load_model  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()                                   # warm-up (module load, scratch buffers)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), max_ms=float(np.max(ts)))


def dq_dt_tangents(model, q, dev):
    """t_q [n_q * nd, n] float64 CUDA tensor: the unit velocities e_k in q's coordinates (DESIGN.md section 7.23) by the tests' dq_dt
    (a floating base's quaternion rate 1/2 q_b (x) (e, 0) and position rate R_b e, a spherical joint's 1/2 q (x) (e, 0), a REVOLUTE_AXIS
    joint's |axis|, else 1), evaluated per environment on the host."""
    import sys as _s
    _s.path.insert(0, os.path.join(ROOT, "tests"))
    from test_point_motion_on_host import dq_dt
    n, nd = q.shape[0], int(model[4])
    t = np.stack([np.stack([dq_dt(model, x, e) for e in np.eye(nd)], axis=1) for x in q])   # [n, n_q, nd]
    return torch.tensor(t.reshape(n, -1).T.copy(), dtype=torch.float64, device=dev)


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    q = q.astype(np.float32).astype(np.float64)
    qd, qdd = rng.normal(size=(n, nd)), rng.normal(size=(n, nd))

    def soa(x, dt=torch.float32):
        o = torch.zeros((x.shape[1], ns), dtype=dt, device=dev)
        o[:, :n] = torch.tensor(x.T, dtype=dt)
        return o
    qs, qds, qdds = soa(q), soa(qd), soa(qdd)
    nn = nd * nd
    A, B = (torch.zeros((nn, ns), dtype=torch.float64, device=dev) for _ in range(2))
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd)
    out["derivatives"] = timed(lambda: sim.inverse_dynamics_derivatives_device(qs, qds, qdds, A, B), reps)
    tau = torch.zeros((nd, ns), dtype=torch.float64, device=dev)
    out["tau"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, qdds, tau), reps)
    n_in = n_q + 2 * nd
    for m in (1, n_in):
        t = torch.tensor(rng.normal(size=(n_in * m, ns)), dtype=torch.float64, device=dev).view(n_in, m, ns)
        tq, tqd, tqdd = (t[a:b].reshape(-1, ns).contiguous() for a, b in ((0, n_q), (n_q, n_q + nd), (n_q + nd, n_in)))
        tA, tB = (torch.zeros((nn * m, ns), dtype=torch.float64, device=dev) for _ in range(2))
        out[f"jvp_m{m}"] = timed(lambda: sim.inverse_dynamics_derivatives_jvp_device(qs, qds, qdds, m, tq, tqd, tqdd, None, tA, tB), reps)
        del t, tq, tqd, tqdd, tA, tB
    GA, GB = (torch.tensor(rng.normal(size=(nn, ns)), dtype=torch.float64, device=dev) for _ in range(2))
    gq, gqd, gqdd = (torch.zeros((d, ns), dtype=torch.float64, device=dev) for d in (n_q, nd, nd))
    out["vjp"] = timed(lambda: sim.inverse_dynamics_derivatives_vjp_device(qs, qds, qdds, GA, GB, gq, gqd, gqdd), reps)
    qt, qdt, qddt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, qdd))
    Gt = torch.tensor(rng.normal(size=(n, nd, nd)), dtype=torch.float64, device=dev)

    def bwd():
        x, y, z = (v.clone().requires_grad_(True) for v in (qt, qdt, qddt))
        a, b = tds_b200.autograd.inverse_dynamics_derivatives(sim, x, y, z)
        ((a + b) * Gt).sum().backward()
    out["autograd_backward"] = timed(bwd, reps)
    # the route replaced: inverse_dynamics_jvp at m = n_q + n_qd (the unit tangents of q in its own coordinates, then of qd), and the
    # map of the n_q-coordinate columns to velocity coordinates, J_q T with T [n_q, n_qd] = dq_dt(q, e_k), a batched product on the device
    # (T depends on q alone and is formed on the host beforehand, not timed)
    m = n_q + nd
    TQ = torch.zeros((n_q * m, ns), dtype=torch.float64, device=dev)
    TQD = torch.zeros((nd * m, ns), dtype=torch.float64, device=dev)
    TQ.view(n_q, m, ns)[torch.arange(n_q), torch.arange(n_q), :] = 1.0
    TQD.view(nd, m, ns)[torch.arange(nd), n_q + torch.arange(nd), :] = 1.0
    T = dq_dt_tangents(model, q, dev).view(n_q, nd, n).permute(2, 0, 1).contiguous()   # [n, n_q, n_qd]
    dtau = torch.zeros((nd * m, ns), dtype=torch.float64, device=dev)
    res = {}

    def old_route():
        sim.inverse_dynamics_jvp_device(qs, qds, qdds, m, TQ, TQD, None, None, dtau)
        J = dtau[:, :n].view(nd, m, n).permute(2, 0, 1)                                  # [n, n_qd, n_q + n_qd]
        res["dq"] = torch.bmm(J[:, :, :n_q], T)
        res["dqd"] = J[:, :, n_q:]
    out["old_route_inverse_dynamics_jvp_and_map"] = timed(old_route, reps)
    sim.inverse_dynamics_derivatives_device(qs, qds, qdds, A, B)
    torch.cuda.synchronize()
    new_q = A[:, :n].view(nd, nd, n).permute(2, 0, 1)
    new_qd = B[:, :n].view(nd, nd, n).permute(2, 0, 1)
    out["max_abs_diff_dq"] = float((new_q - res["dq"]).abs().max())
    out["max_abs_diff_dqd"] = float((new_qd - res["dqd"]).abs().max())
    out["max_abs_dq"] = float(new_q.abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info())))
    for name in ("laikago", "humanoid"):
        print(json.dumps(case(name, a.n, a.reps)))


if __name__ == "__main__":
    main()
