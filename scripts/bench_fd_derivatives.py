"""The derivatives of the forward dynamics on the GPU (DESIGN.md section 7.24): qdd, d qdd / dq, d qdd / dqd and d qdd / dtau in one call
(BatchSim.forward_dynamics_derivatives_device), their JVP at m = 1 and m = n_q + 2 n_qd, their VJP, the backward of
tds_b200.autograd.forward_dynamics_derivatives, the product kernel's share of the value's kernel time (torch.profiler, in a run of its
own after the timings), and in the same run the two routes the query replaces, each timed and compared with it:
  1. constrained_dynamics_jvp_device (K = 0) at m = n_q + 2 n_qd along the unit tangents of q (its own coordinates), qd and tau, then the
     map of the q columns to velocity coordinates through dq_dt (a batched product on the device; dq_dt itself on the host, untimed);
  2. constrained_dynamics_device -> qdd rounded to fp32 -> inverse_dynamics_derivatives_device -> mass_inverse_device -> torch.bmm; its
     deviation shows the error of evaluating d tau / dq at the fp32-rounded qdd.
On Laikago and the humanoid.  CUDA events after a warm-up, median of --reps runs; prints the GPU's name, power limit and maximum SM clock
read in the same run.

    python scripts/bench_fd_derivatives.py [--n 4096] [--reps 7]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tds_b200  # noqa: E402
from tds_b200.model import fixture_path, load_model  # noqa: E402
from bench_dynamics_derivatives import dq_dt_tangents, gpu_info, timed  # noqa: E402


def product_share(fn, iters=5):
    """Share of the product kernel (fdd_product_kernel) in the kernel time of fn, from torch.profiler's CUDA activities."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total = prod = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if ev.key.startswith("cuda") or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        total += t
        if "fdd_product_kernel" in ev.key:
            prod += t
    return dict(product_us_per_call=prod / iters, kernels_us_per_call=total / iters, share=prod / total if total else float("nan"))


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    nn = nd * nd
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    q = q.astype(np.float32).astype(np.float64)
    qd, tau = rng.normal(size=(n, nd)) * 0.5, rng.normal(size=(n, nd)) * 3.0

    def soa(x, dt=torch.float32):
        o = torch.zeros((x.shape[1], ns), dtype=dt, device=dev)
        o[:, :n] = torch.tensor(x.T, dtype=dt)
        return o
    z64 = lambda r: torch.zeros((r, ns), dtype=torch.float64, device=dev)
    qs, qds, taus = soa(q), soa(qd), soa(tau)
    QDD, A, B, C = z64(nd), z64(nn), z64(nn), z64(nn)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd)
    value = lambda: sim.forward_dynamics_derivatives_device(qs, qds, taus, QDD, A, B, C)
    out["value"] = timed(value, reps)
    cq = z64(nd)
    out["constrained_dynamics_K0"] = timed(lambda: sim.constrained_dynamics_device(qs, qds, taus, None, None, 3, 0.0, cq), reps)
    DA, DB = z64(nn), z64(nn)
    q32 = torch.zeros((nd, ns), dtype=torch.float32, device=dev)   # (a qdd input, built outside the timed window)
    out["inverse_dynamics_derivatives"] = timed(lambda: sim.inverse_dynamics_derivatives_device(qs, qds, q32, DA, DB), reps)
    n_in = n_q + 2 * nd
    for m in (1, n_in):
        t = torch.tensor(rng.normal(size=(n_in * m, ns)), dtype=torch.float64, device=dev).view(n_in, m, ns)
        tq, tqd, tt = (t[a:b].reshape(-1, ns).contiguous() for a, b in ((0, n_q), (n_q, n_q + nd), (n_q + nd, n_in)))
        T4 = [z64(nd * m)] + [z64(nn * m) for _ in range(3)]
        out[f"jvp_m{m}"] = timed(lambda: sim.forward_dynamics_derivatives_jvp_device(qs, qds, taus, m, tq, tqd, tt, None, *T4), reps)
        del t, tq, tqd, tt, T4
    G = [torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (nd, nn, nn, nn)]
    gq, gqd, gt = z64(n_q), z64(nd), z64(nd)
    out["vjp"] = timed(lambda: sim.forward_dynamics_derivatives_vjp_device(qs, qds, taus, *G, gq, gqd, gt), reps)
    qt, qdt, tt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, tau))
    Gt = [torch.tensor(rng.normal(size=s), dtype=torch.float64, device=dev) for s in ((n, nd), (n, nd, nd), (n, nd, nd), (n, nd, nd))]

    def bwd():
        x, y, w = (v.clone().requires_grad_(True) for v in (qt, qdt, tt))
        outs = tds_b200.autograd.forward_dynamics_derivatives(sim, x, y, w)
        sum((o * g).sum() for o, g in zip(outs, Gt)).backward()
    out["autograd_backward"] = timed(bwd, reps)

    value()
    torch.cuda.synchronize()
    sq = lambda X: X[:, :n].view(nd, nd, n).permute(2, 0, 1)
    new = dict(dq=sq(A).clone(), dqd=sq(B).clone(), dtau=sq(C).clone())
    out["max_abs"] = {k: float(v.abs().max()) for k, v in new.items()}

    # route 1: the constrained dynamics' JVP along unit tangents, the q columns mapped through dq_dt (T formed beforehand, untimed)
    m = n_in
    TQ, TQD, TT = z64(n_q * m), z64(nd * m), z64(nd * m)
    TQ.view(n_q, m, ns)[torch.arange(n_q), torch.arange(n_q), :] = 1.0
    TQD.view(nd, m, ns)[torch.arange(nd), n_q + torch.arange(nd), :] = 1.0
    TT.view(nd, m, ns)[torch.arange(nd), n_q + nd + torch.arange(nd), :] = 1.0
    T = dq_dt_tangents(model, q, dev).view(n_q, nd, n).permute(2, 0, 1).contiguous()   # [n, n_q, n_qd]
    dqdd = z64(nd * m)
    r1 = {}

    def route1():
        sim.constrained_dynamics_jvp_device(qs, qds, taus, None, None, 3, 0.0, m, TQ, TQD, TT, None, dqdd)
        J = dqdd[:, :n].view(nd, m, n).permute(2, 0, 1)                                  # [n, n_qd, n_q + 2 n_qd]
        r1["dq"] = torch.bmm(J[:, :, :n_q], T)
        r1["dqd"] = J[:, :, n_q:n_q + nd]
        r1["dtau"] = J[:, :, n_q + nd:]
    out["route1_constrained_dynamics_jvp_and_map"] = timed(route1, reps)
    out["route1_max_abs_diff"] = {k: float((new[k] - r1[k]).abs().max()) for k in new}

    # route 2: four queries; d tau / dq at the fp32-rounded qdd
    r2 = {}
    Mi = z64(nn)

    def route2():
        sim.constrained_dynamics_device(qs, qds, taus, None, None, 3, 0.0, cq)
        q32.copy_(cq)
        sim.inverse_dynamics_derivatives_device(qs, qds, q32, DA, DB)
        sim.mass_inverse_device(qs, None, None, Mi)
        M = sq(Mi)
        r2["dq"] = -torch.bmm(M, sq(DA))
        r2["dqd"] = -torch.bmm(M, sq(DB))
        r2["dtau"] = M
    out["route2_four_queries_and_bmm"] = timed(route2, reps)
    out["route2_max_abs_diff"] = {k: float((new[k] - r2[k]).abs().max()) for k in new}
    out["product_kernel"] = product_share(value)
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
