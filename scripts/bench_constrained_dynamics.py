"""The point-constrained forward dynamics on the GPU (DESIGN.md section 7.21): the value at K = 0 and with four points held in their linear
rows (Laikago's toes, the humanoid's last four leaf links), the JVP at m = 1 and m = n_q, the VJP (constrained_dynamics_jvp_device,
constrained_dynamics_vjp_device), the backward of tds_b200.autograd.constrained_dynamics, and the same qdd and f by hand: inverse_dynamics +
mass_inverse with Lambda^-1 + point_motion + a batched torch.linalg.solve, with the largest differences between the two paths.  CUDA
events after a warm-up, median of --reps runs; prints the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_constrained_dynamics.py [--n 4096] [--reps 7]
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
from bench_mass_inverse import gpu_info, leaves, timed  # noqa: E402


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    lk = [9, 13, 17, 21] if name == "laikago" else leaves(model)
    lc = np.zeros((len(lk), 3))
    K, R = len(lk), 3 * len(lk)
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qd, tau = rng.normal(size=(n, nd)) * 0.5, rng.normal(size=(n, nd)) * 3.0
    soa = lambda x: torch.zeros((x.shape[1], ns), dtype=torch.float32, device=dev).index_copy_(
        1, torch.arange(n, device=dev), torch.tensor(x.T, dtype=torch.float32, device=dev))
    qs, qds, ts = soa(q), soa(qd), soa(tau)
    z = lambda rows: torch.zeros((rows, ns), dtype=torch.float64, device=dev)
    qdd, f = z(nd), z(R)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, points=lk, dims=3)
    out["value_K0"] = timed(lambda: sim.constrained_dynamics_device(qs, qds, ts, None, None, 3, 0.0, qdd), reps)
    out["value"] = timed(lambda: sim.constrained_dynamics_device(qs, qds, ts, lk, lc, 3, 0.0, qdd, f), reps)
    for m in (1, n_q):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), dtype=torch.float64, device=dev)
        tqdd, tf = z(nd * m), z(R * m)
        out[f"jvp_m{m}"] = timed(lambda: sim.constrained_dynamics_jvp_device(qs, qds, ts, lk, lc, 3, 0.0, m, tq, None, None, None, tqdd, tf),
                                 reps)
        del tq, tqdd, tf
    Gq, Gf = (torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (nd, R))
    gq, gqd, gt = z(n_q), z(nd), z(nd)
    out["vjp"] = timed(lambda: sim.constrained_dynamics_vjp_device(qs, qds, ts, lk, lc, 3, 0.0, Gq, Gf, gq, gqd, gt), reps)
    qt, qdt, tt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, tau))
    Gqt = torch.tensor(rng.normal(size=(n, nd)), dtype=torch.float64, device=dev)
    Gft = torch.tensor(rng.normal(size=(n, K, 3)), dtype=torch.float64, device=dev)

    def bwd():
        x, y, w = (t.clone().requires_grad_(True) for t in (qt, qdt, tt))
        a, b = tds_b200.autograd.constrained_dynamics(sim, x, y, w, lk, lc, 3)
        ((a * Gqt).sum() + (b * Gft).sum()).backward()
    out["autograd_backward"] = timed(bwd, reps)
    lin = torch.tensor(np.concatenate([np.arange(6 * k + 3, 6 * k + 6) for k in range(K)]), device=dev)

    def by_hand():
        h = tds_b200.autograd.inverse_dynamics(sim, qt, qdt)
        Mi, Lam = tds_b200.autograd.mass_inverse(sim, qt, lk, lc)
        J, _, drift = tds_b200.autograd.point_motion(sim, qt, qdt, lk, lc)
        Jc, dc = J.reshape(n, 6 * K, nd)[:, lin], drift.reshape(n, 6 * K)[:, lin]
        r = tt.double() - h
        fh = -torch.linalg.solve(Lam[:, lin][:, :, lin], (Jc @ (Mi @ r[..., None]))[..., 0] + dc)
        return (Mi @ (r + (Jc.mT @ fh[..., None])[..., 0])[..., None])[..., 0], fh
    out["by_hand"] = timed(by_hand, reps)
    hq, hf = by_hand()
    sim.constrained_dynamics_device(qs, qds, ts, lk, lc, 3, 0.0, qdd, f)
    torch.cuda.synchronize()
    out["by_hand_max_abs_diff"] = [float((hq - qdd[:, :n].t()).abs().max()), float((hf - f[:, :n].t()).abs().max())]
    out["max_abs"] = [float(hq.abs().max()), float(hf.abs().max())]
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
