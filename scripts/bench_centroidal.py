"""The centroidal query on the GPU (DESIGN.md section 7.16): the body record, A_G and its bias (BatchSim.centroidal_device), its JVP at
m = 1 and m = n_in = n_q + n_qd (centroidal_jvp_device), its VJP (centroidal_vjp_device), the backward of tds_b200.autograd.centroidal,
and for context M(q) (mass_matrix_device) and ID (inverse_dynamics_device), on Laikago and the humanoid.  CUDA events after a warm-up,
median of --reps runs; prints the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_centroidal.py [--n 4096] [--reps 7]
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
from bench_mass_matrix import gpu_info, timed  # noqa: E402


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    n_in = n_q + nd
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qd = rng.normal(size=(n, nd))

    def soa(x, dt=torch.float32):
        t = torch.zeros((x.shape[1], ns), dtype=dt, device=dev)
        t[:, :n] = torch.tensor(x.T, dtype=dt)
        return t
    qs, qds = soa(q), soa(qd)
    z = lambda rows: torch.zeros((rows, ns), dtype=torch.float64, device=dev)
    com, A, bias = z(10), z(6 * nd), z(6)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_in=n_in)
    out["centroidal"] = timed(lambda: sim.centroidal_device(qs, qds, com, A, bias), reps)
    for m in (1, n_in):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), dtype=torch.float64, device=dev)
        tqd = torch.tensor(rng.normal(size=(nd * m, ns)), dtype=torch.float64, device=dev)
        outs = z(10 * m), z(6 * nd * m), z(6 * m)
        out[f"jvp_m{m}"] = timed(lambda: sim.centroidal_jvp_device(qs, qds, m, tq, tqd, None, *outs), reps)
        del tq, tqd, outs
    G = [torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (10, 6 * nd, 6)]
    g_q, g_qd = z(n_q), z(nd)
    out["vjp"] = timed(lambda: sim.centroidal_vjp_device(qs, qds, *G, g_q, g_qd), reps)
    qt, qdt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd))
    Gc, GA = torch.tensor(rng.normal(size=(n, 3)), device=dev), torch.tensor(rng.normal(size=(n, 6, nd)), device=dev)

    def bwd():
        a, b = qt.clone().requires_grad_(True), qdt.clone().requires_grad_(True)
        _, c, _, Am, bi = tds_b200.autograd.centroidal(sim, a, b)
        ((c * Gc).sum() + (Am * GA).sum() + bi.sum()).backward()
    out["autograd_backward"] = timed(bwd, reps)
    M = z(nd * nd)
    out["mass_matrix"] = timed(lambda: sim.mass_matrix_device(qs, M), reps)
    tau = z(nd)
    out["inverse_dynamics"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, None, tau), reps)
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
