"""Inverse dynamics on the GPU (DESIGN.md section 7.14): tau = ID(q, qd, qdd) alone (BatchSim.inverse_dynamics_device), its JVP at m = 1
and m = n_in = n_q + 2 n_qd (inverse_dynamics_jvp_device), its VJP (inverse_dynamics_vjp_device), the backward of
tds_b200.autograd.inverse_dynamics, and for context M(q) (mass_matrix_device) and the world-frame step (BatchSim.step_device in fp64 on
the world-frame kernel, MODE_FULL), on Laikago and the humanoid.  CUDA events after a warm-up, median of --reps runs; prints the GPU's
name, power limit and maximum SM clock read in the same run.

    python scripts/bench_inverse_dynamics.py [--n 4096] [--reps 7]
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
    n_in = n_q + 2 * nd
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qd, qdd = rng.normal(size=(n, nd)), rng.normal(size=(n, nd))

    def soa(x, dt=torch.float32):
        t = torch.zeros((x.shape[1], ns), dtype=dt, device=dev)
        t[:, :n] = torch.tensor(x.T, dtype=dt)
        return t
    qs, qds, qdds = soa(q), soa(qd), soa(qdd)
    tau = torch.zeros((nd, ns), dtype=torch.float64, device=dev)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_in=n_in)
    out["ID"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, qdds, tau), reps)
    out["bias_forces"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, None, tau), reps)
    for m in (1, n_in):
        t = [torch.tensor(rng.normal(size=(d * m, ns)), dtype=torch.float64, device=dev) for d in (n_q, nd, nd)]
        tt = torch.zeros((nd * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.inverse_dynamics_jvp_device(qs, qds, qdds, m, *t, None, tt), reps)
        del t, tt
    G = torch.tensor(rng.normal(size=(nd, ns)), dtype=torch.float64, device=dev)
    gs = [torch.zeros((d, ns), dtype=torch.float64, device=dev) for d in (n_q, nd, nd)]
    out["vjp"] = timed(lambda: sim.inverse_dynamics_vjp_device(qs, qds, qdds, G, *gs), reps)
    xt = [torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, qdd)]
    Gt = torch.tensor(rng.normal(size=(n, nd)), dtype=torch.float64, device=dev)

    def bwd():
        xs = [x.clone().requires_grad_(True) for x in xt]
        (tds_b200.autograd.inverse_dynamics(sim, *xs) * Gt).sum().backward()
    out["autograd_backward"] = timed(bwd, reps)
    M = torch.zeros((nd * nd, ns), dtype=torch.float64, device=dev)
    out["mass_matrix"] = timed(lambda: sim.mass_matrix_device(qs, M), reps)
    os.environ["TDS_B200_KERNEL"] = "world"
    step_sim = tds_b200.BatchSim(model, n, precision=1)
    q2, qd2, qo, qdo = qs.clone(), qds.clone(), qs.clone(), qds.clone()
    out["step_world_f64"] = timed(lambda: step_sim.step_device(2, q2, qd2, q_out=qo, qd_out=qdo), reps)
    out["step_kernel"] = step_sim.kernel_name()
    del os.environ["TDS_B200_KERNEL"]
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
