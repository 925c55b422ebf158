"""Joint-torque and energy regressors on the GPU (DESIGN.md section 7.19): the value (BatchSim.regressor_device) with and without yT and
yV, its JVP at m = 1 (regressor_jvp_device), its VJP (regressor_vjp_device), the backward of tds_b200.autograd.regressor, and for context
ID (inverse_dynamics_device), on Laikago and the humanoid.  CUDA events after a warm-up, median of --reps runs; prints the bytes of Y the
value writes over its time as achieved store bandwidth, and the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_regressor.py [--n 4096] [--reps 7]
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
    ns, n_q, nd, npi = sim.n_stride, sim.n_q, sim.n_qd, sim.n_pi
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
    z = lambda rows: torch.zeros((rows, ns), dtype=torch.float64, device=dev)
    Y, yT, yV = z(nd * npi), z(npi), z(npi)
    y_bytes = 8 * nd * npi * n
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_pi=npi, Y_MB=y_bytes / 1e6)
    out["regressor"] = timed(lambda: sim.regressor_device(qs, qds, qdds, Y, yT, yV), reps)
    out["regressor_Y_only"] = timed(lambda: sim.regressor_device(qs, qds, qdds, Y), reps)
    out["Y_store_TB_per_s"] = y_bytes / (out["regressor_Y_only"]["median_ms"] * 1e-3) / 1e12
    t = [torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (n_q, nd, nd)]
    outs = z(nd * npi), z(npi), z(npi)
    out["jvp_m1"] = timed(lambda: sim.regressor_jvp_device(qs, qds, qdds, 1, *t, *outs), reps)
    del t, outs, Y
    G = [torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (nd * npi, npi, npi)]
    g = z(n_q), z(nd), z(nd)
    out["vjp"] = timed(lambda: sim.regressor_vjp_device(qs, qds, qdds, *G, *g), reps)
    del G
    qt, qdt, qddt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, qdd))
    GY, GT, GV = (torch.tensor(rng.normal(size=s), device=dev) for s in ((n, nd, npi), (n, npi), (n, npi)))

    def bwd():
        a, b, c = (x.clone().requires_grad_(True) for x in (qt, qdt, qddt))
        Yo, To, Vo = tds_b200.autograd.regressor(sim, a, b, c)
        ((Yo * GY).sum() + (To * GT).sum() + (Vo * GV).sum()).backward()
    out["autograd_backward"] = timed(bwd, reps)
    tau = z(nd)
    out["inverse_dynamics"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, qdds, tau), reps)
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
