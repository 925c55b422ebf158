"""The Coriolis matrix on the GPU (DESIGN.md section 7.22): C(q, qd) alone (BatchSim.coriolis_device), its JVP at m = 1 and m = n_q
(coriolis_jvp_device), its VJP (coriolis_vjp_device), the backward of tds_b200.autograd.coriolis, and as context M (mass_matrix_device)
and the bias forces h (inverse_dynamics_device at qdd = 0), on Laikago and the humanoid.  On Laikago (a fixed base whose joints all have
one dof) also the by-hand Christoffel path: n_qd mass-matrix JVPs along the unit velocities and a torch contraction.  CUDA events after a
warm-up, median of --reps runs; prints the GPU's name, power limit and maximum SM clock read in the same run, and the largest difference
between C and the by-hand path.

    python scripts/bench_coriolis.py [--n 4096] [--reps 7]
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


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qd = rng.normal(size=(n, nd))
    qs = torch.zeros((n_q, ns), dtype=torch.float32, device=dev)
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    qds = torch.zeros((nd, ns), dtype=torch.float32, device=dev)
    qds[:, :n] = torch.tensor(qd.T, dtype=torch.float32)
    C = torch.zeros((nd * nd, ns), dtype=torch.float64, device=dev)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, bytes_C_per_env=8 * nd * nd)
    out["C"] = timed(lambda: sim.coriolis_device(qs, qds, C), reps)
    for m in (1, n_q):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), dtype=torch.float64, device=dev)
        tC = torch.zeros((nd * nd * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.coriolis_jvp_device(qs, qds, m, tq, None, None, tC), reps)
        del tq, tC
    G = torch.tensor(rng.normal(size=(nd * nd, ns)), dtype=torch.float64, device=dev)
    gq = torch.zeros((n_q, ns), dtype=torch.float64, device=dev)
    gqd = torch.zeros((nd, ns), dtype=torch.float64, device=dev)
    out["vjp"] = timed(lambda: sim.coriolis_vjp_device(qs, qds, G, gq, gqd), reps)
    qt = torch.tensor(q, dtype=torch.float32, device=dev)
    qdt = torch.tensor(qd, dtype=torch.float32, device=dev)
    Gt = torch.tensor(rng.normal(size=(n, nd, nd)), dtype=torch.float64, device=dev)

    def bwd():
        x, y = qt.clone().requires_grad_(True), qdt.clone().requires_grad_(True)
        (tds_b200.autograd.coriolis(sim, x, y) * Gt).sum().backward()
    out["autograd_backward"] = timed(bwd, reps)
    M = torch.zeros((nd * nd, ns), dtype=torch.float64, device=dev)
    out["M"] = timed(lambda: sim.mass_matrix_device(qs, M), reps)
    h = torch.zeros((nd, ns), dtype=torch.float64, device=dev)
    out["h"] = timed(lambda: sim.inverse_dynamics_device(qs, qds, None, h), reps)
    if not int(model[2]) and n_q == nd:
        # by hand: D_k M along the unit velocities (dq/dt = e_k: Laikago's joints have unit axes), then C_ij = 1/2 (D_k M_ij + D_j M_ik -
        # D_i M_jk) qd_k
        eye = torch.zeros((n_q * nd, ns), dtype=torch.float64, device=dev)
        eye.view(n_q, nd, ns)[torch.arange(n_q), torch.arange(nd), :] = 1.0
        dM = torch.zeros((nd * nd * nd, ns), dtype=torch.float64, device=dev)
        res = {}

        def by_hand():
            sim.mass_matrix_jvp_device(qs, nd, eye, None, dM)
            D = dM[:, :n].reshape(nd, nd, nd, n)            # [i, j, k, e] = D_k M_ij
            v = qds[:, :n].double()
            res["C"] = 0.5 * (torch.einsum("ijke,ke->eij", D, v) + torch.einsum("ikje,ke->eij", D, v) - torch.einsum("jkie,ke->eij", D, v))
        out["christoffel_by_hand"] = timed(by_hand, reps)
        sim.coriolis_device(qs, qds, C)
        torch.cuda.synchronize()
        Ce = C[:, :n].t().reshape(n, nd, nd)
        out["christoffel_max_abs_diff"] = float((Ce - res["C"]).abs().max())
        out["C_max_abs"] = float(Ce.abs().max())
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
