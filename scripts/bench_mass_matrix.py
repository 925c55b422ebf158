"""The joint-space mass matrix on the GPU (DESIGN.md section 7.12): M(q) alone (BatchSim.mass_matrix_device), its JVP at m = 1 and
m = n_q (mass_matrix_jvp_device), its VJP (mass_matrix_vjp_device), the backward of tds_b200.autograd.mass_matrix, and the world-frame
step for context (BatchSim.step_device in fp64 on the world-frame kernel, MODE_FULL), on Laikago and the humanoid.  CUDA events after a
warm-up, median of --reps runs; prints the bytes M writes per environment (8 n_qd^2) and the GPU's name, power limit and maximum SM clock
read in the same run.

    python scripts/bench_mass_matrix.py [--n 4096] [--reps 7]
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
    qs = torch.zeros((n_q, ns), dtype=torch.float32, device=dev)
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    qds = torch.zeros((nd, ns), dtype=torch.float32, device=dev)
    M = torch.zeros((nd * nd, ns), dtype=torch.float64, device=dev)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, bytes_M_per_env=8 * nd * nd)
    out["M"] = timed(lambda: sim.mass_matrix_device(qs, M), reps)
    for m in (1, n_q):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), dtype=torch.float64, device=dev)
        tM = torch.zeros((nd * nd * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.mass_matrix_jvp_device(qs, m, tq, None, tM), reps)
        del tq, tM
    G = torch.tensor(rng.normal(size=(nd * nd, ns)), dtype=torch.float64, device=dev)
    gq = torch.zeros((n_q, ns), dtype=torch.float64, device=dev)
    out["vjp"] = timed(lambda: sim.mass_matrix_vjp_device(qs, G, gq), reps)
    qt = torch.tensor(q, dtype=torch.float32, device=dev)
    Gt = torch.tensor(rng.normal(size=(n, nd, nd)), dtype=torch.float64, device=dev)

    def bwd():
        x = qt.clone().requires_grad_(True)
        (tds_b200.autograd.mass_matrix(sim, x) * Gt).sum().backward()
    out["autograd_backward"] = timed(bwd, reps)
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
