"""The inverse mass matrix and the operational-space inverse inertia on the GPU (DESIGN.md section 7.20): M^-1 alone
(BatchSim.mass_inverse_device), M^-1 with J M^-1 J^T of four points (Laikago's toes, the humanoid's last four leaf links), the JVP at
m = 1 and m = n_q and the VJP (mass_inverse_jvp_device, mass_inverse_vjp_device, with the points), the backward of
tds_b200.autograd.mass_inverse, the mass matrix alone for context, and the same quantities by hand: mass_matrix + torch.linalg.cholesky +
torch.cholesky_inverse + J @ Minv @ J^T with J of point_motion.  CUDA events after a warm-up, median of --reps runs; prints the GPU's
name, power limit and maximum SM clock read in the same run.

    python scripts/bench_mass_inverse.py [--n 4096] [--reps 7]
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


def leaves(model):
    nl = int(model[1])
    parents = {int(model[16 + 13 + i * 34]) for i in range(nl)}
    return [i for i in range(nl) if i not in parents][-4:]


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    lk = [9, 13, 17, 21] if name == "laikago" else leaves(model)
    lc = np.zeros((len(lk), 3))
    R = 6 * len(lk)
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qs = torch.zeros((n_q, ns), dtype=torch.float32, device=dev)
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    z = lambda rows: torch.zeros((rows, ns), dtype=torch.float64, device=dev)
    M, Mi, L = z(nd * nd), z(nd * nd), z(R * R)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, points=lk)
    out["M"] = timed(lambda: sim.mass_matrix_device(qs, M), reps)
    out["Minv"] = timed(lambda: sim.mass_inverse_device(qs, None, None, Mi), reps)
    out["Minv_Linv"] = timed(lambda: sim.mass_inverse_device(qs, lk, lc, Mi, L), reps)
    for m in (1, n_q):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), dtype=torch.float64, device=dev)
        tM, tL = z(nd * nd * m), z(R * R * m)
        out[f"jvp_m{m}"] = timed(lambda: sim.mass_inverse_jvp_device(qs, lk, lc, m, tq, None, tM, tL), reps)
        del tq, tM, tL
    GM, GL = (torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (nd * nd, R * R))
    gq = z(n_q)
    out["vjp"] = timed(lambda: sim.mass_inverse_vjp_device(qs, lk, lc, GM, GL, gq), reps)
    qt = torch.tensor(q, dtype=torch.float32, device=dev)
    GMt = torch.tensor(rng.normal(size=(n, nd, nd)), dtype=torch.float64, device=dev)
    GLt = torch.tensor(rng.normal(size=(n, R, R)), dtype=torch.float64, device=dev)

    def bwd():
        x = qt.clone().requires_grad_(True)
        a, b = tds_b200.autograd.mass_inverse(sim, x, lk, lc)
        ((a * GMt).sum() + (b * GLt).sum()).backward()
    out["autograd_backward"] = timed(bwd, reps)

    def by_hand():
        Mt = tds_b200.autograd.mass_matrix(sim, qt)
        Minv = torch.cholesky_inverse(torch.linalg.cholesky(Mt))
        J = tds_b200.autograd.point_motion(sim, qt, None, lk, lc)[0].reshape(n, R, nd)
        return Minv, J @ Minv @ J.mT
    out["by_hand_Minv_Linv"] = timed(by_hand, reps)
    hm, hl = by_hand()
    out["by_hand_max_abs_diff"] = [float((hm - Mi[:, :n].t().reshape(n, nd, nd)).abs().max()),
                                   float((hl - L[:, :n].t().reshape(n, R, R)).abs().max())]
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
