"""Forward kinematics and linear point Jacobians on the GPU (DESIGN.md section 7.13): the kinematics alone (BatchSim.kinematics_device),
the JVP at m = 1 and m = n_q (kinematics_jvp_device), the VJP (kinematics_vjp_device), the backward of
tds_b200.autograd.forward_kinematics, and the world-frame step for context (BatchSim.step_device in fp64 on the world-frame kernel,
MODE_FULL), on Laikago with its 4 toes and the humanoid with the origins of its four leaf links (hands and feet).  CUDA events after a
warm-up, median of --reps runs; prints the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_kinematics.py [--n 4096] [--reps 7]
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


def points(name, model):
    """Laikago: the four toes; the humanoid: the links without children (hands and feet), each at its origin."""
    if name == "laikago":
        lk = [9, 13, 17, 21]
    else:
        nl = int(model[1])
        parents = {int(model[16 + 13 + i * 34]) for i in range(nl)}
        lk = [i for i in range(nl) if i not in parents]
    return lk, np.zeros((len(lk), 3))


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd, nl = sim.n_stride, sim.n_q, sim.n_qd, sim.n_links
    lk, lc = points(name, model)
    K = len(lk)
    rng = np.random.default_rng(0)
    q = rng.normal(size=(n, n_q)) * 0.3
    if int(model[2]):
        q[:, :4] /= np.linalg.norm(q[:, :4], axis=1, keepdims=True)
    qs = torch.zeros((n_q, ns), dtype=torch.float32, device=dev)
    qs[:, :n] = torch.tensor(q.T, dtype=torch.float32)
    qds = torch.zeros((nd, ns), dtype=torch.float32, device=dev)
    z = dict(dtype=torch.float64, device=dev)
    xf, x, J = torch.zeros((nl * 12, ns), **z), torch.zeros((3 * K, ns), **z), torch.zeros((3 * K * nd, ns), **z)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_links=nl, points=lk, bytes_out_per_env=8 * (12 * nl + 3 * K + 3 * K * nd))
    out["kinematics"] = timed(lambda: sim.kinematics_device(qs, lk, lc, xf, x, J), reps)
    for m in (1, n_q):
        tq = torch.tensor(rng.normal(size=(n_q * m, ns)), **z)
        t_xf, t_x, t_J = torch.zeros((nl * 12 * m, ns), **z), torch.zeros((3 * K * m, ns), **z), torch.zeros((3 * K * nd * m, ns), **z)
        out[f"jvp_m{m}"] = timed(lambda: sim.kinematics_jvp_device(qs, lk, lc, m, tq, t_xf, t_x, t_J), reps)
        del tq, t_xf, t_x, t_J
    Gxf, Gx, GJ = (torch.tensor(rng.normal(size=(r, ns)), **z) for r in (nl * 12, 3 * K, 3 * K * nd))
    gq = torch.zeros((n_q, ns), **z)
    out["vjp"] = timed(lambda: sim.kinematics_vjp_device(qs, lk, lc, Gxf, Gx, GJ, gq), reps)
    qt = torch.tensor(q, dtype=torch.float32, device=dev)
    Gt = [torch.tensor(rng.normal(size=s), **z) for s in ((n, nl, 3, 3), (n, nl, 3), (n, K, 3), (n, K, 3, nd))]

    def bwd():
        v = qt.clone().requires_grad_(True)
        sum((o * g).sum() for o, g in zip(tds_b200.autograd.forward_kinematics(sim, v, lk, lc), Gt)).backward()
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
