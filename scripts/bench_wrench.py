"""The step with external wrenches on the GPU (DESIGN.md section 7.18): its value in MODE_FULL and MODE_FD (BatchSim.step_wrench_device),
the JVP at m = 1 and m = n_in (step_wrench_jvp_device, tangents of the step's inputs and of the wrenches), the VJP
(step_wrench_vjp_device) and the backward of tds_b200.autograd.step_wrench, at the simulator's default precision, on Laikago (with PD, one
point on the trunk) and the humanoid (a point on each hand and foot); as context the contact-reporting step (step_contacts_device) and the
world-frame step without wrenches (step_device with TDS_B200_KERNEL=world).  CUDA events after a warm-up, median of --reps runs; prints
the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_wrench.py [--n 4096] [--reps 7]
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
from bench_contacts import make  # noqa: E402
from bench_mass_matrix import gpu_info, timed  # noqa: E402

POINTS = {"laikago": ([5], [[0.0, 0.0, 0.0]]),                                 # the trunk
          "humanoid": ([13, 22, 27, 32], [[0.0, 0.0, 0.0]] * 4)}               # hands and feet


def case(name, n, reps):
    dev = "cuda:0"
    sim, w, pd = make(name, n)
    links, local = POINTS[name]
    K = len(links)
    ns, n_q, nd, npts = sim.n_stride, sim.n_q, sim.n_qd, sim.n_contact_points
    rows, cols = sim.jacobian_dims(2, pd)
    rng = np.random.default_rng(0)

    def soa(x, dt=torch.float32):
        t = torch.zeros((max(x.shape[1], 1), ns), dtype=dt, device=dev)
        t[:x.shape[1], :n] = torch.tensor(np.asarray(x).T, dtype=dt)
        return t
    qs, qds = soa(w["q"]), soa(w["qd"])
    acts = soa(w["action"]) if pd else None
    Wn = rng.normal(size=(n, K, 6)) * 10.0
    Ws = soa(Wn.reshape(n, -1))
    qo, qdo, qddo = qs.clone(), qds.clone(), qds.clone()
    C = torch.zeros((10 * npts, ns), dtype=torch.float32, device=dev)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, K=K, n_in=cols + 6 * K, precision=sim.precision)
    out["step_wrench_full"] = timed(lambda: sim.step_wrench_device(2, qs, qds, acts, links, local, Ws, qo, qdo, use_pd=pd), reps)
    out["step_wrench_fd"] = timed(lambda: sim.step_wrench_device(0, qs, qds, acts, links, local, Ws, qdd_out=qddo, use_pd=pd), reps)
    out["step_contacts"] = timed(lambda: sim.step_contacts_device(2, qs, qds, acts, qo, qdo, C, use_pd=pd), reps)
    os.environ["TDS_B200_KERNEL"] = "world"
    wsim = make(name, n)[0]
    del os.environ["TDS_B200_KERNEL"]
    wsim.set_precision(sim.precision)
    out["step_world"] = timed(lambda: wsim.step_device(2, qs, qds, acts, q_out=qo, qd_out=qdo, use_pd=pd), reps)
    out["step_world_fd"] = timed(lambda: wsim.step_device(0, qs, qds, acts, q_out=qo, qd_out=qdo, qdd_out=qddo, use_pd=pd), reps)
    for m in (1, cols + 6 * K):
        t_in = torch.tensor(rng.normal(size=(cols * m, ns)), dtype=torch.float64, device=dev)
        t_W = torch.tensor(rng.normal(size=(6 * K * m, ns)), dtype=torch.float64, device=dev)
        t_out = torch.zeros((rows * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.step_wrench_jvp_device(2, qs, qds, acts, links, local, Ws, m, t_in, t_W, None, t_out, use_pd=pd),
                                 reps)
        del t_in, t_W, t_out
    G = torch.tensor(rng.normal(size=(rows, ns)), dtype=torch.float64, device=dev)
    g_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    g_W = torch.zeros((6 * K, ns), dtype=torch.float64, device=dev)
    out["vjp"] = timed(lambda: sim.step_wrench_vjp_device(2, qs, qds, acts, links, local, Ws, G, g_in, g_W, use_pd=pd), reps)
    xt = [torch.tensor(np.asarray(x), dtype=torch.float32, device=dev) for x in (w["q"], w["qd"])]
    at = torch.tensor(np.asarray(w["action"]), dtype=torch.float32, device=dev) if pd else None
    Wt = torch.tensor(Wn, dtype=torch.float32, device=dev)
    Gq = torch.tensor(rng.normal(size=(n, n_q)), dtype=torch.float32, device=dev)

    def bwd():
        xs = [x.clone().requires_grad_(True) for x in xt + [Wt]]
        q1, _ = tds_b200.autograd.step_wrench(sim, xs[0], xs[1], at, links, local, xs[2], use_pd=pd)
        (q1 * Gq).sum().backward()
    out["autograd_backward"] = timed(bwd, reps)
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
