"""The step that reports its contacts on the GPU (DESIGN.md section 7.15): the contact-reporting step (BatchSim.step_contacts_device), the
world-frame step without records (step_device with TDS_B200_KERNEL=world), the default kernel's step (step_device), the JVP at m = 1 and
m = n_in (step_contacts_jvp_device), the VJP (step_contacts_vjp_device) and the backward of tds_b200.autograd.step_contacts, in MODE_FULL
at the simulator's default precision, on Laikago (with PD) and the humanoid.  CUDA events after a warm-up, median of --reps runs; prints
the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_contacts.py [--n 4096] [--reps 7]
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
import tds_b200.workloads as wl  # noqa: E402
from tds_b200.model import fixture_path, load_model  # noqa: E402
from bench_mass_matrix import gpu_info, timed  # noqa: E402


def make(name, n):
    if name == "laikago":
        return tds_b200.laikago_sim(n), wl.laikago_perturbed(n), True
    model = load_model(fixture_path(name))
    w = wl.humanoid(n)
    return tds_b200.BatchSim(model, n), dict(q=w["q"], qd=w["qd"], action=None), False


def case(name, n, reps):
    dev = "cuda:0"
    sim, w, pd = make(name, n)
    ns, n_q, nd, npts = sim.n_stride, sim.n_q, sim.n_qd, sim.n_contact_points
    rows, cols = sim.contact_rows(2, pd)

    def soa(x, dt=torch.float32):
        t = torch.zeros((max(x.shape[1], 1), ns), dtype=dt, device=dev)
        t[:x.shape[1], :n] = torch.tensor(np.asarray(x).T, dtype=dt)
        return t
    qs, qds = soa(w["q"]), soa(w["qd"])
    acts = soa(w["action"]) if pd else None
    qo, qdo = qs.clone(), qds.clone()
    C = torch.zeros((10 * npts, ns), dtype=torch.float32, device=dev)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_contact_points=npts, n_in=cols, precision=sim.precision)
    out["step_contacts"] = timed(lambda: sim.step_contacts_device(2, qs, qds, acts, qo, qdo, C, use_pd=pd), reps)
    out["step_default"] = timed(lambda: sim.step_device(2, qs, qds, acts, q_out=qo, qd_out=qdo, use_pd=pd), reps)
    out["default_kernel"] = sim.kernel_name()
    os.environ["TDS_B200_KERNEL"] = "world"
    wsim = make(name, n)[0]
    del os.environ["TDS_B200_KERNEL"]
    wsim.set_precision(sim.precision)
    out["step_world"] = timed(lambda: wsim.step_device(2, qs, qds, acts, q_out=qo, qd_out=qdo, use_pd=pd), reps)
    rng = np.random.default_rng(0)
    for m in (1, cols):
        t_in = torch.tensor(rng.normal(size=(cols * m, ns)), dtype=torch.float64, device=dev)
        t_out = torch.zeros((rows * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.step_contacts_jvp_device(2, qs, qds, acts, m, t_in, None, t_out, use_pd=pd), reps)
        del t_in, t_out
    G = torch.tensor(rng.normal(size=(rows, ns)), dtype=torch.float64, device=dev)
    g_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    out["vjp"] = timed(lambda: sim.step_contacts_vjp_device(2, qs, qds, acts, G, g_in, use_pd=pd), reps)
    xt = [torch.tensor(np.asarray(x), dtype=torch.float32, device=dev) for x in (w["q"], w["qd"])]
    at = torch.tensor(np.asarray(w["action"]), dtype=torch.float32, device=dev) if pd else None
    Gc = torch.tensor(rng.normal(size=(n, npts, 10)), dtype=torch.float32, device=dev)

    def bwd():
        xs = [x.clone().requires_grad_(True) for x in xt]
        _, _, Co = tds_b200.autograd.step_contacts(sim, *xs, at, use_pd=pd)
        (Co * Gc).sum().backward()
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
