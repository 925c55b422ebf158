"""Spatial point Jacobians, point velocities and accelerations on the GPU (DESIGN.md section 7.17): the value
(BatchSim.point_motion_device), its JVP at m = 1 and m = n_in = n_q + 2 n_qd (point_motion_jvp_device), its VJP (point_motion_vjp_device),
the backward of tds_b200.autograd.point_motion, and for context the kinematics (kinematics_device, positions and linear Jacobians of the
same points) and ID (inverse_dynamics_device), on Laikago's four toes and the humanoid's hands and feet (its four leaf links).  CUDA events
after a warm-up, median of --reps runs; prints the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_point_motion.py [--n 4096] [--reps 7]
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

POINTS = {"laikago": [9, 13, 17, 21], "humanoid": [13, 22, 27, 32]}


def case(name, n, reps):
    dev = "cuda:0"
    model = load_model(fixture_path(name))
    sim = tds_b200.BatchSim(model, n, precision=1)
    ns, n_q, nd = sim.n_stride, sim.n_q, sim.n_qd
    n_in = n_q + 2 * nd
    links = POINTS[name]
    K = len(links)
    local = np.zeros((K, 3))
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
    J, vel, acc = z(6 * K * nd), z(6 * K), z(6 * K)
    out = dict(model=name, n_envs=n, n_q=n_q, n_qd=nd, n_in=n_in, points=K)
    out["point_motion"] = timed(lambda: sim.point_motion_device(qs, qds, qdds, links, local, J, vel, acc), reps)
    for m in (1, n_in):
        t = [torch.tensor(rng.normal(size=(r * m, ns)), dtype=torch.float64, device=dev) for r in (n_q, nd, nd)]
        outs = z(6 * K * nd * m), z(6 * K * m), z(6 * K * m)
        out[f"jvp_m{m}"] = timed(lambda: sim.point_motion_jvp_device(qs, qds, qdds, links, local, m, *t, *outs), reps)
        del t, outs
    G = [torch.tensor(rng.normal(size=(r, ns)), dtype=torch.float64, device=dev) for r in (6 * K * nd, 6 * K, 6 * K)]
    g = z(n_q), z(nd), z(nd)
    out["vjp"] = timed(lambda: sim.point_motion_vjp_device(qs, qds, qdds, links, local, *G, *g), reps)
    qt, qdt, qddt = (torch.tensor(x, dtype=torch.float32, device=dev) for x in (q, qd, qdd))
    GJ, Gv, Ga = (torch.tensor(rng.normal(size=s), device=dev) for s in ((n, K, 6, nd), (n, K, 6), (n, K, 6)))

    def bwd():
        a, b, c = (x.clone().requires_grad_(True) for x in (qt, qdt, qddt))
        Jo, vo, ao = tds_b200.autograd.point_motion(sim, a, b, links, local, qdd=c)
        ((Jo * GJ).sum() + (vo * Gv).sum() + (ao * Ga).sum()).backward()
    out["autograd_backward"] = timed(bwd, reps)
    x, Jk = z(3 * K), z(3 * K * nd)
    out["kinematics"] = timed(lambda: sim.kinematics_device(qs, links, local, None, x, Jk), reps)
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
