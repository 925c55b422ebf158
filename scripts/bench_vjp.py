"""Reverse mode against forward mode on the GPU: the vector-Jacobian product of one step (BatchSim.step_vjp_device: taping
instance + reverse sweep) against the dense Jacobian (step_jacobian_device: one dual-number lane per input direction) followed by
the contraction g^T J, and the checkpointed rigid-world VJP.  CUDA events after a warm-up, several repetitions each; prints the
GPU's name and power limit beside the numbers (DESIGN.md section 7.8).

    python scripts/bench_vjp.py [--n 4096] [--reps 5]
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
import tds_b200.workloads as wl  # noqa: E402
from tds_b200.model import fixture_path, load_model  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()                                   # warm-up (also grows the tape capacity to what the workload needs)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def soa(x, ns, dev):
    t = torch.zeros((max(x.shape[1], 1), ns), dtype=torch.float32, device=dev)
    t[:x.shape[1], :x.shape[0]] = torch.tensor(x.T, dtype=torch.float32)
    return t


def step_case(name, sim, mode, q, qd, t, pd, reps):
    dev = "cuda:0"
    ns = sim.n_stride
    qs, qds, ts = soa(q, ns, dev), soa(qd, ns, dev), (soa(t, ns, dev) if t is not None else None)
    rows, cols = sim.jacobian_dims(mode, pd)
    g = torch.randn((rows, ns), dtype=torch.float64, device=dev)
    g_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    jac = torch.zeros((rows * cols, ns), dtype=torch.float64, device=dev)
    st = ctypes_stream()

    def vjp():
        sim.step_vjp_device(mode, qs, qds, ts, g, g_in, use_pd=pd)

    def fwd():
        rc = sim._L.tds_b200_step_jacobian_device(sim._h, mode, int(pd), qs.data_ptr(), qds.data_ptr(),
                                                   ts.data_ptr() if ts is not None else None, jac.data_ptr(), st)
        assert rc == 0, rc
        g_in.copy_(torch.einsum("rn,rcn->cn", g, jac.view(rows, cols, ns)))   # the contraction g^T J per environment
    r_vjp = timed(vjp, reps)
    v1 = g_in.clone()
    r_fwd = timed(fwd, reps)
    agree = float(((g_in - v1).abs() / v1.abs().clamp(min=1.0))[:, :sim.n_envs].max())
    cap, per_chunk = sim.vjp_tape_info()
    return dict(case=name, n_envs=sim.n_envs, rows=rows, cols=cols, vjp_ms=r_vjp, jacobian_plus_contraction_ms=r_fwd,
                tape_cap_nodes=cap, envs_per_chunk=per_chunk, max_rel_diff=agree)


def ctypes_stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vjp.py measures on the GPU; no CUDA device found")
    # a non-default stream: the rigid-world calls read a NULL stream handle (torch's default stream) as the world's own stream
    torch.cuda.set_stream(torch.cuda.Stream())
    res = [dict(gpu=gpu_info())]
    n = a.n
    w = wl.laikago_perturbed(n, seed=1)
    res.append(step_case("laikago_pd", tds_b200.laikago_sim(n), 2, w["q"], w["qd"], w["action"], True, a.reps))
    w = wl.humanoid(n, seed=1)
    sim = tds_b200.BatchSim(load_model(fixture_path("humanoid")), n, **w["params"])
    t = w["tau"][:, -sim.n_tau:] if w.get("tau") is not None else None
    res.append(step_case("humanoid_full", sim, 2, w["q"], w["qd"], t, False, a.reps))
    del sim
    w = wl.rigid_world("billiard", n, seed=1)
    world = tds_b200.RigidWorld(w["bodies"], n, **w["params"])
    ns, nb, dev = world.n_stride, world.n_bodies, "cuda:0"
    s = torch.zeros((13 * nb, ns), dtype=torch.float64, device=dev)
    s[:, :n] = torch.tensor(w["state"].reshape(n, -1).T)
    s[6::13, n:] = 1.0
    f = torch.zeros((3 * nb, ns), dtype=torch.float64, device=dev)
    f[:, :n] = torch.tensor(w["force"].reshape(n, -1).T)
    g = torch.randn((13 * nb, ns), dtype=torch.float64, device=dev)
    gs, gf = torch.zeros_like(g), torch.zeros_like(f)
    out = torch.zeros_like(s)
    stream = torch.cuda.current_stream()
    for steps in (1, 20):
        r_vjp = timed(lambda: world.step_vjp_device(s, f, g, gs, gf, steps, stream=stream), a.reps)
        r_fwd = timed(lambda: world.step_device(s, out, f, steps, stream=stream), a.reps)
        res.append(dict(case=f"rigid_billiard7_steps{steps}", n_worlds=n, vjp_ms=r_vjp, forward_ms=r_fwd))
    lines = [json.dumps(r) for r in res]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
