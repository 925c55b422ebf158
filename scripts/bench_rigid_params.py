"""Per-world physical parameters of the rigid-body world on the GPU (DESIGN.md section 7.11).  For the 7-ball billiard and the stack
world, 4096 worlds, 1 and 20 steps: the step without a parameter set and with every id installed at the description's values (and the
largest difference of the two outputs, expected 0), the parameter Jacobian (host entry: its time includes the transfers and the
host-side transposition of [n][13 n_bodies][k]), the JVP with m = 1 and m = k parameter tangents, and the VJP without and with
parameters.  CUDA events after a warm-up, median of --reps runs, on a stream of its own that every device call is given; prints the
GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_rigid_params.py [--n 4096] [--reps 7]
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
import tds_b200.rigid as rg  # noqa: E402
import tds_b200.workloads as wl  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps, stream):
    fn()                                   # warm-up (module load, buffers, tape capacity)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), max_ms=float(np.max(ts)))


def case(kind, n, steps, reps, st):
    dev = "cuda:0"
    w = wl.rigid_world(kind, n, seed=5)
    world = tds_b200.RigidWorld(w["bodies"], n, **w["params"])
    nb, ns = world.n_bodies, world.n_stride
    ids = rg.param_ids(w["bodies"], rg.param_names(w["bodies"]))
    k = len(ids)
    vals = rg.param_values(w["bodies"], friction=w["params"].get("friction", 0.5), restitution=w["params"].get("restitution", 0.0))

    def soa(a, d):
        t = torch.zeros((d, ns), dtype=torch.float64, device=dev)
        t[:, :n] = torch.tensor(a.reshape(n, d).T, device=dev)
        return t
    s, f = soa(w["state"], 13 * nb), soa(w["force"], 3 * nb)
    out0, out1 = torch.empty_like(s), torch.empty_like(s)
    g = soa(np.random.default_rng(6).normal(size=(n, 13 * nb)), 13 * nb)
    gs, gf, gp = torch.zeros_like(s), torch.zeros_like(f), torch.zeros((k, ns), dtype=torch.float64, device=dev)
    t1 = torch.zeros((k, ns), dtype=torch.float64, device=dev)
    t1[0] = 1.0
    tk = torch.zeros((k * k, ns), dtype=torch.float64, device=dev)
    for j in range(k):
        tk[j * k + j] = 1.0
    to1, tok = torch.zeros((13 * nb, ns), dtype=torch.float64, device=dev), torch.zeros((13 * nb * k, ns), dtype=torch.float64, device=dev)
    r = dict(world=kind, n_worlds=n, n_bodies=nb, steps=steps, k=k)
    r["step_without_params"] = timed(lambda: world.step_device(s, out0, f, steps, stream=st), reps, st)
    r["vjp_without_params"] = timed(lambda: world.step_vjp_device(s, f, g, gs, gf, steps, stream=st), reps, st)
    world.set_physical_params(ids, vals)
    r["step_with_params"] = timed(lambda: world.step_device(s, out1, f, steps, stream=st), reps, st)
    torch.cuda.synchronize()
    r["max_abs_diff_with_params"] = float((out1[:, :n] - out0[:, :n]).abs().max())
    r["param_jacobian_host_entry"] = timed(lambda: world.step_param_jacobian(w["state"], w["force"], steps), reps, st)
    r["jvp_params_m1"] = timed(lambda: world.step_jvp_device(s, f, 1, None, None, None, to1, steps, stream=st, t_par=t1), reps, st)
    r["jvp_params_mk"] = timed(lambda: world.step_jvp_device(s, f, k, None, None, None, tok, steps, stream=st, t_par=tk), reps, st)
    r["vjp_with_params"] = timed(lambda: world.step_vjp_params_device(s, f, g, gs, gf, gp, steps, stream=st), reps, st)
    world.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rigid_params: no CUDA device (there is nothing to measure on the CPU)")
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    st = torch.cuda.Stream()
    for kind in ("billiard", "stack"):
        for steps in (1, 20):
            print(json.dumps(case(kind, a.n, steps, a.reps, st)), flush=True)


if __name__ == "__main__":
    main()
