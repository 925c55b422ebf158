"""Cost of per-environment physical parameters on the GPU (DESIGN.md section 7.9), Laikago with PD control, MODE_FULL:
  * the world-frame step without parameters against the same step with every link's inertial parameters installed (at the model's
    values, so the outputs must agree; their largest difference is reported),
  * the parameter Jacobian (dual numbers, k directions per environment) at k = 4 and k = 40,
  * the vector-Jacobian product without parameters and with the link inertial parameters installed.
CUDA events after a warm-up, median of --reps runs; prints the GPU's name and power limit read in the same run.

    python scripts/bench_params.py [--n 4096] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["TDS_B200_KERNEL"] = "world"   # both sides of the step comparison on the world-frame kernel

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tds_b200  # noqa: E402
import tds_b200.workloads as wl  # noqa: E402
from tds_b200.model import param_names, param_values  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()                                   # warm-up (module load, tape capacity, scratch buffers)
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


def soa(x, ns, dev):
    t = torch.zeros((max(x.shape[1], 1), ns), dtype=torch.float32, device=dev)
    t[:x.shape[1], :x.shape[0]] = torch.tensor(x.T, dtype=torch.float32)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_params.py measures on the GPU; no CUDA device found")
    import ctypes
    n, dev = a.n, "cuda:0"
    w = wl.laikago_perturbed(n, seed=1)
    sim = tds_b200.laikago_sim(n)
    ns = sim.n_stride
    q, qd, act = soa(w["q"], ns, dev), soa(w["qd"], ns, dev), soa(w["action"], ns, dev)
    qo, qdo = torch.zeros_like(q), torch.zeros_like(qd)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    names = param_names(sim.model)
    link_ids = [i for i, nm in enumerate(names) if nm.startswith("link") and not nm.endswith(("stiffness", "damping"))]
    vals = param_values(sim.model, friction=1.0)
    res = [dict(gpu=gpu_info(), n_envs=n, workload="laikago FULL + PD")]

    def step():
        sim.step_device(2, q, qd, act, q_out=qo, qd_out=qdo, use_pd=True)
    r0 = timed(step, a.reps)
    out0 = (qo.clone(), qdo.clone())
    sim.set_physical_params(link_ids, vals[link_ids])
    r1 = timed(step, a.reps)
    diff = max(float((qo - out0[0]).abs().max()), float((qdo - out0[1]).abs().max()))
    res.append(dict(case="step_world_kernel", kernel=sim.kernel_name(), no_params=r0, link_inertials_installed=r1,
                    k=len(link_ids), max_abs_output_diff=diff))

    rows, cols = sim.jacobian_dims(2, True)
    for k in (4, 40):
        ids = link_ids[:k]
        sim.set_physical_params(ids, vals[ids])
        jac = torch.zeros((rows * k, ns), dtype=torch.float64, device=dev)

        def pj():
            rc = sim._L.tds_b200_step_param_jacobian_device(sim._h, 2, 1, q.data_ptr(), qd.data_ptr(), act.data_ptr(), jac.data_ptr(), st)
            assert rc == 0, rc
        res.append(dict(case=f"param_jacobian_k{k}", rows=rows, k=k, time=timed(pj, a.reps)))

    g = torch.randn((rows, ns), dtype=torch.float64, device=dev)
    g_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    sim.set_physical_params(None)
    r_plain = timed(lambda: sim.step_vjp_device(2, q, qd, act, g, g_in, use_pd=True), a.reps)
    gi0 = g_in.clone()
    sim.set_physical_params(link_ids, vals[link_ids])
    g_par = torch.zeros((len(link_ids), ns), dtype=torch.float64, device=dev)
    r_par = timed(lambda: sim.step_vjp_params_device(2, q, qd, act, g, g_in, g_par, use_pd=True), a.reps)
    agree = float(((g_in - gi0).abs() / gi0.abs().clamp(min=1.0))[:, :n].max())
    res.append(dict(case="vjp", no_params=r_plain, link_inertials_installed=r_par, k=len(link_ids), g_in_max_rel_diff=agree))
    lines = [json.dumps(r) for r in res]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
