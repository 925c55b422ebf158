"""Forward mode on the GPU (DESIGN.md section 7.10): Jacobian-vector products of one step (BatchSim.step_jvp_device: one dual-number
lane per environment and tangent) at m = 1, 4, 16 and m = cols, against the dense Jacobian (step_jacobian_device) and the
vector-Jacobian product (step_vjp_device); the rigid-world JVP of a 20-step billiard rollout against the checkpointed rigid VJP; and
the gradient of the cartpole system identification (tests/test_params_on_host.py) by forward mode (m = 4 fp64 tangents carried
between steps) against reverse mode through tds_b200.autograd.step(..., params=).  CUDA events after a warm-up, median of --reps
runs; prints the GPU's name, power limit and maximum SM clock read in the same run.

    python scripts/bench_jvp.py [--n 4096] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the system identification problem is defined with the test-suite

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tds_b200  # noqa: E402
import tds_b200.workloads as wl  # noqa: E402
from tds_b200.model import fixture_path, load_model  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps):
    fn()                                   # warm-up (module load, scratch buffers, tape capacity)
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


def step_case(name, sim, q, qd, t, pd, reps):
    import ctypes
    dev, mode = "cuda:0", 2
    ns, n = sim.n_stride, sim.n_envs
    qs, qds, ts = soa(q, ns, dev), soa(qd, ns, dev), (soa(t, ns, dev) if t is not None else None)
    rows, cols = sim.jacobian_dims(mode, pd)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    jac = torch.zeros((rows * cols, ns), dtype=torch.float64, device=dev)

    def jacobian():
        rc = sim._L.tds_b200_step_jacobian_device(sim._h, mode, int(pd), qs.data_ptr(), qds.data_ptr(), ts.data_ptr() if ts is not None else None,
                                                   jac.data_ptr(), st)
        assert rc == 0, rc
    out = dict(case=name, n_envs=n, rows=rows, cols=cols, directions_per_launch=sim.jacobian_chunk(), jacobian=timed(jacobian, reps))
    g = torch.randn((rows, ns), dtype=torch.float64, device=dev)
    g_in = torch.zeros((cols, ns), dtype=torch.float64, device=dev)
    out["vjp"] = timed(lambda: sim.step_vjp_device(mode, qs, qds, ts, g, g_in, use_pd=pd), reps)
    for m in (1, 4, 16, cols):
        t_in = torch.randn((cols * m, ns), dtype=torch.float64, device=dev) if m != cols else \
            torch.eye(cols, dtype=torch.float64, device=dev).reshape(cols * cols, 1).expand(cols * cols, ns).contiguous()
        t_out = torch.zeros((rows * m, ns), dtype=torch.float64, device=dev)
        out[f"jvp_m{m}"] = timed(lambda: sim.step_jvp_device(mode, qs, qds, ts, m, t_in, None, t_out, use_pd=pd), reps)
        if m == cols:   # identity tangents: the Jacobian itself (another instance; nvcc may contract differently)
            d = (t_out - jac).abs() / jac.abs().clamp(min=1.0)
            out["jvp_identity_vs_jacobian_max_rel_diff"] = float(d[:, :n].max())
    return out


def rigid_case(n, reps):
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
    m, steps = 3, 20
    t_force = torch.zeros((3 * nb * m, ns), dtype=torch.float64, device=dev)
    for j in range(3):
        t_force[j * m + j] = 1.0                   # the cue ball's force, one component per tangent
    t_out = torch.zeros((13 * nb * m, ns), dtype=torch.float64, device=dev)
    so = torch.zeros_like(s)
    stream = torch.cuda.current_stream()
    r_jvp = timed(lambda: world.step_jvp_device(s, f, m, None, t_force, so, t_out, steps, stream=stream), reps)
    r_vjp = timed(lambda: world.step_vjp_device(s, f, g, gs, gf, steps, stream=stream), reps)
    return dict(case=f"rigid_billiard{nb}_steps{steps}", n_worlds=n, jvp_m3_force_of_one_ball=r_jvp, vjp=r_vjp)


def sysid_case(reps):
    from test_params_on_host import SYSID_ENVS, SYSID_STEPS, sysid_problem
    model, ids, truth, start, q0, qd0, tau, kw = sysid_problem()
    n, dev, k = SYSID_ENVS, "cuda:0", 4
    sim = tds_b200.BatchSim(model, n, **kw)
    sim.set_physical_params(ids, start)
    ns = sim.n_stride
    rows, cols = sim.jacobian_dims(2)
    tau_t = [torch.tensor(tau[s], dtype=torch.float32, device=dev) for s in range(SYSID_STEPS)]
    tau_s = [soa(tau[s], ns, dev) for s in range(SYSID_STEPS)]
    x0, xd0 = torch.tensor(q0, dtype=torch.float32, device=dev), torch.tensor(qd0, dtype=torch.float32, device=dev)
    p_start = torch.tensor(start, dtype=torch.float64, device=dev)

    def rollout(p):
        xs, x, xd = [], x0, xd0
        for s in range(SYSID_STEPS):
            x, xd = tds_b200.autograd.step(sim, x, xd, tau_t[s], params=p.unsqueeze(0).expand(n, -1).contiguous())
            xs.append((x, xd))
        return xs
    with torch.no_grad():
        target = [(a.detach().double(), b.detach().double()) for a, b in rollout(torch.tensor(truth, dtype=torch.float64, device=dev))]
    res = {}

    def reverse():
        p = p_start.clone().requires_grad_(True)
        xs = rollout(p)
        loss = sum(((a.double() - ta) ** 2).sum() + ((b.double() - tb) ** 2).sum() for (a, b), (ta, tb) in zip(xs, target)) / n
        loss.backward()
        res["reverse"] = p.grad
    t_par = torch.zeros((k * k, ns), dtype=torch.float64, device=dev)
    for j in range(k):
        t_par[j * k + j, :n] = 1.0
    tgt = [torch.cat([a.t(), b.t()], 0) for a, b in target]

    def forward():
        sim.set_physical_params(ids, p_start)
        qs, qds = soa(q0, ns, dev), soa(qd0, ns, dev)
        T = torch.zeros((rows * k, ns), dtype=torch.float64, device=dev)
        grad = torch.zeros(k, dtype=torch.float64, device=dev)
        for s in range(SYSID_STEPS):
            t_in = torch.zeros((cols * k, ns), dtype=torch.float64, device=dev)
            t_in[:rows * k] = T
            T = torch.empty((rows * k, ns), dtype=torch.float64, device=dev)
            sim.step_jvp_device(2, qs, qds, tau_s[s], k, t_in, t_par, T)
            q1, qd1 = torch.empty_like(qs), torch.empty_like(qds)
            sim.step_device(2, qs, qds, tau_s[s], q_out=q1, qd_out=qd1)
            qs, qds = q1, qd1
            res_ = torch.cat([qs[:, :n], qds[:, :n]], 0).double() - tgt[s]
            grad += 2 * (T[:, :n].reshape(rows, k, n) * res_[:, None, :]).sum(dim=(0, 2)) / n
        res["forward"] = grad
    r_rev = timed(reverse, reps)
    r_fwd = timed(forward, reps)
    gr, gf = res["reverse"].cpu().numpy(), res["forward"].cpu().numpy()
    return dict(case="sysid_cartpole_gradient", n_envs=n, steps=SYSID_STEPS, k=k, forward_m4=r_fwd, reverse_autograd=r_rev,
                max_rel_diff=float(np.max(np.abs(gf - gr)) / np.max(np.abs(gr))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jvp.py measures on the GPU; no CUDA device found")
    # a non-default stream: the rigid-world calls read a NULL stream handle (torch's default stream) as the world's own stream
    torch.cuda.set_stream(torch.cuda.Stream())
    res = [dict(gpu=gpu_info())]
    n = a.n
    w = wl.laikago_perturbed(n, seed=1)
    res.append(step_case("laikago_pd_full", tds_b200.laikago_sim(n), w["q"], w["qd"], w["action"], True, a.reps))
    w = wl.humanoid(n, seed=1)
    sim = tds_b200.BatchSim(load_model(fixture_path("humanoid")), n, **w["params"])
    t = w["tau"][:, -sim.n_tau:] if w.get("tau") is not None else None
    res.append(step_case("humanoid_full", sim, w["q"], w["qd"], t, False, a.reps))
    del sim
    res.append(rigid_case(n, a.reps))
    res.append(sysid_case(a.reps))
    lines = [json.dumps(r) for r in res]
    print("\n".join(lines))
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
