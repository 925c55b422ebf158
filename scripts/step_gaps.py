"""Where the step period of the headline workload goes: tile work, or the gap between one step's grid and the next.

    python scripts/step_gaps.py [--envs 4096] [--steps 50]

K Laikago env-steps (full step + PD, actions from a ring of 768 tensors larger than L2) are captured back to back into
one CUDA graph, as bench.py runs them, and every step writes its own profiling record (tds_b200_debug_phase_clocks_device):
per (tile, role) the clock64 stamps of the phase boundaries (slots 0..13) and two %globaltimer stamps, slot 14 = kernel
entry (role 0) or the return from griddepcontrol.wait (roles 1..3), slot 15 = after the role's last store.  %globaltimer
is one clock for the whole device, so the gap from the last CTA of step n to the first CTA of step n+1 can be read across
SMs.  Prints per step the first entry, the first post-wait stamp and the last exit (ns, relative to the first step), the
gaps between steps, the median share of the step period that is not tile work, and the per-phase cycle table (as
scripts/phase_profile.py)."""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import tds_b200
import tds_b200.workloads as wl

PHASES = ["load+PD", "pass1 FK+contacts", "pass2 ABA+CRBA", "base+pass3", "cholesky", "J+Y", "PGS", "backsub", "integrate+write"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--show", type=int, default=12, help="steps printed one per line")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_gaps.py: no CUDA device")
    n, K = args.envs, args.steps
    dev = torch.device("cuda", 0)
    sim = tds_b200.laikago_sim(n, device=0, auto_reset=True)
    w = wl.laikago(n, seed=wl.SEED)
    sim.env_set_state(w["q"], w["qd"])
    ns = sim.n_stride
    g = torch.Generator(device="cpu").manual_seed(1234)
    actions = (torch.rand((768, 12, ns), generator=g) * 0.8 - 0.4).to(dev)
    reward, done = torch.zeros(ns, device=dev), torch.zeros(ns, device=dev)
    zero = torch.zeros((12, ns), device=dev)
    for _ in range(10):
        sim.env_step_device(zero, reward, done)
    for i in range(100):
        sim.env_step_device(actions[i % 768], reward, done)
    torch.cuda.synchronize()

    L = tds_b200.lib()
    L.tds_b200_debug_phase_clocks.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    L.tds_b200_debug_phase_clocks_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    nw = L.tds_b200_debug_phase_clocks(sim._h, 0, None, 0)
    rec = torch.zeros((K, nw, 16), dtype=torch.int64, device=dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        for i in range(K):
            L.tds_b200_debug_phase_clocks_device(sim._h, ctypes.c_void_p(rec[i].data_ptr()))
            sim.env_step_device(actions[(100 + i) % 768], reward, done)
    L.tds_b200_debug_phase_clocks_device(sim._h, None)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(20):
        graph.replay()
    ev0.record()
    graph.replay()
    ev1.record()
    torch.cuda.synchronize()
    period_ev = ev0.elapsed_time(ev1) * 1e3 / K

    tiles = (n + 31) // 32
    b = rec[:, :tiles * 4].cpu().numpy().reshape(K, tiles, 4, 16)
    entry = b[:, :, 0, 14]                       # [step][tile] kernel entry, ns
    postwait = b[:, :, 1:, 14].min(axis=2)       # [step][tile] first return from griddepcontrol.wait
    exit_ = b[:, :, :, 15].max(axis=2)           # [step][tile] last store of the tile
    t0 = entry[0].min()
    first_entry, first_wait, last_exit = entry.min(axis=1) - t0, postwait.min(axis=1) - t0, exit_.max(axis=1) - t0
    stamps = np.unique(np.concatenate([entry.ravel(), postwait.ravel(), exit_.ravel()]))
    res = np.min(np.diff(stamps)) if stamps.size > 1 else 0
    print(f"device: {torch.cuda.get_device_name(0)}   library: {tds_b200.lib()._name}   kernel: {sim.kernel_name()}")
    print(f"laikago x{n}: {tiles} tiles, {K} steps in one CUDA graph; %globaltimer: smallest step between distinct stamps {res} ns")
    print(f"step period (CUDA events around the replay): {period_ev:.2f} us")
    print("step  first entry  first post-wait  last exit    (ns since the first entry) | gap: last exit(n-1) -> entry(n), -> post-wait(n)")
    for i in range(K):
        gap = "" if i == 0 else f"{first_entry[i] - last_exit[i - 1]:8d} {first_wait[i] - last_exit[i - 1]:8d}"
        if i < args.show or i == K - 1:
            print(f"{i:4d} {first_entry[i]:12d} {first_wait[i]:16d} {last_exit[i]:10d}    | {gap}")
    period = np.diff(last_exit)                            # exit(n) - exit(n-1)
    work = (last_exit - first_wait)[1:]                    # first post-wait -> last exit of step n
    tile_work = np.median(exit_ - postwait, axis=1)[1:]    # median tile: post-wait -> its last store
    gap_entry = first_entry[1:] - last_exit[:-1]
    gap_wait = first_wait[1:] - last_exit[:-1]
    med = lambda x: float(np.median(x))
    print(f"median over steps 1..{K - 1}: period {med(period) / 1e3:.2f} us | grid span (first post-wait -> last exit) "
          f"{med(work) / 1e3:.2f} us | median tile {med(tile_work) / 1e3:.2f} us")
    print(f"  gap last exit(n-1) -> first entry(n) {med(gap_entry) / 1e3:.2f} us, -> first post-wait(n) {med(gap_wait) / 1e3:.2f} us")
    print(f"  share of the period that is not tile work: {100 * med(1 - work / period):.1f} % (outside the grid span), "
          f"{100 * med(1 - tile_work / period):.1f} % (outside the median tile)")

    clk = b[1:, :, :, :].reshape(-1, 4, 16)                # every tile of every step but the first
    c0 = clk[:, :, 0].min(axis=1, keepdims=True)
    tot = (clk[:, :, len(PHASES)].max(axis=1) - c0[:, 0]).astype(np.float64)
    print("cycles per tile (clock64): total median %.0f (min %.0f max %.0f)" % (np.median(tot), tot.min(), tot.max()))
    print("  phase end (cycles since tile start), median over tiles and steps:  role0 role1 role2 role3 | role-0 duration")
    prev = np.zeros(4)
    for k, nm in enumerate(PHASES):
        end = np.median((clk[:, :, k + 1] - c0).astype(np.float64), axis=0)
        print(f"  {nm:18s} " + " ".join(f"{x:8.0f}" for x in end) + f" | {end[0] - prev[0]:8.0f}")
        prev = end
    ex = np.median((clk[:, 0, 10:14] - c0[:, 0:1]).astype(np.float64), axis=0)
    print("  role 0 extra stamps (cycles since tile start): pass1a start %.0f end %.0f | pass2a end %.0f | trunk leaf->root end %.0f"
          % (ex[2], ex[3], ex[0], ex[1]))


if __name__ == "__main__":
    main()
