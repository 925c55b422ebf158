"""The table-driven tree kernels as the library runs them on the GPU: the trees and states of
tests/test_team_kernel_source_on_host.py through BatchSim, with the role-warp and then the lane-team kernel forced
(TDS_B200_KERNEL, read by tds_b200_create).  A run counts for the kernel it was meant to test only if sim.kernel_name() says
that kernel ran: a model whose role-warp tile does not fit in shared memory falls back to the lane-team kernel, and one that
tds_build_team does not decompose to the world-frame kernel.  Against the fp64 C oracle, against the world-frame kernel in mixed
precision, and against the host build of the same kernel source."""
import numpy as np
import pytest

import emu
import emu_team
import tds_b200
from oracle import port
from test_team_kernel_source_on_host import MODES, TOL64, _random_model, _served, out_key, rel_err, tree, tree_ids

pytestmark = pytest.mark.gpu

NAMES = {"role": "tds_stepr_kernel", "team": "tds_stept_kernel"}
C_MIXED_GPU = 4.0   # err_tree <= C_MIXED_GPU * err_world + 1e-6 in mixed precision, both on the GPU (rcp.approx); see below


SMEM_OPTIN = 227 * 1024   # shared memory a CTA may opt into on the H100


def gpu_trees(precision):
    """The host test's trees, then further random trees whose role-warp tile fits in shared memory in `precision`: most random
    trees with contacts need more than 227 KB per role-warp tile, and the library runs those on the lane-team kernel."""
    extra = [s for s in range(40, 400) if _served(_random_model(s)) and emu_team.info(_random_model(s))["role_tile_bytes"][precision] <= SMEM_OPTIN]
    return tree_ids() + [f"random-{s}" for s in extra]


def _states(tid, n):
    """The first n environments of tree(tid), repeated when n exceeds the host test's batch."""
    model, q, qd, tau = tree(tid)
    idx = np.arange(n) % q.shape[0]
    return model, q[idx], qd[idx], tau[idx]


def _run(kernel, monkeypatch, model, n, precision):
    monkeypatch.setenv("TDS_B200_KERNEL", kernel)
    sim = tds_b200.BatchSim(model, n)
    sim.set_precision(precision)
    return sim


@pytest.mark.parametrize("kernel", ["role", "team"])
@pytest.mark.parametrize("n", [37, 256])
def test_fp64_on_the_gpu_against_the_oracle_and_the_host_build(kernel, n, monkeypatch):
    """fp64: |x - ref| <= 2e-7 max(1, |ref|) against the oracle and against the host build of the same kernel source, every tree
    and mode.  At least 24 of the random trees must really have run on the kernel under test."""
    ran = {"random": 0, "other": 0}
    for tid in gpu_trees(1):
        model, q, qd, tau = _states(tid, n)
        sim = _run(kernel, monkeypatch, model, n, tds_b200.PREC_F64)
        P = port.make_params()
        ok = True
        for mode in MODES:
            out = sim.step_host(mode, q, qd, tau)
            if NAMES[kernel] not in sim.kernel_name():
                ok = False
                break
            idx = range(0, n, max(1, n // 40))
            refs = [port.step(model, P, mode, q[i], qd[i], tau[i]) for i in idx]
            host = emu_team.step(model, mode, q, qd, tau, map=kernel, precision=1)
            world = emu.step(model, mode, q[list(idx)], qd[list(idx)], tau[list(idx)], precision=1)
            for k in out_key(mode):
                ref = np.array([r[k] for r in refs])
                # (no worse than the world-frame kernel where that misses 2e-7: the humanoid's contact step, 2.9e-7)
                assert rel_err(out[k][list(idx)], ref) <= max(TOL64, rel_err(world[k], ref)), (tid, mode, k)
                assert rel_err(out[k], host[k]) <= TOL64, (tid, mode, k)
        sim.close()
        if ok:
            ran["random" if tid.startswith("random") else "other"] += 1
    print(f"{kernel} n={n}: ran on {ran['random']} random trees and {ran['other']} fixture / hand-made trees")
    assert ran["random"] >= 24, ran


@pytest.mark.parametrize("kernel", ["role", "team"])
def test_mixed_on_the_gpu_against_the_world_kernel(kernel, monkeypatch):
    """Mixed precision with the real rcp.approx: each tree kernel is held to the world-frame kernel on the GPU in the same precision,
    err_tree <= C_MIXED_GPU * err_world + 1e-6 against the fp64 oracle.  The worst observed ratio err_tree / err_world (where
    err_world > 1e-6) over every tree and mode was 2.8 for both kernels on an NVIDIA H100 80GB HBM3 (700 W power limit);
    C_MIXED_GPU = 4."""
    n = 37
    worst = 0.0
    ran = 0
    for tid in gpu_trees(0):
        model, q, qd, tau = _states(tid, n)
        P = port.make_params()
        sim = _run(kernel, monkeypatch, model, n, tds_b200.PREC_MIXED)
        world = _run("world", monkeypatch, model, n, tds_b200.PREC_MIXED)
        ok = True
        for mode in MODES:
            out = sim.step_host(mode, q, qd, tau)
            if NAMES[kernel] not in sim.kernel_name():
                ok = False
                break
            w = world.step_host(mode, q, qd, tau)
            assert "tds_stepw_kernel" in world.kernel_name()
            refs = [port.step(model, P, mode, q[i], qd[i], tau[i]) for i in range(n)]
            for k in out_key(mode):
                ref = np.array([r[k] for r in refs])
                err, err_w = rel_err(out[k], ref), rel_err(w[k], ref)
                if err_w > 1e-6:
                    worst = max(worst, err / err_w)
                assert err <= C_MIXED_GPU * err_w + 1e-6, (tid, mode, k, err, err_w)
        sim.close(); world.close()
        ran += ok and tid.startswith("random")
    print(f"{kernel}: ran on {ran} random trees, worst mixed-precision ratio err_tree / err_world = {worst:.3g}")
    assert ran >= 24


def test_the_model_with_29_local_links_in_one_role_runs_on_the_world_kernel(monkeypatch):
    """tds_build_team refuses the model (TDS_TEAM_MAXK): asking for a tree kernel gets the world-frame kernel, with the oracle's result."""
    from test_team_kernel_source_on_host import PLANE, _maxk_29_urdf, compile_urdf
    model = compile_urdf(_maxk_29_urdf(), PLANE, floating=True)
    n = 4
    q = np.zeros((n, int(model[3]))); q[:, 3] = 1.0; q[:, 6] = 2.0
    qd = np.random.default_rng(2).uniform(-1, 1, (n, int(model[4]))).astype(np.float32).astype(np.float64)
    sim = _run("role", monkeypatch, model, n, tds_b200.PREC_F64)
    out = sim.step_host(1, q, qd)
    assert "tds_stepw_kernel" in sim.kernel_name()
    P = port.make_params()
    ref = np.array([port.step(model, P, 1, q[i], qd[i], None)["qd"] for i in range(n)])
    assert rel_err(out["qd"], ref) <= TOL64
    sim.close()
