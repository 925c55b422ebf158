"""Back-to-back steps of the specialised kernel overlap on the GPU (programmatic dependent launch: the next step's CTAs are
scheduled while the previous step runs and wait for it in griddepcontrol.wait).  The overlap must not change a single bit
of what the steps compute: K steps captured into one CUDA graph, or enqueued together with the policy kernel of a device
rollout, give exactly the state of the same K steps launched one at a time with a device synchronisation in between."""
import numpy as np
import pytest
import torch

import tds_b200
import tds_b200.workloads as wl

pytestmark = pytest.mark.gpu

K = 50


def _sim(name, n):
    if name == "laikago":
        sim = tds_b200.laikago_sim(n, auto_reset=True)
        w = wl.laikago(n, seed=wl.SEED)
        sim.env_set_state(w["q"], w["qd"])
    else:
        sim = tds_b200.ant_sim(n, auto_reset=True)
        sim.env_reset_device(seed=3)
        torch.cuda.synchronize()
    return sim


def _outputs(sim, rewards, dones):
    q, qd = sim.env_get_state()
    return q, qd, torch.stack(rewards).cpu().numpy(), torch.stack(dones).cpu().numpy()


@pytest.mark.parametrize("name,n", [("laikago", 4096), ("laikago", 1000), ("laikago", 65536), ("ant", 4096)])
def test_graph_of_steps_equals_serial_steps(name, n):
    """n = 4096 / 1000: one wave (the kernel lets the next step start at its entry); 65536: several waves (trigger after
    the tile's last store)."""
    sim = _sim(name, n)
    dev, ns, na = torch.device("cuda", 0), sim.n_stride, sim.n_act
    g = torch.Generator(device="cpu").manual_seed(77)
    acts = [(torch.rand((na, ns), generator=g) * 0.8 - 0.4).to(dev) for _ in range(K)]
    rew = [torch.zeros(ns, device=dev) for _ in range(K)]
    don = [torch.zeros(ns, device=dev) for _ in range(K)]
    for i in range(3):
        sim.env_step_device(acts[i], rew[i], don[i])
    torch.cuda.synchronize()
    assert "model-specialised" in sim.kernel_name()
    q0, qd0 = sim.env_get_state()

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        for i in range(K):
            sim.env_step_device(acts[i], rew[i], don[i])
    torch.cuda.synchronize()
    sim.env_set_state(q0, qd0)
    graph.replay()
    torch.cuda.synchronize()
    overlapped = _outputs(sim, rew, don)

    for t in rew + don:
        t.zero_()
    sim.env_set_state(q0, qd0)
    for i in range(K):
        sim.env_step_device(acts[i], rew[i], don[i])
        torch.cuda.synchronize()
    serial = _outputs(sim, rew, don)
    for a, b in zip(overlapped, serial):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("name", ["laikago", "ant"])
def test_device_rollout_equals_serial_steps(name):
    """tds_b200_env_rollout_device enqueues policy kernel -> step -> reward accumulation per step: the step follows a kernel
    that writes its actions and never triggers early.  One K-step rollout against K one-step rollouts, synchronised."""
    n = 4096
    sim = _sim(name, n)
    dev, ns = torch.device("cuda", 0), sim.n_stride
    n_params = sim.n_act * (sim.n_q + sim.n_qd) + sim.n_act
    g = torch.Generator(device="cpu").manual_seed(5)
    policy = ((torch.rand((n_params, ns), generator=g) - 0.5) * 0.02).to(dev)
    tot = torch.zeros(ns, device=dev)
    steps = torch.zeros(ns, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    q0, qd0 = sim.env_get_state()

    sim.env_rollout_device(policy, K, 0.0, tot, steps)
    torch.cuda.synchronize()
    overlapped = sim.env_get_state()

    sim.env_set_state(q0, qd0)
    for _ in range(K):
        sim.env_rollout_device(policy, 1, 0.0, tot, steps)
        torch.cuda.synchronize()
    serial = sim.env_get_state()
    assert not np.array_equal(overlapped[0], q0)
    for a, b in zip(overlapped, serial):
        assert np.array_equal(a, b)
