"""The search's launch counter (`MCTSAgent.launch_count`) against the kernel plan of a search, and against the kernels the
profiler sees.  Each search kernel is counted where it is launched and a graph replay adds the launches its capture
enqueued; the network counts its own kernels the same way (tests/test_net_gpu.py).  The tests add both counters up, so
that a kernel moving from one to the other -- the stem convolution, which a float16 search with Threads = 2 runs on its
tree stream -- cannot hide an error."""
import collections

import numpy as np
import pytest

from oracle import net as onet

B = 8
K = 3  # thread_iteration(K)
CONFIGS = [(backend, threads, trees) for backend in ("fake", "float16", "float32") for threads in (1, 2) for trees in (1, 3)]
IDS = [f"{b}-threads{t}-trees{n}" for b, t, n in CONFIGS]


@pytest.fixture(scope="module")
def blob(tmp_path_factory):
    from crazyara_b200.weights import export_blob
    arch = onet.arch_risev2(34, 81)
    return export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path_factory.mktemp("net") / "risev2.arab"), input_version=10)


def _agent(blob, backend, threads, trees):
    from crazyara_b200.engine import BoardState, MCTSAgent, default_settings
    from crazyara_b200.nn import NeuralNetAPI
    net = None if backend == "fake" else NeuralNetAPI("gpu", 0, trees * B, blob, precision=backend)
    agent = MCTSAgent(net, default_settings("crazyhouse", batch_size=B, simulations=2000, threads=threads), 0, trees)
    state = BoardState().set("", False, 1)
    for t in range(trees):
        agent.set_position(state, t)
    return net, agent


def _launches(agent, net):
    return agent.launch_count() + (net.launch_count() if net is not None else 0)


def _forward_launches(net):
    """The network's kernels per device forward: the second forward of a size replays the graph the first captured."""
    net.forward_device(0, 1)
    before = net.launch_count()
    net.forward_device(0, 1)
    return net.launch_count() - before


def _go(agent, net):
    """begin() and two thread_iteration(K) calls: what each added to the counters"""
    counts = [_launches(agent, net)]
    agent.begin()
    counts.append(_launches(agent, net))
    for _ in range(2):
        agent.thread_iteration(K)
        counts.append(_launches(agent, net))
    return list(np.diff(counts))


@pytest.mark.gpu
@pytest.mark.parametrize("backend,threads,trees", CONFIGS, ids=IDS)
def test_search_launch_count_follows_the_kernel_plan(blob, backend, threads, trees):
    net, agent = _agent(blob, backend, threads, trees)
    agent.begin()  # a first go warms the handle and the network's graphs of every size up
    agent.thread_iteration(K)
    replayed = _go(agent, net)  # Threads = 1: iteration graphs; Threads = 2: the first S0 S1 of a go captured, then replays
    agent.set_profile(True)
    eager = _go(agent, net)  # profiling runs every iteration and turn eagerly
    agent.close()
    evaluation = 1 if net is None else _forward_launches(net)  # fake_eval_kernel, or one network forward
    if net is not None:
        net.close()
    many = int(trees > 1)  # pack_kernel
    begin = 1 + many + 1 + evaluation + 3  # root, pack, expand, evaluation, scatter, backup, prepare
    if threads == 1:  # select, pack, expand, evaluation, then update_kernel (many trees) or backup + scatter_prepare
        per_call = K * (1 + many + 1 + evaluation + (1 if many else 2))
        first_call = per_call
    else:  # a cycle: per logical thread update, select, pack, expand, evaluation; the first S0 S1 of a go has no update
        per_call = K * 2 * (1 + 1 + many + 1 + evaluation)
        first_call = per_call - 2
    expected = [begin, first_call + 1, per_call + 1]  # (+ result_kernel)
    assert replayed == expected
    assert eager == expected


@pytest.mark.gpu
@pytest.mark.parametrize("backend,threads,trees", CONFIGS, ids=IDS)
def test_search_launch_count_equals_the_kernels_traced(blob, backend, threads, trees):
    """On a new handle the first thread_iteration runs eagerly, captures its graphs (the network's too) and replays
    them; the second only replays.  Either way the counters advance by the kernels that ran."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    net, agent = _agent(blob, backend, threads, trees)
    agent.begin()
    torch.cuda.synchronize()
    for call in range(2):
        before = _launches(agent, net)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            agent.thread_iteration(K)
            torch.cuda.synchronize()
        counted = _launches(agent, net) - before
        kernels = [e.name for e in prof.events()
                   if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
        assert len(kernels) == counted, (call, counted, collections.Counter(kernels))
    agent.close()
    if net is not None:
        net.close()
