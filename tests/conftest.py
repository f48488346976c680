import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")
    # the C-ABI library is built in-tree; build it if a checkout has none yet (nvcc cross-compiles without a GPU)
    # CPU oracle runs: a container that shows 100+ CPUs but is throttled to a few thrashes when torch spawns one thread
    # per visible CPU -- use the affinity mask capped by the cgroup quota (oracle/cpu_step.usable_cores)
    try:
        import torch
        from oracle import cpu_step
        torch.set_num_threads(cpu_step.usable_cores())
    except Exception:
        pass
    lib = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "libb2ddpbert.so")
    if not os.path.exists(lib):
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def cuda_dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)
