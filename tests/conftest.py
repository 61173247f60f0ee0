import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the CPU oracle (torch convs + OpenMP C scan) on the physical cores inside the cgroup quota: all SMT threads of a GPU host
    # with a small CPU quota make it ~100x slower
    import torch
    from oracle import cscan
    torch.set_num_threads(cscan.host_threads())


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def net_sisr_tiny():
    """input "x", output "y" and state_dict "sd/<key>" of the tiny reference SR net (tests/golden/make_golden.py gen_net),
    stored in two files so that neither exceeds 1 MB"""
    import numpy as np
    z = {}
    for name in ("net_sisr_tiny.npz", "net_sisr_tiny_up4_3.npz"):
        with np.load(os.path.join(GOLDEN, name)) as f:
            z.update({k: f[k] for k in f.files})
    return z
