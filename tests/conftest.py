import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _usable_cpus():
    n = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    try:
        q, per = open('/sys/fs/cgroup/cpu.max').read().split()
        if q != 'max':
            n = min(n, max(1, int(float(q) / float(per) + 0.5)))
    except Exception:
        pass
    return max(1, min(n, 32))


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run with -m gpu on an H100)')
    # the oracle runs on the host: a box that shows 100+ cores but grants a small cgroup quota makes torch's default
    # thread pool thrash (one GPU-box run of this suite took 8 min instead of 30 s)
    import torch
    torch.set_num_threads(_usable_cpus())


@pytest.fixture(scope='session')
def golden():
    import numpy as np
    out = {}
    for name in ('reference_golden.npz', 'reference_golden_sampler.npz'):
        with np.load(os.path.join(ROOT, 'tests', 'golden', name)) as z:
            out.update({k: z[k] for k in z.files})
    return out
