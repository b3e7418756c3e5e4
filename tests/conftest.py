import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kinematic-icp_b200", "python")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure): oracle/libkicp_oracle.so via ctypes."""
    from oracle import kicp_oracle_py as ko
    ko.build()
    ko.lib()
    return ko


@pytest.fixture(scope="session")
def gpu_ctx():
    import kinematic_icp_b200 as kb
    ctx = kb.Context(0)
    yield ctx
    ctx.close()


_WORKLOADS = {}


@pytest.fixture(scope="session")
def workload(oracle):
    from oracle import workloads as W

    def get(cfg_id, **kw):
        key = (cfg_id, tuple(sorted(kw.items())))
        if key not in _WORKLOADS:
            _WORKLOADS[key] = W.Workload(cfg_id, **kw)
        return _WORKLOADS[key]

    return get
