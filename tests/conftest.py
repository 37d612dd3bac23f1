import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without a CUDA device (or without the built library) skips the gpu-marked tests instead of failing."""
    import torch
    lib = os.path.join(ROOT, "fatezero_b200", "libfatezero_b200.so")
    reason = None
    if not torch.cuda.is_available():
        reason = "needs a CUDA device (H100)"
    elif not os.path.exists(lib):
        reason = f"{lib} is not built (python -c 'import __graft_entry__ as g; g.build()')"
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


_REPORT = {}


@pytest.fixture
def report(request):
    """Collect error statistics per test; dumped to gpurun_out/test_report.json at session end."""
    d = {}
    _REPORT[request.node.nodeid] = d
    return d


def pytest_sessionfinish(session, exitstatus):
    if _REPORT:
        out = os.path.join(ROOT, "gpurun_out")
        try:
            os.makedirs(out, exist_ok=True)
            path = os.path.join(out, "test_report.json")
            old = {}
            if os.path.exists(path):
                try:
                    old = json.load(open(path))
                except Exception:
                    old = {}
            old.update(_REPORT)
            json.dump(old, open(path, "w"), indent=1, default=str)
        except OSError:
            pass
