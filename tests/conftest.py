import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# a missing peer must fail a test quickly instead of hanging the GPU box
os.environ.setdefault("MXKV_B200_SPIN_TIMEOUT_S", "20")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


SIM = bool(os.environ.get("MXKV_SIM"))
if SIM:
    # tests/sim: the engine runs on a stand-in libcudart.so.12; the real torch cannot be loaded into the same
    # process (it needs the real runtime under the same SONAME), so tests that want torch are skipped
    sys.modules["torch"] = None


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_call(item):
    outcome = yield
    if SIM and outcome.excinfo is not None:
        etype, evalue = outcome.excinfo[0], outcome.excinfo[1]
        if issubclass(etype, ImportError) and "torch" in str(evalue):
            outcome.force_exception(pytest.skip.Exception("torch cannot be loaded next to the simulated CUDA runtime"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs")


def _ngpu():
    try:
        import mxnet_b200 as mx
        return mx.num_gpus()
    except Exception:
        return 0


@pytest.fixture(scope="session")
def ngpu():
    return _ngpu()


def pytest_collection_modifyitems(config, items):
    n = None
    for item in items:
        if "multigpu" in item.keywords:
            if n is None:
                n = _ngpu()
            if n < 2:
                item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
