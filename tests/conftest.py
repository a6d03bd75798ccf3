import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


@pytest.hookimpl(tryfirst=True)
def pytest_cmdline_main(config):
    """The CPU tier (``-m "not gpu"``) is dominated by multi-process gloo tests that spend their time spawning workers
    and importing torch: run it on 4 xdist workers when pytest-xdist is available and no ``-n`` was given
    (``TORCHACC_B200_TEST_WORKERS=0`` keeps it serial).  The GPU tiers are never parallelised: their tests share one
    device and the driver inspects the pytest process itself."""
    try:
        n = int(os.environ.get("TORCHACC_B200_TEST_WORKERS", "4"))
    except ValueError:
        n = 0
    opt = config.option
    if (n > 1 and getattr(opt, "markexpr", "") == "not gpu" and config.pluginmanager.hasplugin("xdist")
            and not getattr(opt, "numprocesses", None) and not getattr(opt, "usepdb", False)
            and not os.environ.get("PYTEST_XDIST_WORKER")):
        opt.numprocesses = n
        if getattr(opt, "dist", "no") == "no":
            opt.dist = "load"
    return None


def pytest_collection_modifyitems(config, items):
    import torch
    has_gpu = torch.cuda.is_available()
    ngpu = torch.cuda.device_count() if has_gpu else 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    """On a GPU box the native library must exist: build it in-tree if it is missing."""
    import torch
    if torch.cuda.is_available():
        from torchacc_b200 import _native
        if not _native.available():
            from torchacc_b200 import build_native
            build_native.build()
            _native._TRIED = False
            assert _native.available()
    yield
