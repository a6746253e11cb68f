import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """Tests marked `gpu` need a CUDA device AND the built library: without them they are skipped, not failed
    (a plain `pytest tests/` on a CPU host used to report 75 failures that hid real regressions)."""
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    lib = os.path.join(ROOT, "neupan_b200", "lib", "libneupan_b200.so")
    if have_gpu and not os.path.exists(lib):
        raise pytest.UsageError(f"CUDA device present but {lib} is missing: run `python -m neupan_b200.build` (no CPU fallback)")
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100, -m gpu)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True)
def _inference_tests_run_without_autograd(request):
    """With autograd recording, PAN.forward runs in differentiable mode and returns tensors that require grad (the reference's
    behaviour: cvxpylayers builds the graph to NRMP.adjust_parameters).  The parity / feature tests are about inference, so they
    run under torch.no_grad(); the modules that test gradients, the facade's info tensors or training manage grad mode themselves."""
    name = request.module.__name__
    if name in ("test_gpu_grad", "test_facade", "test_gpu_train", "test_dune_train"):
        yield
        return
    import torch

    with torch.no_grad():
        yield
