import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")
    # The CPU oracle runs on oneDNN: on boxes whose CPU quota is far below the visible core count (GPU box:
    # 128 visible, 16 usable) the default thread count makes it ~25x slower.
    import torch
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


# Run order: the north-star path (MI-GAN generator, its ops) first, then the widened rows (uint8 path, Co-Mod-GAN,
# staged paths), so that under `-x` a failure in a newer row cannot hide the state of the headline path.
_ORDER = ["test_oracle", "test_host", "test_split_precision", "test_generator_gpu", "test_ops_gpu", "test_parallel",
          "test_u8_gpu", "test_comodgan_emul", "test_comodgan_gpu", "test_staged_gpu"]


def pytest_collection_modifyitems(session, config, items):
    def key(item):
        name = os.path.splitext(os.path.basename(str(item.fspath)))[0]
        return _ORDER.index(name) if name in _ORDER else len(_ORDER)
    items.sort(key=key)          # stable: order inside a file is kept


@pytest.fixture(scope="session")
def lib():
    """The C-ABI library, built on demand (nvcc cross-compiles without a GPU)."""
    import migan_b200
    from migan_b200 import _abi

    migan_b200.build.build()
    return _abi.load()


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("this test is marked gpu but no CUDA device is visible")
    return torch.device("cuda:0")
