import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


# The driver runs `pytest -x`: one failing auxiliary test must never hide the hot-path parity rows (round-1 lesson).
# Hot-path parity files are collected first, the input-pipeline (SURVEY 8f N4) tests last.
_ORDER = ["test_gpu_a_parity", "test_gpu_b_tc", "test_gpu_c_plugin", "test_gpu_d_", "test_gpu_z_augment"]


def pytest_collection_modifyitems(session, config, items):
    def rank(item):
        name = os.path.basename(str(item.fspath))
        for i, prefix in enumerate(_ORDER):
            if name.startswith(prefix):
                return i
        return -1 if not name.startswith("test_gpu") else len(_ORDER) - 1
    items.sort(key=rank)            # stable: order within a file is kept
