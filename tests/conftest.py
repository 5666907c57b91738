import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.hookimpl(optionalhook=True)
def pytest_xdist_auto_num_workers(config):
    """`-n auto` (pytest.ini): parallel workers only for the CPU tier; the GPU tier stays in one process (one handle owns the device and its pinned staging)."""
    expr = getattr(config.option, "markexpr", "") or ""
    if "not gpu" in expr:
        return min(4, max(1, (os.cpu_count() or 2) // 2))
    return 0


def pytest_addoption(parser, pluginmanager):
    """pytest.ini passes `-n auto`; without pytest-xdist (or with `-p no:xdist`) accept and ignore it, so that the suite still runs (serially)."""
    if not pluginmanager.hasplugin("xdist"):
        parser.getgroup("xdist-fallback")._addoption("-n", "--numprocesses", dest="numprocesses_ignored", default=None, help="ignored: pytest-xdist is not active")
