"""Fixtures the test modules share; a module imports the ones it uses (`from gpu_fixtures import ctx, pkg`)."""
import importlib

import pytest

TH = (2, 3, 4, 5, 6, 8, 12, 16, 64)         # rows per warp (CFB_TH) a split test covers


@pytest.fixture(scope="module")
def pkg():
    return importlib.import_module("cineform-sdk_b200")


@pytest.fixture(scope="module")
def ctx():
    """One CUDA context on device 0 for the module."""
    c = importlib.import_module("cineform-sdk_b200").Context(0)
    yield c
    c.close()


@pytest.fixture
def splits(monkeypatch):
    """splits(values) iterates over `values` with CFB_TH set to each (the library reads it at every launch)."""
    def gen(values=TH):
        for th in values:
            monkeypatch.setenv("CFB_TH", str(th))
            yield th
    return gen
