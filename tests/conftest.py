"""pytest configuration: registers the `gpu` marker and exposes the two shared libraries.

* `lib`  -- whisper.cpp_b200/libwhisper_b200.so, the product (C ABI of include/whisper_b200.h)
* `ref`  -- oracle/_ref/libwhisper_ref.so, the UNMODIFIED reference CPU build (test infrastructure only)
"""
import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def ref():
    from wbtest import load_ref
    return load_ref()


@pytest.fixture(scope="session")
def lib():
    from wbtest import load_lib
    return load_lib()
