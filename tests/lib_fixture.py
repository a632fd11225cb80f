"""The `lib` fixture of the CPU tests of the C ABI: the library, built first when it is missing.  The entry points check
their arguments before any CUDA work, so these tests need no GPU."""
import os

import pytest


@pytest.fixture(scope='module')
def lib():
    from distributedes_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build_library()
    return _lib.load()
