import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # The reference is not deterministic on a dirty heap for some FLUSH sequences (brotli_libs.zeroed_malloc): the CPU suite,
    # whose randomized sim tests can meet such a sequence, runs with zeroed malloc.  The GPU suite (-m gpu) keeps the allocator
    # as it is: none of its call sequences runs a block across the ring's end in the first lap behind a short first write, and
    # nothing about the process that drives CUDA should differ from a user's.
    markexpr = (getattr(config.option, "markexpr", "") or "").replace(" ", "")
    if markexpr != "gpu":
        from brotli_libs import zeroed_malloc
        zeroed_malloc()
