import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import binding
    binding.build()
    return binding.lib()


@pytest.fixture(scope="session")
def emul_lib():
    """CPU harness: the product's host code + the single-lane shape of the decision routine (tests/emul)."""
    from modelmesh_b200 import _lib
    here = os.path.join(ROOT, "tests", "emul")
    so = os.path.join(here, "_build", "libmmplace_emul.so")
    srcs = [os.path.join(here, "emul.cpp"), os.path.join(ROOT, "modelmesh_b200", "csrc", "host_state.hpp"),
            os.path.join(ROOT, "modelmesh_b200", "csrc", "place_core.cuh"), os.path.join(ROOT, "include", "mmplace.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so, srcs[0]])
    return _lib.load(so, require_all=False)


@pytest.fixture(scope="session")
def product_lib():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from modelmesh_b200 import _lib
    return _lib.load_product()
