"""modelmesh_b200 — H100-native placement / LRU-eviction solver for ModelMesh (libmmplace).

The product is the CUDA library ``csrc/libmmplace.so`` behind the C ABI of ``include/mmplace.h``; this package is the
ctypes binding used by the tests and bench.py plus the synthetic-fleet generator.  There is no CPU implementation.
"""
from . import _lib  # noqa: F401
from .fleet import Fleet, MmpError  # noqa: F401
