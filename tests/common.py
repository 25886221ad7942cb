"""Constants and Java long arithmetic shared by the restatements (tests/*_oracle.py) and the tests: one definition each."""
import ctypes as C

from modelmesh_b200.synth import LONG_MAX  # noqa: F401  (Long.MAX_VALUE)

HOUR = 3_600_000
EXPIRY = 900_000        # LOAD_FAILURE_EXPIRY_MS
GONE_MS = 600_000       # ASSUME_INSTANCE_GONE_AFTER_MS
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def jlong(x: int) -> int:
    return ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)


def jdiv(a: int, b: int) -> int:
    """Java long a / b (truncates toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def jsub(a: int, b: int) -> int:
    """Java long a - b"""
    return ((int(a) - int(b) + (1 << 63)) % (1 << 64)) - (1 << 63)
