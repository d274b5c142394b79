"""parsec_b200 -- H100-native device-side DAG execution engine behind PaRSEC's device API.

Only what the hot path needs lives here: ``csrc/`` (the sm_90a kernels, the C-ABI library and the
host-side mirror of the reference's device module / DSL hooks) and thin ctypes mirrors of that ABI.
"""
from . import _lib  # noqa: F401
from ._lib import Pb2Error  # noqa: F401

__all__ = ["_lib", "Pb2Error"]
