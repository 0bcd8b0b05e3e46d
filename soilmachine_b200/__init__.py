"""soilmachine_b200 -- H100-native particle/terrain hot path of weigert/SoilMachine.

The product is lib/libsoilmachine_b200.so (CUDA, sm_90a) behind the C ABI in
include/soilmachine_b200.h; `capi` is a thin ctypes binding used by tests and bench.py.
"""
from . import capi  # noqa: F401
from .capi import Context, SoilMachineError  # noqa: F401
