"""granite_b200 -- H100-native (sm_90a) executor for Granite's clustered deferred lighting and
HDR post chain.  The product is the C-ABI shared library libgranite_b200.so (include/granite_b200.h)
plus the C++ host layer mirroring Granite's RenderGraph pass interface; this Python package is the
thin ctypes/torch harness used by the tests and bench.py."""

__all__ = ["capi", "synth", "build"]
