"""dalle_mtf_b200 — H100-native (sm_90a) engine behind the DALLE-mtf config / model_fn surface.

Only what the data-parallel training hot path needs lives here:
  csrc/            hand-written CUDA kernels + the C ABI (include/dalle_b200.h) -> libdalle_b200.so
  lib.py, ops.py   ctypes binding and tensor-level wrappers
  (host-side mirrors of the reference interface are added next to these)
"""
__version__ = "0.1.0"
