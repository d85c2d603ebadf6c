"""cocosnet_b200 — H100-native (sm_90a) hot path of CoCosNet.

Layout:
  csrc/            hand-written CUDA kernels + the C-ABI (libcocos_b200.so)
  _lib.py          ctypes binding of include/cocos_b200.h (no CPU fallback)
  ops.py           torch-tensor wrappers + autograd Functions over the C-ABI
  networks/ ...    host-side mirror of the reference module API
"""
__version__ = "0.1.0"
