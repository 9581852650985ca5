"""dasr_b200 — H100-native (sm_90a) implementation of the DASR SRN training / inference hot path.

Layout:
  csrc/     hand-written CUDA kernels + the C ABI (include/dasr_b200.h)  -> lib/libdasr_b200.so
  _lib.py   ctypes binding;  ops.py  typed wrappers;  engine.py  whole-network runners / autograd nodes
  srn/      drop-in mirror of the reference's codes/SRN python API (models, options, utils)
  dp.py     data-parallel gradient all-reduce (one flat bucket per step)
"""
__version__ = '0.1.0'
