"""etl_b200 — H100-native batched pgoutput (CDC) decode engine for supabase/etl's streaming hot path.

Layout:
  csrc/        hand-written sm_90a CUDA kernels + the extern "C" ABI (include/etl_decode.h)
  abi.py       ctypes binding of that ABI (what a Rust/cgo/JNI shim would bind; see INTEGRATION.md)
  decoder.py   host-side mirror of the reference interface for this path
  pgoutput.py  wire-format writer (fixtures, synthetic workloads)
  workloads.py the BASELINE.json stream shapes (C1..C5)
"""
__version__ = "0.1.0"
