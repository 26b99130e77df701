"""llama.cpp_b200 -- H100-native (sm_90a) quantised mat-mul backend for ggml (the MUL_MAT / MUL_MAT_ID hot path only).

Layout
  csrc/      hand-written sm_90a CUDA + the C ABI (include/b200_qmm.h)  -> libb200qmm.so
  backend/   the ggml backend plugin (ggml_backend_reg_i ... ggml_backend_i) -> libggml-b200.so
  host.py    ctypes binding of the C ABI for the Python test / bench harness (torch only supplies device memory)
  build.py   in-tree build of both shared objects

The product never imports oracle/.
"""
__all__ = ["host", "build"]
