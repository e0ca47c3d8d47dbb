"""bwa-mem2_b200 — H100-native seed-and-extend hot path of bwa-mem2 behind a C ABI.

The product is `libbm2b200.so` (csrc/, hand-written CUDA for sm_90a; include/bm2_b200.h).
This Python package is only the host-side mirror used by tests and bench: a ctypes binding
(`capi`), the synthetic-input generator (`synth`) and index tooling (`index_build`).
Import name: `bwa_mem2_b200` (the directory name carries the reference's hyphen; use
`__graft_entry__.load_package()`).
"""
from . import capi  # noqa: F401
