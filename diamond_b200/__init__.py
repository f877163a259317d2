"""diamond_b200 — GPU-native (H100, sm_90a) implementation of DIAMOND's data-parallel hot path.

Host code is Python/PyTorch and mirrors the reference's module surface (eloialonso/diamond, src/models/...);
every conv / norm / attention / SiLU on the path runs in hand-written CUDA kernels behind the C ABI declared in
include/diamond_b200.h (libdiamond_b200.so, built in-tree by __graft_entry__.build()).
There is no CPU or eager-PyTorch fallback: using a model without the library, or on a non-CUDA tensor, raises.
"""
__version__ = "0.1.0"
