"""actionmesh_b200 — H100-native (sm_90a) Stage-I denoising hot path of ActionMesh behind the reference's own seams.

Host code is Python/PyTorch plumbing; all arithmetic runs in hand-written CUDA kernels loaded through a C ABI
(include/actionmesh_b200.h).  There is no CPU fallback: importing the package is cheap, but every op raises if
libactionmesh_b200.so has not been built.
"""
from ._lib import AmbError, load_library  # noqa: F401

__all__ = ["AmbError", "load_library"]
