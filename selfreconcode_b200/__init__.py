"""selfrecon-b200: H100-native (sm_90a) implementation of SelfRecon's per-frame hot path.

Layout
  csrc/        CUDA kernels + the C ABI (include/selfrecon_b200.h) -> lib/libselfrecon_b200.so
  _lib.py      ctypes binding of the C ABI
  ops.py       torch-tensor wrappers (torch = memory + streams only)
  dropin/      modules with the reference's import names: FastMinv, MCGpu, GridSamplerMine,
               interp2x_boundary3d/2d, model/, utils/, MCAcc/  (put this directory on sys.path
               ahead of the reference's own packages; see INTEGRATION.md)
  parallel.py  one-process-per-GPU data parallel helpers (NCCL)
  synth.py     seeded synthetic workloads of SURVEY.md section 8d
"""
import os
import sys

__version__ = "0.1.0"

DROPIN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")


def enable_dropin():
    """Puts the drop-in modules (reference import names) at the front of sys.path."""
    if DROPIN_DIR not in sys.path:
        sys.path.insert(0, DROPIN_DIR)
    return DROPIN_DIR
