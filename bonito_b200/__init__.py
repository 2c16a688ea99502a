"""
bonito_b200: H100-native drop-in for the chunked forward + decode path of nanoporetech/bonito.

Mirrors the reference's plugin surface for that path (`bonito.nn` registry, `bonito.util`
loader / chunking helpers, `bonito.crf.Model` + `basecall`) over hand-written sm_90a kernels
reached through the C ABI in include/bonito_b200.h.
"""

__version__ = "0.1.0"

import os as _os

# The tile-pipelined engine drives up to 16 CUDA streams; with the default of 8 hardware work queues streams that share
# a queue pick up false dependencies.  Must be set before the CUDA context exists; respects an explicit user setting.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
