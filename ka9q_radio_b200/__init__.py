"""ka9q_radio_b200 -- H100-native overlap-save channelizer behind ka9q-radio's filter.h surface.

Only what the hot path needs lives here: csrc/ (hand-written sm_90a kernels + the C-ABI shared
library libka9qgpu.so) and thin host-side mirrors (capi.py: ctypes binding of include/ka9q_gpu.h;
channelizer.py: a torch-tensor convenience wrapper used by tests and bench.py).
"""
from . import capi  # noqa: F401
from .capi import KGPU_COMPLEX, KGPU_REAL, KGPU_FMT_F32, KGPU_FMT_I16, KgpuError  # noqa: F401
