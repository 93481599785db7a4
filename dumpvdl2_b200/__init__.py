"""dumpvdl2_b200 — H100 (sm_90a) implementation of dumpvdl2's per-channel DSP hot path.

Only what the path needs lives here: csrc/ (CUDA kernels + C-ABI, built into libvdl2gpu.so),
api.py (ctypes mirror of the reference's process_buf_* / frame-push interface), synth.py (synthetic
VDL2 burst generator for tests and the benchmark), build.py (nvcc driver).
"""
from .api import (Vdl2Channels, Vdl2Receivers, Vdl2MixedReceivers, Vdl2GpuError, Frame, load_library, FMT_U8, FMT_S16, FLAG_TRACE, FLAG_KEEP_DEC,
                  FLAG_K1_SCALAR, FLAG_NO_OVERLAP, FLAG_NO_GRAPH, FLAG_RAGGED, FLAG_INPUT_LEVELS, level_metrics,
                  FLAG_CHANNEL_LEVELS, channel_level_metrics, FLAG_SPECTRUM, spectrum_metrics, LIB_PATH)

__all__ = ["Vdl2Channels", "Vdl2Receivers", "Vdl2MixedReceivers", "Vdl2GpuError", "Frame", "load_library", "FMT_U8", "FMT_S16", "FLAG_TRACE",
           "FLAG_KEEP_DEC", "FLAG_K1_SCALAR", "FLAG_NO_OVERLAP", "FLAG_NO_GRAPH", "FLAG_RAGGED", "FLAG_INPUT_LEVELS", "level_metrics", "FLAG_CHANNEL_LEVELS",
           "channel_level_metrics", "FLAG_SPECTRUM", "spectrum_metrics", "LIB_PATH"]
