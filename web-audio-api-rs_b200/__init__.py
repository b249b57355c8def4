"""web-audio-api-rs_b200 — H100-native render-quantum engine for web-audio-api-rs's OfflineAudioContext path.

The directory name carries a hyphen (it mirrors the reference's name), so import it through
`__graft_entry__.load_package()` / tests/conftest.py, which register it as `web_audio_api_rs_b200`.

Layout:
  csrc/            hand-written sm_90a CUDA kernels + the C-ABI implementation (include/wae.h)
  _binding.py      ctypes view of the C ABI
  context.py       host-side mirror of the reference's control API (OfflineAudioContext, AudioNode, AudioParam)

There is NO CPU fallback: `engine()` raises if libwae_b200.so is missing or no GPU is usable.
"""
import ctypes
import os

from . import _binding
from ._binding import Api, WaeError
from .context import *  # noqa: F401,F403
from . import context
from . import parallel

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwae_b200.so")

_api = None


def api():
    """Bind libwae_b200.so (built in-tree by __graft_entry__.build()). Fails loudly when absent."""
    global _api
    if _api is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback in this package)")
        _api = Api(ctypes.CDLL(LIB_PATH), "wae_")
    return _api


class Engine:
    """wae_engine_create(device_ordinal): one engine per GPU / process rank."""

    def __init__(self, device=0):
        a = api()
        h = ctypes.c_void_p()
        a.check(a.engine_create(int(device), ctypes.byref(h)))
        self.handle = h
        self.backend = context.Backend(a, h, int(device))
        self.device = device

    def set_option(self, option, value):
        a = api()
        a.check(a.engine_set_option(self.handle, option, int(value)))

    def stream(self):
        a = api()
        p = ctypes.c_void_p()
        a.check(a.engine_stream(self.handle, ctypes.byref(p)))
        return p.value

    def context(self, number_of_channels, length, sample_rate):
        return context.OfflineAudioContext(number_of_channels, length, sample_rate, self.backend)

    def resample(self, samples, from_rate, to_rate):
        """AudioBuffer::resample of one channel on the GPU (wae_resample_linear; src/buffer.rs:311-363)."""
        import math
        import numpy as np
        a = api()
        x = np.ascontiguousarray(samples, np.float32)
        cap = max(len(x), int(math.ceil(len(x) * (float(to_rate) / float(from_rate)))) + 1)
        out = np.zeros(cap, np.float32)
        n = ctypes.c_uint64(0)
        fp = ctypes.POINTER(ctypes.c_float)
        a.check(a.resample_linear(self.handle, x.ctypes.data_as(fp), len(x), float(from_rate), float(to_rate),
                                  out.ctypes.data_as(fp), cap, ctypes.byref(n)))
        return out[:n.value]

    def close(self):
        if self.handle:
            self.backend.close_batches()
            api().engine_destroy(self.handle)
            self.handle = None


OPT_CHUNK_FRAMES, OPT_FUSE, OPT_SERIAL_FILTERS, OPT_PIPELINE_GROUPS, OPT_PARAM_PARALLEL = 1, 2, 3, 4, 5
OPT_BIND_NUMA, OPT_HOST_WORKERS, OPT_CHAIN_TMA, OPT_CHAIN_WAVES, OPT_CHAIN_PREPASS, OPT_VOICE_SUM = 6, 7, 8, 9, 10, 11
