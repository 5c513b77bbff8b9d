"""Host-side mirror of the reference's channelizer block over the C ABI (SURVEY.md 8f row N1).

``channelizer(samp_rate, center_freq, channel_list, bandwidth, decimation)`` keeps the constructor of
``lora::channelizer::make`` (include/lora/channelizer.h:49, lib/channelizer_impl.cc:40-60) and its
``apply_cfo`` (:68-71, reached through the "cfo" control message, lib/controller_impl.cc:52-57).  The
filtering (GNU Radio's freq_xlating_fir_filter_ccf with firdes::low_pass taps) runs on the GPU for every
channel of ``channel_list``; the reference wires only channel_list[0]."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N


class channelizer:
    def __init__(self, samp_rate, center_freq, channel_list, bandwidth, decimation, *, device=-1):
        self._L = N.lib()
        self._h = None
        cl = (C.c_float * len(channel_list))(*[float(f) for f in channel_list])
        h = self._L.lora_b200_channelizer_create(float(samp_rate), float(center_freq), cl, len(channel_list),
                                                 int(bandwidth), int(decimation), int(device))
        if not h:
            raise RuntimeError("lora_b200_channelizer_create failed: " + self._L.lora_b200_channelizer_last_error().decode())
        self._h = h
        self.samp_rate, self.center_freq, self.channel_list = samp_rate, center_freq, list(channel_list)
        self.bandwidth, self.decimation = bandwidth, int(decimation)
        self.ntaps = int(self._L.lora_b200_channelizer_ntaps(h))
        self.n_out = 0

    @classmethod
    def make(cls, samp_rate, center_freq, channel_list, bandwidth, decimation, **kw):
        return cls(samp_rate, center_freq, channel_list, bandwidth, decimation, **kw)

    def close(self):
        if self._h:
            self._L.lora_b200_channelizer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, where):
        if rc < 0:
            raise RuntimeError(f"{where} failed ({rc}): " + self._L.lora_b200_channelizer_last_error().decode())

    def taps(self) -> np.ndarray:
        out = np.empty(self.ntaps, np.float32)
        self._check(self._L.lora_b200_channelizer_taps(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), out.size), "channelizer_taps")
        return out

    def apply_cfo(self, cfo, channel=0):
        self._check(self._L.lora_b200_channelizer_apply_cfo(self._h, int(channel), float(cfo)), "channelizer_apply_cfo")

    def set_conjugate(self, on=True):
        """Conjugate every output sample on the device (lora_receiver's optional conjugate_cc, python/lora_receiver.py:70-75)."""
        self._check(self._L.lora_b200_channelizer_set_conjugate(self._h, int(bool(on))), "channelizer_set_conjugate")

    def work(self, samples) -> int:
        """Filter a host buffer (length a multiple of the decimation); the result stays on the device.
        Returns the number of output items per channel."""
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        n = C.c_size_t(0)
        self._check(self._L.lora_b200_channelizer_work_host(self._h, x.ctypes.data, x.size, C.byref(n)), "channelizer_work_host")
        self.n_out = int(n.value)
        return self.n_out

    def output_ptr(self, channel=0):
        """(device pointer, stride in items) of one channel's output of the last work() call."""
        stride = C.c_size_t(0)
        p = self._L.lora_b200_channelizer_output(self._h, int(channel), C.byref(stride))
        return int(p or 0), int(stride.value)

    def read_output(self, channel=0, n_items=None) -> np.ndarray:
        """One channel's output of the last work() call, copied to a host array."""
        n = self.n_out if n_items is None else int(n_items)
        out = np.empty(n, np.complex64)
        self._check(self._L.lora_b200_channelizer_read_output(self._h, int(channel), out.ctypes.data, n), "channelizer_read_output")
        return out

    def work_dev(self, in_dev, n_in, out_dev, out_stride, cuda_stream=0) -> int:
        n = C.c_size_t(0)
        ptr = lambda t: int(t.data_ptr()) if hasattr(t, "data_ptr") else int(t)
        self._check(self._L.lora_b200_channelizer_work_dev(self._h, ptr(in_dev), int(n_in), ptr(out_dev), int(out_stride),
                                                          C.byref(n), int(cuda_stream)), "channelizer_work_dev")
        return int(n.value)


def firdes_low_pass_reference(fs, cutoff, tw):
    """float64 restatement of GNU Radio's firdes::low_pass(1, fs, cutoff, tw, WIN_HAMMING) used by tests to
    check the library's taps (gr-filter is not part of the reference tree: parity is with this formula)."""
    ntaps = int(53.0 * fs / (22.0 * tw))
    ntaps += (ntaps & 1) == 0
    m = (ntaps - 1) // 2
    n = np.arange(-m, m + 1)
    w = 0.54 - 0.46 * np.cos(2 * np.pi * np.arange(ntaps) / (ntaps - 1))
    fw = 2 * np.pi * cutoff / fs
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.where(n == 0, fw / np.pi, np.sin(n * fw) / (n * np.pi)) * w
    return t / t.sum()
