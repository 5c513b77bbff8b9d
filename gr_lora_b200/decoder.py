"""Host-side mirror of the reference's decoder block over the C ABI.

``decoder`` keeps the name, constructor arguments, ``set_sf``/``set_samp_rate`` behaviour,
stdout side effects and message-port semantics of ``gr::lora::decoder``
(include/lora/decoder.h:693-709, lib/decoder_impl.cc:41-122, 740-915) so that tests read like
the reference's own; the GNU Radio scheduler is replaced by ``run()`` (a fake scheduler
honouring ``set_output_multiple(2*sps)`` and the consume protocol).  All arithmetic happens in
liblora_b200.so on the GPU: there is no Python/NumPy compute path here.
"""
from __future__ import annotations

import ctypes as C
import sys

import numpy as np

from . import _native as N
from .loraphy import parse_frame

LORATAP_LEN = 15   # sizeof(loratap_header_t), include/lora/loratap.h:48-55
LORAPHY_LEN = 3    # sizeof(loraphy_header_t), include/lora/loraphy.h:25-32


def _dev_ptr(x) -> int:
    """Device pointer of a torch tensor / anything with data_ptr(), or a raw int."""
    if x is None:
        return 0
    if hasattr(x, "data_ptr"):
        return int(x.data_ptr())
    return int(x)


class decoder:
    """lora.decoder(samp_rate, bandwidth, sf, implicit, cr, crc, reduced_rate, disable_drift_correction)

    Extra keyword arguments select what the reference cannot express: ``n_streams`` independent
    (channel, SF) streams sharing the configuration, the demodulator (``"gradient"`` = the
    reference's live path, ``"fft"`` = the north-star dechirp+FFT path) and the CUDA device.
    """

    def __init__(self, samp_rate, bandwidth, sf, implicit, cr, crc, reduced_rate=False,
                 disable_drift_correction=False, *, n_streams=1, demod="gradient", device=-1,
                 max_items_per_call=0, max_frames_per_call=0, trace_capacity=0, quiet=False):
        self._L = N.lib()
        self._h = None
        demod_id = {"gradient": N.DEMOD_GRADIENT, "fft": N.DEMOD_FFT}[demod] if isinstance(demod, str) else int(demod)
        cfg = N.Config(samp_rate=float(samp_rate), bandwidth=int(bandwidth), sf=int(sf), implicit=int(bool(implicit)),
                       cr=int(cr), crc=int(bool(crc)), reduced_rate=int(bool(reduced_rate)),
                       disable_drift_correction=int(bool(disable_drift_correction)), demod=demod_id,
                       n_streams=int(n_streams), device=int(device), max_items_per_call=int(max_items_per_call),
                       max_frames_per_call=int(max_frames_per_call), trace_capacity=int(trace_capacity))
        self.cfg = cfg
        h = self._L.lora_b200_create(C.byref(cfg))
        if not h:
            msg = self._L.lora_b200_last_error().decode(errors="replace")
            if sf < 6 or sf > 13:
                # the reference prints this to std::cerr and exit(1)s (lib/decoder_impl.cc:57-61)
                print(msg, file=sys.stderr)
                raise SystemExit(1)
            raise RuntimeError("lora_b200_create failed: " + msg)
        self._h = h
        self.n_streams = int(n_streams)
        self.sps = self._L.lora_b200_samples_per_symbol(h)
        self.n_bins = self._L.lora_b200_bins(h)
        self.decim = self._L.lora_b200_decimation(h)
        self.quiet = quiet
        self.frames = []            # what was published on message port "frames": (stream, bytes)
        self.implicit = bool(implicit)
        self.header_checks = {"ok": 0, "bad": 0}   # explicit-header checksum of the published frames (loraphy.py; the
                                                   # reference never checks it, include/lora/utilities.h:396-404)
        self._handlers = []
        self._cb = N.FRAME_CB(self._on_frame)
        buf = C.create_string_buffer(512)
        self._L.lora_b200_banner(h, buf, len(buf))
        self.banner = buf.value.decode()
        if not quiet:
            sys.stdout.write(self.banner)     # lib/decoder_impl.cc:93-103

    # -- gr::lora::decoder::make -------------------------------------------------------------
    @classmethod
    def make(cls, samp_rate, bandwidth, sf, implicit, cr, crc, reduced_rate, disable_drift_correction, **kw):
        return cls(samp_rate, bandwidth, sf, implicit, cr, crc, reduced_rate, disable_drift_correction, **kw)

    def close(self):
        if self._h:
            self._L.lora_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- unsupported setters, lib/decoder_impl.cc:905-915 --------------------------------------
    def set_sf(self, sf):
        self._L.lora_b200_set_sf(self._h, int(sf))
        print(self._L.lora_b200_last_error().decode(), file=sys.stderr)

    def set_samp_rate(self, samp_rate):
        self._L.lora_b200_set_samp_rate(self._h, float(samp_rate))
        print(self._L.lora_b200_last_error().decode(), file=sys.stderr)

    # -- message port "frames" -----------------------------------------------------------------
    def message_port_subscribe(self, handler):
        """handler(stream, frame_bytes) is called for every published frame."""
        self._handlers.append(handler)

    def _on_frame(self, _user, stream, data, length):
        self._publish(int(stream), bytes(C.string_at(data, length)))

    def _publish(self, stream, blob):
        self.frames.append((int(stream), blob))
        if not self.implicit and len(blob) >= 18:     # side channel only: the published bytes are never touched
            self.header_checks["ok" if parse_frame(blob).header_ok else "bad"] += 1
        for h in self._handlers:
            h(int(stream), blob)

    def output_multiple(self):
        return 2 * self.sps          # set_output_multiple, lib/decoder_impl.cc:91

    # -- work(): one scheduler call -------------------------------------------------------------
    def work(self, input_items, stream=0):
        """Hand a host buffer of gr_complex to the GPU state machine; returns items consumed.
        Frames completed inside the call are published before it returns."""
        x = np.ascontiguousarray(input_items, dtype=np.complex64)
        consumed = C.c_size_t(0)
        N.check(self._L.lora_b200_work(self._h, int(stream), x.ctypes.data, x.size, C.byref(consumed), self._cb, None),
                "lora_b200_work")
        self._emit_stdout(stream)
        return int(consumed.value)

    FRAME_DTYPE = np.dtype([("stream", "<u4"), ("seq", "<u4"), ("len", "<u4"), ("n_hdr_print", "u1"), ("hdr_print", "u1", (4,)),
                            ("pad", "u1", (3,)), ("bytes", "u1", (564,))])

    def frames_last(self) -> np.ndarray:
        """Structured array (FRAME_DTYPE) of the frames the last work call published, in delivery order: the bulk
        alternative to one Python callback per frame (lora_b200_frames_last)."""
        ptr = C.c_void_p(0)
        n = int(self._L.lora_b200_frames_last(self._h, C.byref(ptr)))
        if n == 0:
            return np.zeros(0, self.FRAME_DTYPE)
        buf = C.string_at(ptr.value, n * self.FRAME_DTYPE.itemsize)
        return np.frombuffer(buf, dtype=self.FRAME_DTYPE)

    def frames_crc_last(self) -> np.ndarray:
        """uint8 per frame of frames_last(): the payload CRC status (lora_b200_frames_crc_last) -- N.CRC_NONE (no CRC in the
        header, or a payload under 2 bytes), CRC_OK, CRC_BAD or CRC_RECOVERED (OK after list decoding, receive(crc_list=K))."""
        ptr = C.c_void_p(0)
        n = int(self._L.lora_b200_frames_crc_last(self._h, C.byref(ptr)))
        return np.frombuffer(C.string_at(ptr.value, n), dtype=np.uint8).copy() if n else np.zeros(0, np.uint8)

    def work_batch(self, iq, n_items=None, stride_items=None, host=None, sc16_scale=None, callbacks=True, sc8_scale=None):
        """All streams at once. ``iq``: host ndarray [n_streams, n_items] (complex64, or int16 / int8 [n_streams, n_items, 2]
        together with ``sc16_scale`` / ``sc8_scale``) or a device tensor/pointer.  ``sc16_scale`` / ``sc8_scale`` select the
        int16 / int8 I/Q entry points: the device computes x * scale, PCIe moves 4 / 2 bytes per sample."""
        if isinstance(iq, np.ndarray) and (sc16_scale is not None or sc8_scale is not None):
            x = np.ascontiguousarray(iq, dtype=np.int16 if sc16_scale is not None else np.int8)
            assert x.ndim == 3 and x.shape[0] == self.n_streams and x.shape[2] == 2
            ptr, n_items, stride_items, host = x.ctypes.data, x.shape[1], x.shape[1], 1
        elif isinstance(iq, np.ndarray):
            x = np.ascontiguousarray(iq, dtype=np.complex64)
            assert x.ndim == 2 and x.shape[0] == self.n_streams
            ptr, n_items, stride_items, host = x.ctypes.data, x.shape[1], x.shape[1], 1
        else:
            ptr = _dev_ptr(iq)                                    # device tensor, or a raw host / device address with host=1 / 0
            host = 0 if host is None else int(host)
            if stride_items is None:
                stride_items = n_items
        consumed = np.zeros(self.n_streams, dtype=np.uint64)      # size_t[n_streams]
        cptr = consumed.ctypes.data_as(C.POINTER(C.c_size_t))
        cb = self._cb if callbacks else N.FRAME_CB()              # callbacks=False: drain with frames_last() instead
        if sc16_scale is not None:
            N.check(self._L.lora_b200_work_batch_sc16(self._h, ptr, float(sc16_scale), int(n_items), int(stride_items), host,
                                                      cptr, cb, None), "lora_b200_work_batch_sc16")
        elif sc8_scale is not None:
            N.check(self._L.lora_b200_work_batch_sc8(self._h, ptr, float(sc8_scale), int(n_items), int(stride_items), host,
                                                     cptr, cb, None), "lora_b200_work_batch_sc8")
        else:
            N.check(self._L.lora_b200_work_batch(self._h, ptr, int(n_items), int(stride_items), host, cptr, cb, None),
                    "lora_b200_work_batch")
        if not self.quiet:
            for s in range(self.n_streams):
                self._emit_stdout(s)
        return consumed.astype(np.int64)

    RX_INFO_DTYPE = np.dtype([("start", "<u8"), ("data_start", "<u8"), ("stream", "<u4"), ("cfo_hz", "<f4"), ("snr_db", "<f4"),
                              ("sfo_ppm", "<f4")])       # struct lora_b200_rx_info

    def receive(self, iq, n_items=None, stride_items=None, host=None, sync_word=0x12, implicit_len=0, min_preamble=0,
                max_cfo_hz=0.0, sfo_ppm=0.0, carrier_hz=0.0, soft=False, antennas=1, crc_list=0, wide_cfo=False,
                fine_toa=False):
        """The dechirp-synchronised receiver (lora_b200_receive): decodes frames below the noise floor.  ``iq`` as for
        work_batch (host ndarray [n_streams, n_items] or a device tensor / pointer).  Returns (consumed, frames, info):
        consumed[s] = where stream s must be re-presented from, frames = FRAME_DTYPE records, info = RX_INFO_DTYPE records
        (first preamble sample, first data sample, stream, CFO in Hz, SNR in dB in the LoRa bandwidth, clock offset in ppm),
        one per frame.  Clock offset of a frame: sfo_ppm, plus its CFO / carrier_hz when carrier_hz (the channel's RF
        frequency) is given -- one crystal sets a radio's carrier and its sample clock.  soft: decode every code word from
        its bits' LLRs (the spectrum of each data window, demod_llr) to the most likely nibble, instead of from the argmax.
        ``self.header_drops`` counts the explicit headers of the call whose checksum failed.
        antennas = M (1..4, dividing n_streams): rows g M .. g M + M - 1 are the phase-coherent antennas of receiver g
        (lora_b200_receive_antennas): combined screen and synchronisation, maximum-ratio-combined data windows; consumed has
        one entry per receiver, frames and info carry stream = g and the combined SNR, and rx_channels_last() gives each
        frame's channel estimates.
        crc_list = K (1..12, needs soft): a frame whose payload CRC fails gets its K least reliable code words tried at their
        runner-up nibbles, and the cheapest combination that satisfies the CRC is published (frames_crc_last() reports it
        RECOVERED).  A frame whose errors lie outside the list passes a wrong combination with probability about
        (2^K - 1) / 2^16; 0 (the default) is off.
        wide_cfo: receive frames up to max_cfo_hz off carrier (finite, in (0, (fs - bw) / 2]: 3.5 bw at fs/bw = 8, bw / 2 at 2,
        7.5 bw at 16, 15.5 bw at 32),
        beyond the BW / 4 to which max_cfo_hz is clamped without it.  The screen then searches coarse offsets c * bw / 2,
        c = -C..C, C = ceil((max_cfo_hz - bw / 4) / (bw / 2)), each costing about one more screen.
        fine_toa: also time each published frame's arrival to a fraction of a sample from its dechirped preamble and SFD
        windows, read with rx_toa_last() afterwards; nothing published changes."""
        if isinstance(iq, np.ndarray):
            x = np.ascontiguousarray(iq, dtype=np.complex64)
            assert x.ndim == 2 and x.shape[0] == self.n_streams
            ptr, n_items, stride_items, host = x.ctypes.data, x.shape[1], x.shape[1], 1
        else:
            ptr = _dev_ptr(iq)
            if n_items is None and hasattr(iq, "shape"):
                n_items = int(iq.shape[-1])
            host = 0 if host is None else int(host)
            if stride_items is None:
                stride_items = n_items
        p = N.RxParams(sync_word=int(sync_word) & 0xFF, implicit_len=int(implicit_len), min_preamble=int(min_preamble),
                       max_cfo_hz=float(max_cfo_hz), sfo_ppm=float(sfo_ppm), carrier_hz=float(carrier_hz), soft=int(soft),
                       crc_list=int(crc_list), wide_cfo=int(wide_cfo), fine_toa=int(fine_toa))
        m = int(antennas)
        consumed = np.zeros(max(self.n_streams // m, 1) if m > 0 else 1, dtype=np.uint64)
        cptr = consumed.ctypes.data_as(C.POINTER(C.c_size_t))
        if m == 1:
            N.check(self._L.lora_b200_receive(self._h, ptr, int(n_items), int(stride_items), host, C.byref(p), cptr), "lora_b200_receive")
        else:
            N.check(self._L.lora_b200_receive_antennas(self._h, ptr, int(n_items), int(stride_items), host, m, C.byref(p), cptr),
                    "lora_b200_receive_antennas")
        iptr, drops = C.c_void_p(0), C.c_uint32(0)
        n = int(self._L.lora_b200_rx_info_last(self._h, C.byref(iptr), C.byref(drops)))
        info = (np.frombuffer(C.string_at(iptr.value, n * self.RX_INFO_DTYPE.itemsize), dtype=self.RX_INFO_DTYPE) if n
                else np.zeros(0, self.RX_INFO_DTYPE))
        self.header_drops = int(drops.value)
        return consumed.astype(np.int64), self.frames_last(), info

    def rx_toa_last(self) -> np.ndarray:
        """float64 per frame of the last receive(..., fine_toa=True) call, parallel to its frames (lora_b200_rx_toa_last): the
        row position, in that call's coordinates like info["start"], at which the frame's first preamble sample arrived, to a
        fraction of a sample (NaN for a frame without a preamble or SFD window inside the row).  Empty after a call without
        fine_toa and after work()."""
        ptr = C.c_void_p(0)
        n = int(self._L.lora_b200_rx_toa_last(self._h, C.byref(ptr)))
        if n == 0:
            return np.zeros(0, np.float64)
        return np.frombuffer(C.string_at(ptr.value, n * 8), dtype=np.float64).copy()

    def rs_toa(self, iq_dev, n_items, group, start, cfo_bins, sfo_ppm, antennas=1, stride=0):
        """The fine time of arrival of given frames on its own (lora_b200_rs_toa_dev): frame i at start[i] with cfo_bins[i] and
        sfo_ppm[i] on receiver group[i] (rows group[i] * M + a, `stride` items apart).  Returns (nu_a, nu_b, toa): the peaks
        of the preamble and SFD window powers in bins from the CFO, and the time of arrival.  group, start, cfo_bins, sfo_ppm:
        host sequences of one length."""
        g = np.ascontiguousarray(group, dtype=np.uint32)
        s = np.ascontiguousarray(start, dtype=np.int64)
        f = np.ascontiguousarray(cfo_bins, dtype=np.float32)
        q = np.ascontiguousarray(sfo_ppm, dtype=np.float32)
        assert g.shape == s.shape == f.shape == q.shape and g.ndim == 1
        nu_a, nu_b, toa = np.zeros(g.size, np.float32), np.zeros(g.size, np.float32), np.zeros(g.size, np.float64)
        N.check(self._L.lora_b200_rs_toa_dev(self._h, _dev_ptr(iq_dev), int(n_items), int(antennas), int(stride or n_items), g.size,
                                            g.ctypes.data, s.ctypes.data, f.ctypes.data, q.ctypes.data, nu_a.ctypes.data,
                                            nu_b.ctypes.data, toa.ctypes.data), "lora_b200_rs_toa_dev")
        return nu_a, nu_b, toa

    def rx_channels_last(self) -> np.ndarray:
        """[n_frames, M] complex64: each antenna's channel estimate for every frame of the last receive(..., antennas=M) call,
        parallel to its frames (lora_b200_rx_channels_last): the mean preamble peak over (1 + j) sps, the amplitude per
        sample with a phase reference common to the frame's antennas.  Empty after a one-antenna call."""
        ptr, m = C.c_void_p(0), C.c_uint32(0)
        n = int(self._L.lora_b200_rx_channels_last(self._h, C.byref(ptr), C.byref(m)))
        m = max(int(m.value), 1)
        if n == 0:
            return np.zeros((0, m), np.complex64)
        return np.frombuffer(C.string_at(ptr.value, n * m * 8), dtype=np.complex64).reshape(n, m).copy()

    def _emit_stdout(self, stream):
        if self.quiet:
            return
        buf = C.create_string_buffer(1 << 16)
        n = self._L.lora_b200_stdout_last(self._h, int(stream), buf, len(buf))
        if n > 0:
            sys.stdout.write(buf.value.decode(errors="replace"))   # lib/decoder_impl.cc:832,872

    def run(self, samples, stream=0, chunk_items=None):
        """Fake GNU Radio scheduler over a whole capture (host array): repeatedly calls work()
        with at least 2*sps items and drops what work() consumed.  Returns total consumed."""
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        limit = chunk_items or (self.cfg.max_items_per_call or (1 << 20))
        pos, need = 0, 2 * self.sps
        while x.size - pos >= need:
            c = self.work(x[pos:pos + limit], stream)
            if c == 0:
                break
            pos += c
        return pos

    def set_cfo_estimate(self, enable=True):
        """Also run the reference's experimental_determine_cfo at every SYNC (lib/decoder_impl.cc:730-738,774); off by default."""
        N.check(self._L.lora_b200_set_cfo_estimate(self._h, int(bool(enable))), "lora_b200_set_cfo_estimate")

    def last_cfo(self, stream=0):
        """(latest CFO estimate in Hz, number of estimates so far) of a stream."""
        cfo, n = C.c_float(0.0), C.c_uint32(0)
        N.check(self._L.lora_b200_last_cfo(self._h, int(stream), C.byref(cfo), C.byref(n)), "lora_b200_last_cfo")
        return float(cfo.value), int(n.value)

    def reset(self):
        """Every stream back to a freshly made block's state (a flowgraph restart); buffers and tables are kept."""
        N.check(self._L.lora_b200_reset(self._h), "lora_b200_reset")
        self.frames = []

    def state(self, stream=0):
        return N.check(self._L.lora_b200_stream_state(self._h, int(stream)), "lora_b200_stream_state")

    def trace(self, stream=0):
        cap = max(int(self.cfg.trace_capacity), 1)
        steps = (N.Step * cap)()
        n = C.c_size_t(0)
        rc = self._L.lora_b200_trace_read(self._h, int(stream), steps, cap, C.byref(n))
        if rc not in (N.OK, N.EOVERFLOW):
            N.check(rc, "lora_b200_trace_read")
        m = min(int(n.value), cap)
        return [(steps[i].state, steps[i].consumed, steps[i].bin, steps[i].fine_sync, steps[i].metric) for i in range(m)]

    # -- batch kernels (device-resident) ---------------------------------------------------------
    def demod_fft(self, iq_dev, n_symbols, bins_dev, mags_dev=None, cuda_stream=0):
        """K1 on device memory: dechirp + FFT + argmax of n_symbols aligned windows."""
        N.check(self._L.lora_b200_demod_fft_dev(self._h, _dev_ptr(iq_dev), int(n_symbols), _dev_ptr(bins_dev),
                                               _dev_ptr(mags_dev), int(cuda_stream)), "lora_b200_demod_fft_dev")

    def demod_fft_antennas(self, iq_dev, n_groups, n_antennas, n_symbols, row_stride, bins_dev, mags_dev, cuda_stream=0):
        """The combined screen of the several-antenna receiver (lora_b200_demod_fft_antennas_dev): n_groups groups of n_antennas
        rows (row_stride items apart) of n_symbols aligned windows; bins_dev / mags_dev[g * n_symbols + i] = the first argmax
        of sum_a |tmp_a|^2 over the group's windows i and its square root."""
        N.check(self._L.lora_b200_demod_fft_antennas_dev(self._h, _dev_ptr(iq_dev), int(n_groups), int(n_antennas), int(n_symbols),
                                                        int(row_stride), _dev_ptr(bins_dev), _dev_ptr(mags_dev), int(cuda_stream)),
                "lora_b200_demod_fft_antennas_dev")

    def demod_llr(self, iq_dev, n_symbols, llrs_dev, bins_dev=None, reduced=False, cuda_stream=0):
        """Soft output of n_symbols aligned windows (lora_b200_demod_llr_dev): llrs_dev[i * ppm + j] = the max-log LLR of bit
        j of symbol i's demodulated word in magnitude units (> 0: bit 0), ppm = sf - 2 with reduced, else sf; bins_dev
        (optional) = the argmax bins of demod_fft."""
        N.check(self._L.lora_b200_demod_llr_dev(self._h, _dev_ptr(iq_dev), int(n_symbols), int(bool(reduced)), _dev_ptr(llrs_dev),
                                               _dev_ptr(bins_dev), int(cuda_stream)), "lora_b200_demod_llr_dev")

    def rs_window(self, iq_dev, n_items, pos, cfo_bins, up, bins, out_dev, energy_dev=None, argmax_bins_dev=None, argmax_mags_dev=None,
                  antennas=1, stride=0):
        """The dechirp receiver's window sums (lora_b200_rs_window_dev) on `antennas` rows of n_items samples, `stride` items
        apart: out_dev[i * M + a] (complex64) = bin bins[i] of antenna a's window at pos[i], dechirped with the up-chirp (up[i])
        or the down-chirp and de-rotated by cfo_bins[i] bins; energy_dev[i * M + a] = its energy; argmax_bins_dev[i] (int32)
        / argmax_mags_dev[i] = the argmax bin and magnitude of the combined spectrum of the raw windows at pos[i] (each
        output but out_dev optional).  pos, cfo_bins, up, bins: host sequences of one length."""
        p = np.ascontiguousarray(pos, dtype=np.int64)
        f = np.ascontiguousarray(cfo_bins, dtype=np.float32)
        u = np.ascontiguousarray(up, dtype=np.int32)
        b = np.ascontiguousarray(bins, dtype=np.int32)
        assert p.shape == f.shape == u.shape == b.shape and p.ndim == 1
        N.check(self._L.lora_b200_rs_window_dev(self._h, _dev_ptr(iq_dev), int(n_items), int(antennas), int(stride), p.size,
                                               p.ctypes.data, f.ctypes.data, u.ctypes.data, b.ctypes.data, _dev_ptr(out_dev),
                                               _dev_ptr(energy_dev), _dev_ptr(argmax_bins_dev), _dev_ptr(argmax_mags_dev)),
                "lora_b200_rs_window_dev")

    def rs_frame(self, iq_dev, n_items, group, start, cfo_bins, sfo_ppm, first, cnt, windows_dev, chan_dev=None, snr_dev=None,
                 antennas=1, stride=0):
        """The channel estimates, weights and data windows of given frames (lora_b200_rs_frame_dev): frame i at start[i] with
        cfo_bins[i] and sfo_ppm[i] on receiver group[i] (rows group[i] * M + a, `stride` items apart).  M >= 2: chan_dev[i]
        (complex64[8]) = h[4] | w[4], snr_dev[i] = the combined SNR in dB.  windows_dev[(i * cnt + k) * sps ..] = its data
        window first + k, combined over the antennas and de-rotated by its CFO.  group, start, cfo_bins, sfo_ppm: host
        sequences of one length."""
        g = np.ascontiguousarray(group, dtype=np.uint32)
        s = np.ascontiguousarray(start, dtype=np.int64)
        f = np.ascontiguousarray(cfo_bins, dtype=np.float32)
        q = np.ascontiguousarray(sfo_ppm, dtype=np.float32)
        assert g.shape == s.shape == f.shape == q.shape and g.ndim == 1
        N.check(self._L.lora_b200_rs_frame_dev(self._h, _dev_ptr(iq_dev), int(n_items), int(antennas), int(stride or n_items), g.size,
                                              g.ctypes.data, s.ctypes.data, f.ctypes.data, q.ctypes.data, int(first), int(cnt),
                                              _dev_ptr(chan_dev), _dev_ptr(snr_dev), _dev_ptr(windows_dev)),
                "lora_b200_rs_frame_dev")

    def demod_fft_host(self, iq_host, bins_out=None, mags_out=None):
        """K1 end to end from host memory (copies inside). iq_host: complex64 ndarray or (ptr, n_symbols)."""
        if isinstance(iq_host, tuple):
            ptr, n = int(iq_host[0]), int(iq_host[1])
        else:
            x = np.ascontiguousarray(iq_host, dtype=np.complex64)
            ptr, n = x.ctypes.data, x.size // self.sps
        bins = np.empty(n, np.uint32) if bins_out is None else bins_out
        mags = np.empty(n, np.float32) if mags_out is None else mags_out
        bp = bins.ctypes.data if isinstance(bins, np.ndarray) else int(bins)
        mp = mags.ctypes.data if isinstance(mags, np.ndarray) else int(mags)
        N.check(self._L.lora_b200_demod_fft_host(self._h, ptr, n, bp, mp), "lora_b200_demod_fft_host")
        return bins, mags

    def demod_fft_host_sc16(self, iq_sc16, scale, bins_out=None, mags_out=None):
        """K1 end to end from int16 I/Q host memory. iq_sc16: int16 ndarray [..., 2] or (ptr, n_symbols)."""
        if isinstance(iq_sc16, tuple):
            ptr, n = int(iq_sc16[0]), int(iq_sc16[1])
        else:
            x = np.ascontiguousarray(iq_sc16, dtype=np.int16)
            ptr, n = x.ctypes.data, x.size // (2 * self.sps)
        bins = np.empty(n, np.uint32) if bins_out is None else bins_out
        mags = np.empty(n, np.float32) if mags_out is None else mags_out
        bp = bins.ctypes.data if isinstance(bins, np.ndarray) else int(bins)
        mp = mags.ctypes.data if isinstance(mags, np.ndarray) else int(mags)
        N.check(self._L.lora_b200_demod_fft_host_sc16(self._h, ptr, float(scale), n, bp, mp), "lora_b200_demod_fft_host_sc16")
        return bins, mags

    def tx_symbols(self, values_dev, out_dev, n_symbols, noise_sigma=0.0, seed=0, cfo_hz_dev=None, up_table_dev=None, cuda_stream=0):
        """Synthetic aligned data symbols on the device (chirp shift = value, optional per-symbol CFO and AWGN)."""
        N.check(self._L.lora_b200_tx_symbols_dev(self._h, _dev_ptr(up_table_dev), _dev_ptr(values_dev), _dev_ptr(cfo_hz_dev), float(noise_sigma), int(seed),
                                                int(n_symbols), _dev_ptr(out_dev), int(cuda_stream)), "lora_b200_tx_symbols_dev")

    def tx_expand(self, base_dev, k, n_items, n_streams, out_dev, noise_sigma=0.0, seed=0, cuda_stream=0):
        """n_streams channels from k base captures plus every stream's own AWGN, on the device."""
        N.check(self._L.lora_b200_tx_expand_dev(self._h, _dev_ptr(base_dev), int(k), int(n_items), float(noise_sigma), int(seed),
                                               int(n_streams), _dev_ptr(out_dev), int(cuda_stream)), "lora_b200_tx_expand_dev")

    TX_FRAME_DTYPE = np.dtype([("start", "<u8"), ("stream", "<u4"), ("n_symbols", "<u4"), ("cfo_hz", "<f4"), ("sync_word", "u1"),
                               ("pad", "u1", (3,))])     # struct lora_b200_tx_frame

    def tx_encode(self, payloads_dev, offsets, lengths, shifts_dev, max_symbols, cuda_stream=0):
        """Frame encoder on the device: frame f = payloads_dev[offsets[f] .. + lengths[f]) (host arrays offsets, lengths) ->
        chirp shifts_dev[f * max_symbols + i] for its tx_frame_symbols() data symbols, as tx.encode_frame gives them."""
        off = np.ascontiguousarray(offsets, dtype=np.uint32)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        assert off.shape == ln.shape and off.ndim == 1
        N.check(self._L.lora_b200_tx_encode_dev(self._h, _dev_ptr(payloads_dev), off.ctypes.data, ln.ctypes.data, ln.size,
                                               _dev_ptr(shifts_dev), int(max_symbols), int(cuda_stream)), "lora_b200_tx_encode_dev")

    def tx_frames(self, frames, shifts_dev, max_symbols, n_streams, n_items, out_dev, noise_sigma=0.0, seed=0, up_table_dev=None,
                  cuda_stream=0, sfo_ppm=None):
        """Whole streams of frames on the device: out_dev [n_streams, n_items] cf32.  frames: structured array of TX_FRAME_DTYPE
        (host, any order); frame f's data symbols are shifts_dev[f * max_symbols ..].  sfo_ppm: None, or one clock offset
        per frame (lora_b200_tx_frames_sfo_dev)."""
        fr = np.ascontiguousarray(frames, dtype=self.TX_FRAME_DTYPE)
        if sfo_ppm is None:
            N.check(self._L.lora_b200_tx_frames_dev(self._h, _dev_ptr(up_table_dev), C.cast(fr.ctypes.data, C.POINTER(N.TxFrame)),
                                                   fr.size, _dev_ptr(shifts_dev), int(max_symbols), float(noise_sigma), int(seed),
                                                   int(n_streams), int(n_items), _dev_ptr(out_dev), int(cuda_stream)),
                    "lora_b200_tx_frames_dev")
            return
        ppm = np.ascontiguousarray(sfo_ppm, dtype=np.float32)
        if ppm.shape != fr.shape:
            raise ValueError(f"sfo_ppm needs one value per frame: shape {ppm.shape}, frames {fr.shape}")
        N.check(self._L.lora_b200_tx_frames_sfo_dev(self._h, _dev_ptr(up_table_dev), C.cast(fr.ctypes.data, C.POINTER(N.TxFrame)),
                                                   fr.size, ppm.ctypes.data, _dev_ptr(shifts_dev), int(max_symbols),
                                                   float(noise_sigma), int(seed), int(n_streams), int(n_items), _dev_ptr(out_dev),
                                                   int(cuda_stream)), "lora_b200_tx_frames_sfo_dev")

    def synth_streams(self, payloads_per_stream, n_items, *, lead_symbols=3.0, gap_symbols=4.0, sync_word=0x12, cfo_hz=0.0,
                      noise_sigma=0.0, seed=0, up_table_dev=None, sfo_ppm=0.0):
        """Stream s of a [len(payloads_per_stream), n_items] cf32 device tensor carries the frames of payloads_per_stream[s]
        under this decoder's sf / cr / implicit / crc / reduced_rate, laid out as tx.channel does it: int(lead_symbols * sps)
        of silence, then every frame followed by int(gap_symbols * sps) of silence.  A frame is placed while it and the gap
        after it fit in the row.  cfo_hz and sfo_ppm (the transmitter's clock offset, tx_frames_sfo): one value for every
        frame, or a sequence per stream with one value per payload; a frame with a clock offset is as long as
        tx.drifted_length makes it.  Encoding (tx_encode) and modulation (tx_frames) run on the device, on torch's current
        stream.  Returns (tensor, [(stream, start, payload) of every placed frame])."""
        import torch
        from .tx import drifted_length
        sps, lead, gap = self.sps, int(lead_symbols * self.sps), int(gap_symbols * self.sps)
        n_sym = {}
        placed, rows, ppms = [], [], []
        for s, pays in enumerate(payloads_per_stream):
            pos = lead
            for k, p in enumerate(pays):
                p = bytes(p)
                if len(p) not in n_sym:
                    n_sym[len(p)] = int(self._L.lora_b200_tx_frame_symbols(C.byref(self.cfg), len(p)))
                    if n_sym[len(p)] == 0:
                        raise ValueError(f"payload length {len(p)} is not encodable under this configuration")
                ppm = float(sfo_ppm if np.isscalar(sfo_ppm) else sfo_ppm[s][k])
                flen = drifted_length((12 + n_sym[len(p)]) * sps + sps // 4, ppm)
                if pos + flen + gap > n_items:
                    break
                placed.append((s, pos, p))
                ppms.append(ppm)
                rows.append((pos, s, n_sym[len(p)], float(cfo_hz if np.isscalar(cfo_hz) else cfo_hz[s][k]), int(sync_word) & 0xFF))
                pos += flen + gap
        dev = torch.device("cuda", self.cfg.device if self.cfg.device >= 0 else torch.cuda.current_device())
        stream = torch.cuda.current_stream(dev).cuda_stream
        lengths = np.array([len(p) for _, _, p in placed], np.uint32)
        offsets = (np.cumsum(lengths, dtype=np.uint64) - lengths).astype(np.uint32)
        max_symbols = max([n for _, _, n, _, _ in rows], default=8)
        blob = b"".join(p for _, _, p in placed)
        pay = torch.from_numpy(np.frombuffer(blob, np.uint8).copy()).to(dev) if blob else torch.zeros(1, dtype=torch.uint8, device=dev)
        shifts = torch.empty(max(len(placed), 1) * max_symbols, dtype=torch.int32, device=dev)
        self.tx_encode(pay, offsets, lengths, shifts, max_symbols, stream)
        frames = np.zeros(len(rows), self.TX_FRAME_DTYPE)
        for f, (start, s, n, cfo, sw) in enumerate(rows):
            frames[f] = (start, s, n, cfo, sw, (0, 0, 0))
        out = torch.empty((len(payloads_per_stream), n_items), dtype=torch.complex64, device=dev)
        self.tx_frames(frames, shifts, max_symbols, len(payloads_per_stream), n_items, out, noise_sigma, seed, up_table_dev, stream,
                       sfo_ppm=ppms if any(ppms) else None)
        return out, placed

    def ifreq(self, iq_dev, n_windows, window, out_dev, cuda_stream=0):
        """A3 instantaneous_frequency of n_windows windows of `window` samples (device tensors)."""
        N.check(self._L.lora_b200_ifreq_dev(self._h, _dev_ptr(iq_dev), int(n_windows), int(window), _dev_ptr(out_dev),
                                           int(cuda_stream)), "lora_b200_ifreq_dev")

    def demod_gradient(self, iq_dev, n_symbols, bins_dev, cuda_stream=0):
        N.check(self._L.lora_b200_demod_gradient_dev(self._h, _dev_ptr(iq_dev), int(n_symbols), _dev_ptr(bins_dev),
                                                    int(cuda_stream)), "lora_b200_demod_gradient_dev")

    def decode_codewords(self, cw_dev, lengths_dev, stride, cr_dev, is_header_dev, n_vec, out_dev, out_stride,
                         out_len_dev, cuda_stream=0):
        N.check(self._L.lora_b200_decode_codewords_dev(self._h, _dev_ptr(cw_dev), _dev_ptr(lengths_dev), int(stride),
                                                      _dev_ptr(cr_dev), _dev_ptr(is_header_dev), int(n_vec),
                                                      _dev_ptr(out_dev), int(out_stride), _dev_ptr(out_len_dev),
                                                      int(cuda_stream)), "lora_b200_decode_codewords_dev")

    def deinterleave(self, words_dev, n_words, ppm, n_blocks, cw_dev, cuda_stream=0):
        N.check(self._L.lora_b200_deinterleave_dev(self._h, _dev_ptr(words_dev), int(n_words), int(ppm), int(n_blocks),
                                                  _dev_ptr(cw_dev), int(cuda_stream)), "lora_b200_deinterleave_dev")

    # -- tables ------------------------------------------------------------------------------------
    def tables_bytes(self):
        return int(self._L.lora_b200_tables_bytes(self._h))

    def tables_export(self) -> np.ndarray:
        out = np.empty(self.tables_bytes(), np.uint8)
        N.check(self._L.lora_b200_tables_export(self._h, out.ctypes.data, out.size), "lora_b200_tables_export")
        return out

    def tables_import(self, blob):
        b = np.ascontiguousarray(blob, dtype=np.uint8)
        N.check(self._L.lora_b200_tables_import(self._h, b.ctypes.data, b.size), "lora_b200_tables_import")

    def tables_device_view(self):
        """Zero-copy view of the device table blob as an object with __cuda_array_interface__
        (wrap with torch.as_tensor(view, device="cuda") for the init-time NCCL broadcast)."""
        ptr, n = int(self._L.lora_b200_tables_device_ptr(self._h)), self.tables_bytes()

        class _View:
            __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}
        return _View()

    def tables_commit(self):
        N.check(self._L.lora_b200_tables_commit(self._h), "lora_b200_tables_commit")

    def launch_count(self):
        return int(self._L.lora_b200_launch_count(self._h))


def tables_build_host(samp_rate=1e6, bandwidth=125000, sf=7) -> np.ndarray:
    """The chirp/ifreq/twiddle blob built on the host only (no GPU needed)."""
    L = N.lib()
    cfg = N.Config(samp_rate=float(samp_rate), bandwidth=int(bandwidth), sf=int(sf), n_streams=1)
    n = L.lora_b200_tables_build_host(C.byref(cfg), None, 0)
    if not n:
        raise RuntimeError(L.lora_b200_last_error().decode())
    out = np.empty(n, np.uint8)
    L.lora_b200_tables_build_host(C.byref(cfg), out.ctypes.data, out.size)
    return out


def tx_frame_symbols(payload_len, sf, cr, implicit, crc, reduced_rate, samp_rate=1e6, bandwidth=125000) -> int:
    """Data symbols (8-symbol header block + payload blocks) of one frame carrying payload_len bytes; 0 for an unsupported
    configuration or length (host only, lora_b200_tx_frame_symbols)."""
    cfg = N.Config(samp_rate=float(samp_rate), bandwidth=int(bandwidth), sf=int(sf), implicit=int(bool(implicit)), cr=int(cr),
                   crc=int(bool(crc)), reduced_rate=int(bool(reduced_rate)), n_streams=1)
    return int(N.lib().lora_b200_tx_frame_symbols(C.byref(cfg), int(payload_len)))


def split_tables(blob: np.ndarray, sps: int) -> dict:
    """Views into the blob: layout documented in include/lora_b200.h."""
    o, out = 0, {}
    for name, dt, n in (("downchirp", np.complex64, sps), ("upchirp", np.complex64, sps),
                        ("downchirp_ifreq", np.float32, sps), ("upchirp_ifreq", np.float32, sps),
                        ("upchirp_ifreq_v", np.float32, 3 * sps), ("twiddles", np.complex64, sps)):
        nb = np.dtype(dt).itemsize * n
        out[name] = blob[o:o + nb].view(dt)
        o += nb
    return out


def dissect_frame(blob: bytes):
    """(loratap, phy header, payload) of a published frame (lib/decoder_impl.cc:588-601)."""
    return blob[:LORATAP_LEN], blob[LORATAP_LEN:LORATAP_LEN + LORAPHY_LEN], blob[LORATAP_LEN + LORAPHY_LEN:]
