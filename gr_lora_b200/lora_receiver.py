"""Host-side mirror of the reference's ``lora_receiver`` hier block (python/lora_receiver.py:26-89):
same constructor arguments, same wiring (optional conjugate -> channelizer -> decoder) and the
same 'frames' message port, without GNU Radio.  Decoder and channelizer (SURVEY.md 8f row N1) both run
on the GPU; between them the IQ never leaves device memory."""
from __future__ import annotations

import numpy as np

from . import _native as N
from .decoder import decoder


class _DeviceRow:
    """A zero-copy view of n complex64 samples at a device address, for torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<c8", "data": (int(ptr), False), "version": 3}


class lora_receiver:
    def __init__(self, samp_rate, center_freq, channel_list, bandwidth, sf, implicit, cr, crc, reduced_rate=False,
                 conj=False, decimation=1, disable_channelization=False, disable_drift_correction=False, cfo_feedback=False,
                 sync="reference", sync_word=0x12, implicit_len=0, clock_from_carrier=False, soft=False, antennas=1, crc_list=0,
                 drop_bad_crc=False, max_cfo_hz=0.0, wide_cfo=False, **decoder_kw):
        self.samp_rate, self.center_freq, self.channel_list = samp_rate, center_freq, list(channel_list)
        self.bandwidth, self.sf, self.implicit, self.cr, self.crc = bandwidth, sf, implicit, cr, crc
        self.decimation, self.conj = decimation, conj
        # sync="dechirp": run() goes through the dechirp-synchronised receiver (decoder.receive), which decodes below the
        # noise floor; the default "reference" is the reference's work() state machine
        if sync not in ("reference", "dechirp"):
            raise ValueError(f"sync must be 'reference' or 'dechirp', got {sync!r}")
        self.sync, self.sync_word, self.implicit_len = sync, sync_word, implicit_len
        # clock_from_carrier: the dechirp receiver places every frame's windows with the clock offset its CFO implies
        # (cfo / carrier, one crystal sets a radio's carrier and its sample clock); the carrier is channel_list[0], or
        # center_freq without the channelizer.  The reference state machine tracks drift itself (fine_sync).
        if clock_from_carrier and sync != "dechirp":
            raise ValueError("clock_from_carrier needs sync='dechirp' (the reference state machine has fine_sync)")
        self.clock_from_carrier = bool(clock_from_carrier)
        # soft: the dechirp receiver decodes every code word from its bits' LLRs (soft decisions) instead of from the argmax
        if soft and sync != "dechirp":
            raise ValueError("soft needs sync='dechirp' (the reference state machine makes hard decisions)")
        self.soft = bool(soft)
        # crc_list = K: CRC-aided list decoding of the soft decisions (decoder.receive(..., crc_list=K)); drop_bad_crc: frames
        # whose payload CRC fails are not published (off by default, so that the published stream is the reference's)
        if (crc_list or drop_bad_crc) and sync != "dechirp":
            raise ValueError("crc_list and drop_bad_crc need sync='dechirp'")
        self.crc_list, self.drop_bad_crc = int(crc_list), bool(drop_bad_crc)
        # max_cfo_hz, wide_cfo: the carrier offsets the dechirp receiver searches (decoder.receive(..., max_cfo_hz, wide_cfo));
        # wide_cfo takes max_cfo_hz beyond BW / 4, up to (fs - bw) / 2 of the decoder's rate.  With the channelizer in front,
        # its filter (cutoff bw / 2 + 15 kHz) bounds the offset that reaches the decoder, whatever max_cfo_hz says.
        if (max_cfo_hz or wide_cfo) and sync != "dechirp":
            raise ValueError("max_cfo_hz and wide_cfo need sync='dechirp'")
        self.max_cfo_hz, self.wide_cfo = float(max_cfo_hz), bool(wide_cfo)
        # antennas = M: run() takes an (M, n) capture of M phase-coherent antennas (one LO, one sample clock) and the dechirp
        # receiver combines them (decoder.receive(..., antennas=M)); with the channelizer every antenna gets its own
        # channelizer, which filters and rotates it exactly as the others, so the combining weights stay meaningful
        if antennas != 1 and sync != "dechirp":
            raise ValueError("antennas needs sync='dechirp' (the reference state machine has one input)")
        self.antennas = int(antennas)
        self.disable_channelization = disable_channelization
        self.disable_drift_correction = disable_drift_correction
        self.channelizer = None
        if not disable_channelization:
            # python/lora_receiver.py:52: lora.channelizer(samp_rate, center_freq, channel_list, bandwidth, decimation)
            from .channelizer import channelizer
            self.channelizers = [channelizer(samp_rate, center_freq, self.channel_list, bandwidth, decimation,
                                             device=decoder_kw.get("device", -1)) for _ in range(self.antennas)]
            self.channelizer = self.channelizers[0]
            if conj:                                 # channelizer -> conjugate_cc -> decoder (:62-63,70-75), conjugated on the device
                for ch in self.channelizers:
                    ch.set_conjugate(True)
        if disable_channelization and decimation != 1:
            raise NotImplementedError("fractional_resampler_cc path (python/lora_receiver.py:58-61) is host plumbing, not built")
        # python/lora_receiver.py:53
        if self.antennas != 1:
            decoder_kw.setdefault("n_streams", self.antennas)
        self.decoder = decoder(samp_rate / decimation, bandwidth, sf, implicit, cr, crc, reduced_rate,
                               disable_drift_correction, **decoder_kw)
        if self.decoder.n_streams != self.antennas:
            raise ValueError("lora_receiver feeds one channel (channel_list[0]) to one decoder stream, like the reference; "
                             "use decoder(..., n_streams=N).work_batch for many channels")
        self.frames = self.decoder.frames            # hier-block message port 'frames' (:56,:68)
        # decoder 'control' -> channelizer 'control' (:64): the ("cfo" . x) message the reference's decoder would publish at
        # SYNC (lib/decoder_impl.cc:774-776, commented out there) and lib/controller_impl.cc:52-57 turns into apply_cfo(x).
        # Opt-in here as well: with cfo_feedback the estimates made during a run() retune the channelizer afterwards.
        self.cfo_feedback = bool(cfo_feedback) and self.channelizer is not None
        self._cfo_seen = 0
        if self.cfo_feedback:
            self.decoder.set_cfo_estimate(True)

    def message_port_subscribe(self, handler):
        self.decoder.message_port_subscribe(handler)

    def _front(self, samples):
        x = np.asarray(samples, dtype=np.complex64)
        return np.conj(x) if self.conj else x        # blocks.conjugate_cc, :50,:70-75

    def work(self, samples, stream=0):
        if self.channelizer is None:
            return self.decoder.work(self._front(samples), stream)
        return self.run(samples, stream)

    def run(self, samples, stream=0):
        """Whole capture through (channelizer ->) [conj ->] decoder.  With the channelizer the filtered IQ
        stays in device memory: the decoder consumes the channelizer's output buffer directly.  Only
        channel_list[0] reaches the decoder, as in the reference (lib/channelizer_impl.cc:47,56-57)."""
        if self.antennas != 1:
            return self._run_antennas(samples)
        if self.channelizer is None:
            if self.sync == "dechirp":
                x = np.ascontiguousarray(self._front(samples), np.complex64)
                return self._run_dechirp(x, x.size, int(self.decoder.cfg.max_items_per_call or (1 << 20)))
            return self.decoder.run(self._front(samples), stream)
        x = np.asarray(samples, dtype=np.complex64)
        x = x[: (x.size // self.decimation) * self.decimation]
        limit = int(self.decoder.cfg.max_items_per_call or (1 << 20))
        pos_out, need = 0, 2 * self.decoder.sps
        # the channelizer is stateful (history, rotator), so the capture is filtered once into one device
        # buffer and the decoder walks over it call by call
        n_out = self.channelizer.work(x)
        ptr, stride = self.channelizer.output_ptr(0)
        if self.sync == "dechirp":
            return self._run_dechirp(ptr, n_out, limit) * self.decimation
        while n_out - pos_out >= need:
            n = min(limit, n_out - pos_out)
            c = int(self.decoder.work_batch(ptr + 8 * pos_out, n_items=n, stride_items=n, host=0)[0])
            if c == 0:
                break
            pos_out += c
        if self.cfo_feedback:
            cfo, n = self.decoder.last_cfo(0)
            if n > self._cfo_seen:
                self._cfo_seen = n
                self.channelizer.apply_cfo(cfo)      # channelizer_impl::apply_cfo, lib/channelizer_impl.cc:68-71
        return pos_out * self.decimation

    def _run_antennas(self, samples):
        """An (M, n) capture: each row through its own channelizer, the M filtered rows gathered into one device buffer (device
        to device copies), or the rows straight through; then the dechirp receiver over the M rows as one receiver."""
        x = np.asarray(samples, dtype=np.complex64)
        if x.ndim != 2 or x.shape[0] != self.antennas:
            raise ValueError(f"antennas={self.antennas} needs an ({self.antennas}, n) capture, got shape {x.shape}")
        limit = int(self.decoder.cfg.max_items_per_call or (1 << 20))
        if self.channelizer is None:
            return self._run_dechirp(np.ascontiguousarray(self._front(x)), x.shape[1], limit)
        import torch
        x = x[:, : (x.shape[1] // self.decimation) * self.decimation]
        dev = torch.device("cuda", self.decoder.cfg.device if self.decoder.cfg.device >= 0 else torch.cuda.current_device())
        n_out = [ch.work(row) for ch, row in zip(self.channelizers, x)]
        rows = torch.empty((self.antennas, n_out[0]), dtype=torch.complex64, device=dev)
        torch.cuda.synchronize(dev)                  # (the channelizers run on their own streams)
        for a, ch in enumerate(self.channelizers):
            rows[a].copy_(torch.as_tensor(_DeviceRow(ch.output_ptr(0)[0], n_out[0]), device=dev))
        torch.cuda.synchronize(dev)                  # (receive reads device input on its own stream)
        return self._run_dechirp(int(rows.data_ptr()), n_out[0], limit, stride=n_out[0]) * self.decimation

    def _run_dechirp(self, src, n_out, limit, stride=None):
        """decoder.receive over the channelizer's device output (src: its address) or a host capture (src: ndarray), call by
        call under the consumed rule; every frame is published on the 'frames' port.  Returns the samples consumed.
        A call that consumes nothing while samples remain holds a frame longer than its chunk: the next call presents a
        chunk twice as long (receive() has no per-call size limit), so no frame is lost to the chunk size."""
        pos, n = 0, limit
        carrier = 0.0
        if self.clock_from_carrier:
            carrier = float(self.center_freq if self.channelizer is None else self.channel_list[0])
        while pos < n_out:
            n = min(n, n_out - pos)
            if isinstance(src, np.ndarray):
                part = src[None, pos: pos + n] if src.ndim == 1 else src[:, pos: pos + n]
            else:
                part = src + 8 * pos
            c, frames, _ = self.decoder.receive(part, n_items=n, stride_items=n if stride is None else stride, host=0, sync_word=self.sync_word,
                                                implicit_len=self.implicit_len, carrier_hz=carrier, soft=self.soft,
                                                antennas=self.antennas, crc_list=self.crc_list, max_cfo_hz=self.max_cfo_hz,
                                                wide_cfo=self.wide_cfo)
            crc = self.decoder.frames_crc_last() if self.drop_bad_crc else None
            for k, f in enumerate(frames):
                if crc is not None and crc[k] == N.CRC_BAD:
                    continue
                self.decoder._publish(int(f["stream"]), bytes(f["bytes"][: int(f["len"])]))
            c = int(c[0])
            at_end = pos + n >= n_out
            if c == 0:
                if at_end:
                    break
                n *= 2
                continue
            pos += c
            n = limit
            if at_end:
                break
        return pos
    def get_sf(self):
        return self.sf

    def set_sf(self, sf):                            # :80-82 (decoder warns: unsupported at run time)
        self.sf = sf
        self.decoder.set_sf(sf)

    def get_center_freq(self):
        return self.center_freq
