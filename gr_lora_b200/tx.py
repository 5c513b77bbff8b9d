"""Synthetic LoRa transmitter + channel model (SURVEY.md 8f N3).

The reference is receive-only (README.md:5; the only encoder fragment is
``hamming_encode_soft``, include/lora/utilities.h:257-264) and ships no IQ fixtures, so
every test/bench input is produced here.  The encoder is the exact inverse of the decode
chain in lib/decoder_impl.cc (B1-B5 of SURVEY.md 8a):

    payload bytes -> nibbles (payload: low nibble first, :701-704; header: high first)
                  -> Hamming(8,4) code word            (utilities.h:257-264)
                  -> XOR whitening sequence             (inverse of dewhiten :639-652)
                  -> bit shuffle                        (inverse of deshuffle :611-624)
                  -> diagonal interleave                (inverse of deinterleave :535-565)
                  -> Gray decode                        (inverse of :512)
                  -> x4 for reduced-rate symbols        (inverse of :508)
                  -> chirp cyclically shifted by (g + 1) bins, because the reference's live
                     gradient demodulator returns (shift - 1) mod N (SURVEY 8a row A7).

Frame layout as the reference state machine expects it (SURVEY.md 3.3): n_preamble
upchirps, two sync-word upchirps, 2.25 downchirps, 8 reduced-rate header-block symbols,
payload blocks of (4 + cr) symbols.

This module is host-side numpy (small cases, fixtures).  bench.py generates the large
device-resident batches with the same chirp definition.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from . import whitening

SHUFFLE_PATTERN = (5, 0, 1, 2, 4, 3, 6, 7)  # lib/decoder_impl.cc:568


def hamming84_encode(nibble: int) -> int:
    """Hamming(8,4) code word, bit layout p1 d0 d1 d2 p2 d3 p3 p4 (LSB first),
    include/lora/utilities.h:257-264."""
    b = [(nibble >> i) & 1 for i in range(4)]
    p1 = b[1] ^ b[2] ^ b[3]
    p2 = b[0] ^ b[1] ^ b[2]
    p3 = b[0] ^ b[1] ^ b[3]
    p4 = b[0] ^ b[2] ^ b[3]
    bits = (p1, b[0], b[1], b[2], p2, b[3], p3, p4)
    return sum(v << i for i, v in enumerate(bits))


HAMMING84 = tuple(hamming84_encode(n) for n in range(16))


def shuffle_byte(v: int) -> int:
    """Inverse of deshuffle (:616-624): deshuffle does out[j] = in[pattern[j]]."""
    r = 0
    for j, src in enumerate(SHUFFLE_PATTERN):
        r |= ((v >> j) & 1) << src
    return r


def rotr(bits: int, count: int, size: int) -> int:
    mask = (1 << size) - 1
    count %= size
    bits &= mask
    return ((bits >> count) | (bits << (size - count))) & mask


def gray_decode(word: int) -> int:
    """Inverse of ``bin ^ (bin >> 1)`` (:512)."""
    b = 0
    while word:
        b ^= word
        word >>= 1
    return b


def interleave_block(codewords, n_words: int, ppm: int):
    """Inverse of deinterleave (:535-553): RX takes bit x of rotl(word_i, i) as bit i of
    code word x."""
    assert len(codewords) == ppm
    words = []
    for i in range(n_words):
        v = 0
        for x in range(ppm):
            v |= ((codewords[x] >> i) & 1) << x
        words.append(rotr(v, i, ppm))
    return words


def header_checksum(length: int, cr: int, has_crc: int) -> int:
    """5-bit LoRa explicit-header checksum.  The reference never verifies it
    (include/lora/utilities.h:396-404) but its README golden ``04 90 40`` carries it
    (README.md:67-71): len 4, cr 4, crc on -> 0b00100."""
    h0 = [(length >> (4 + i)) & 1 for i in range(4)]
    h1 = [(length >> i) & 1 for i in range(4)]
    v2 = ((cr & 7) << 1) | (has_crc & 1)
    h2 = [(v2 >> i) & 1 for i in range(4)]
    c4 = h0[3] ^ h0[2] ^ h0[1] ^ h0[0]
    c3 = h0[3] ^ h1[3] ^ h1[2] ^ h1[1] ^ h2[0]
    c2 = h0[2] ^ h1[3] ^ h1[0] ^ h2[3] ^ h2[1]
    c1 = h0[1] ^ h1[2] ^ h1[0] ^ h2[2] ^ h2[1] ^ h2[0]
    c0 = h0[0] ^ h1[1] ^ h2[3] ^ h2[2] ^ h2[1] ^ h2[0]
    return (c4 << 4) | (c3 << 3) | (c2 << 2) | (c1 << 1) | c0


def header_bytes(length: int, cr: int, has_crc: int) -> bytes:
    """The 3 bytes memcpy'd into loraphy_header_t (lib/decoder_impl.cc:833,
    include/lora/loraphy.h:25-32): length | (cr<<5 | crc<<4 | chk4) | (chk3..0 << 4)."""
    chk = header_checksum(length, cr, has_crc)
    return bytes([length & 0xFF, ((cr & 7) << 5) | ((has_crc & 1) << 4) | (chk >> 4), (chk & 0xF) << 4])


def payload_crc(payload: bytes) -> int:
    """Semtech's payload CRC of ``payload`` (L >= 2 bytes, without the CRC): CRC-16, polynomial 0x1021, initial value 0, no
    reflection, no final XOR, over payload[0 .. L-2), XORed with payload[L-1] | payload[L-2] << 8.  de ad be ef -> 0xEC80."""
    if len(payload) < 2:
        raise ValueError("the payload CRC needs at least 2 payload bytes")
    crc = 0
    for b in payload[:-2]:
        crc ^= b << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x1021) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return crc ^ payload[-1] ^ (payload[-2] << 8)


def _data_projection(w: int, cr: int) -> int:
    """The nibble the decode chain makes of a dewhitened byte w: the nearest Hamming(8,4) code word's data (the lowest nibble
    on ties) for CR 4/7 and 4/8, the data bits 1, 2, 3, 5 for CR 4/5 and 4/6 (lib/decoder_impl.cc:654-706)."""
    if cr >= 3:
        return min(range(16), key=lambda s: (bin(w ^ HAMMING84[s]).count("1"), s))
    return ((w >> 1) & 1) | (((w >> 2) & 1) << 1) | (((w >> 3) & 1) << 2) | (((w >> 5) & 1) << 3)


def crc_whitening(length: int, cr: int) -> int:
    """W(L): what the decode chain, which dewhitens every payload nibble, makes of an unwhitened CRC of 0 after an L-byte
    payload -- the data projection of whitening bytes 2L .. 2L+3, published low byte first.  L = 4: 0xE1F0."""
    prng = whitening.payload_sequence(cr)
    nib = [_data_projection(prng[i] if i < len(prng) else 0, cr) for i in range(2 * length, 2 * length + 4)]
    return nib[0] | nib[1] << 4 | nib[2] << 8 | nib[3] << 12


def crc_bytes(payload: bytes, cr: int) -> bytes:
    """The two bytes to append to ``payload`` so that encode_frame(payload + crc_bytes(payload, cr), ...) is the frame a
    radio sends: encode_frame whitens every byte it is given, the radio does not whiten its CRC, so the CRC goes in as
    crc ^ W(L).  The decoder publishes these same two bytes, and the frame checks."""
    v = payload_crc(payload) ^ crc_whitening(len(payload), cr)
    return bytes([v & 0xFF, v >> 8])


def payload_symbols_expected(payload_len: int, cr: int, sf: int, reduced_rate: bool) -> int:
    """Number of payload symbols the reference will read (lib/decoder_impl.cc:842-847),
    evaluated with the same fp32 expressions."""
    spb = cr + 4
    bits_needed = np.float32(payload_len) * np.float32(8.0)
    symbols_needed = bits_needed * (np.float32(spb) / np.float32(4.0)) / np.float32(sf - (2 if reduced_rate else 0))
    blocks = int(math.ceil(float(np.float32(symbols_needed) / np.float32(spb))))
    return blocks * spb


@dataclass
class FrameSymbols:
    """Chirp shifts (in bins, 0..N-1) of the data part of one frame."""
    shifts: list
    n_header_symbols: int = 8
    words: list = field(default_factory=list)       # Gray-coded words as the RX sees them
    codewords: list = field(default_factory=list)   # whitened+shuffled code words


def encode_frame(payload: bytes, sf: int, cr: int, *, explicit: bool = True, has_crc: bool = True,
                 reduced_rate: bool = False, header: bytes | None = None, min_payload_symbols: int | None = None) -> FrameSymbols:
    """Encode ``payload`` (the bytes the reference prints after the header, i.e. including the
    two MAC CRC bytes when has_crc) into chirp shifts.

    explicit: a 3-byte PHY header (``header`` or header_bytes(len(payload)-2*crc, cr, crc))
    occupies the first 5 code words of the 8-symbol header block (:612,631-633).
    """
    n_bins = 1 << sf
    ppm_hdr = sf - 2
    ppm_pay = sf - 2 if reduced_rate else sf
    prng = whitening.payload_sequence(cr)

    # payload code words: low nibble first (:701-704, swap_nibbles :663)
    pay_cw = []
    for b in payload:
        pay_cw += [b & 0xF, b >> 4]
    n_pay_cw_needed = len(pay_cw)

    hdr_cw = []
    if explicit:
        if header is None:
            length = len(payload) - (2 if has_crc else 0)
            header = header_bytes(length, cr, 1 if has_crc else 0)
        nib = [header[0] >> 4, header[0] & 0xF, header[1] >> 4, header[1] & 0xF, header[2] >> 4]
        hdr_cw = [HAMMING84[n] ^ whitening.PRNG_HEADER[i] for i, n in enumerate(nib)]

    spare = ppm_hdr - len(hdr_cw)                    # SF-7 (explicit) or SF-2 (implicit) code words
    # how many payload blocks: enough for our code words AND what the RX will read (:842-847)
    rest = max(0, n_pay_cw_needed - spare)
    n_blocks = -(-rest // ppm_pay)
    if explicit:
        rx_syms = payload_symbols_expected(len(payload), cr, sf, reduced_rate)
        n_blocks = max(n_blocks, rx_syms // (cr + 4))
    if min_payload_symbols is not None:
        n_blocks = max(n_blocks, -(-min_payload_symbols // (cr + 4)))
    total_cw = spare + n_blocks * ppm_pay
    pay_cw = pay_cw + [0] * (total_cw - len(pay_cw))

    def whiten(i, nibble, nbits):
        w = HAMMING84[nibble] ^ (prng[i] if i < len(prng) else 0)
        return shuffle_byte(w) & ((1 << nbits) - 1)

    coded = [whiten(i, n, 8 if i < spare else 4 + cr) for i, n in enumerate(pay_cw)]

    words, shifts, all_cw = [], [], []
    # header block: 8 symbols, ppm = SF-2, always reduced rate (:495,521-523)
    blk = [shuffle_byte(c) for c in hdr_cw] + coded[:spare]
    all_cw += blk
    for w in interleave_block(blk, 8, ppm_hdr):
        words.append(w)
        g = (4 * gray_decode(w)) % n_bins            # inverse of lround(bin/4) % N_hdr (:508)
        shifts.append((g + 1) % n_bins)
    pos = spare
    for _ in range(n_blocks):
        blk = coded[pos:pos + ppm_pay]
        pos += ppm_pay
        all_cw += blk
        for w in interleave_block(blk, 4 + cr, ppm_pay):
            words.append(w)
            g = gray_decode(w)
            if reduced_rate:
                g = (4 * g) % n_bins
            shifts.append((g + 1) % n_bins)
    return FrameSymbols(shifts=shifts, words=words, codewords=all_cw)


# ---------------------------------------------------------------------------------------
# modulation
# ---------------------------------------------------------------------------------------
def base_upchirp(sf: int, bw: float = 125e3, fs: float = 1e6) -> np.ndarray:
    """Unit-amplitude upchirp over one symbol, same phase law as the reference's ideal
    chirp (lib/decoder_impl.cc:149-160: phase = -2*pi*t*(bw/2 - 0.5*bw*sym_rate*t)),
    evaluated in float64.  Cyclic shifts of it are phase continuous."""
    n_bins = 1 << sf
    sym_rate = bw / n_bins
    sps = int(fs / sym_rate)
    t = np.arange(sps, dtype=np.float64) / fs
    phase = -2.0 * np.pi * t * (bw / 2.0 + (-0.5 * bw * sym_rate) * t)
    return np.exp(1j * phase)


def modulate_shifts(shifts, sf: int, bw: float = 125e3, fs: float = 1e6) -> np.ndarray:
    up = base_upchirp(sf, bw, fs)
    sps = up.size
    decim = sps // (1 << sf)
    idx = (np.arange(sps)[None, :] + (np.asarray(shifts, dtype=np.int64)[:, None] * decim)) % sps
    return up[idx].reshape(-1)


def drifted_length(n_samples: int, sfo_ppm: float) -> int:
    """Receiver samples of a frame of n_samples transmitter samples sent with a clock off by sfo_ppm: those n >= 0 with
    n (1 + delta) < n_samples, delta = float32(sfo_ppm) * 1e-6 (the arithmetic of lora_b200_tx_frames_sfo_dev)."""
    rate = 1.0 + 1e-6 * float(np.float32(sfo_ppm))
    n = int(math.ceil(n_samples / rate))
    while n and (n - 1) * rate >= n_samples:
        n -= 1
    while n * rate < n_samples:
        n += 1
    return n


def modulate_frame(fs_syms: FrameSymbols, sf: int, *, bw: float = 125e3, fs: float = 1e6,
                   n_preamble: int = 8, sync_word: int = 0x12, sfo_ppm: float = 0.0, delay: float = 0.0) -> np.ndarray:
    """preamble | 2 sync symbols | 2.25 downchirps | data symbols (complex128, unit power).

    sfo_ppm: the transmitter's clock is off by delta = sfo_ppm * 1e-6 (> 0: fast against the receiver), so receiver sample n
    holds transmitter time u = n (1 + delta) samples; the frame is the base_upchirp phase law evaluated at those fractional
    times (cyclic shifts at fractional positions, the conjugate for the SFD), drifted_length() samples long.  0: exactly the
    undrifted frame.
    delay >= 0: the frame starts `delay` samples (fractional) into the output: receiver sample n holds transmitter time
    u = (n - delay) (1 + delta), 0 before the frame; its time of arrival is `delay`.  0 with sfo_ppm = 0: the undrifted frame."""
    up = base_upchirp(sf, bw, fs)
    sps = up.size
    down = np.conj(up)
    n_bins = 1 << sf
    sync = [((sync_word >> 4) & 0xF) * 8 % n_bins, (sync_word & 0xF) * 8 % n_bins]
    if not delay >= 0.0:
        raise ValueError(f"delay must be >= 0, got {delay}")
    if sfo_ppm == 0 and delay == 0:
        parts = [np.tile(up, n_preamble), modulate_shifts(sync, sf, bw, fs), down, down, down[: sps // 4],
                 modulate_shifts(fs_syms.shifts, sf, bw, fs)]
        return np.concatenate(parts)
    decim = sps // n_bins
    n_sfd = n_preamble + 2                               # first SFD symbol
    data0 = (n_sfd + 2) * sps + sps // 4
    length = data0 + len(fs_syms.shifts) * sps
    rate = 1.0 + 1e-6 * float(np.float32(sfo_ppm))
    if delay == 0:
        u = np.arange(drifted_length(length, sfo_ppm), dtype=np.float64) * rate
    else:
        u = (np.arange(int(math.ceil(delay)) + drifted_length(length, sfo_ppm), dtype=np.float64) - delay) * rate
        u = u[u < length]
    before = u < 0
    u = np.where(before, 0.0, u)
    q = np.floor(u / sps)
    m = u - q * sps                                      # position in the chirp, before any cyclic shift
    shift = np.zeros(u.size, np.int64)
    for i, b in enumerate(sync):
        shift[q == n_preamble + i] = b
    d = u - data0
    data = d >= 0
    k = np.floor(d[data] / sps).astype(np.int64)
    m[data] = d[data] - k * sps
    shift[data] = np.asarray(fs_syms.shifts, np.int64)[k] % n_bins
    m = np.mod(m + shift * decim, sps)
    t = m / fs
    phase = -2.0 * np.pi * t * (bw / 2.0 + (-0.5 * bw * (bw / n_bins)) * t)
    x = np.exp(1j * phase)
    sfd = (q >= n_sfd) & ~data
    x[sfd] = np.conj(x[sfd])
    x[before] = 0.0
    return x


def awgn(n: int, snr_db: float, rng: np.random.Generator) -> np.ndarray:
    """Complex white noise for a unit-power signal at ``snr_db`` measured in the fs bandwidth."""
    sigma = math.sqrt(10.0 ** (-snr_db / 10.0) / 2.0)
    return sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))


def channel(frames, *, sf: int, fs: float = 1e6, gap_symbols: float = 4.0, lead_symbols: float = 3.0,
            tail_symbols: float = 6.0, snr_db: float | None = 20.0, cfo_hz: float = 0.0,
            seed: int = 0x4C6F5201, amplitude: float = 1.0) -> np.ndarray:
    """Concatenate modulated frames with silence between them, apply CFO and AWGN, return cf32.

    Silence is noise only (the implicit-header end-of-packet test needs the energy to drop,
    lib/decoder_impl.cc:861).  The tail is long enough for the decoder's 2*sps look-ahead."""
    sps = int(fs / (125e3 / (1 << sf)))
    rng = np.random.default_rng(seed)
    parts = [np.zeros(int(lead_symbols * sps), dtype=np.complex128)]
    for k, f in enumerate(frames):
        parts.append(amplitude * np.asarray(f, dtype=np.complex128))
        parts.append(np.zeros(int((tail_symbols if k == len(frames) - 1 else gap_symbols) * sps), dtype=np.complex128))
    x = np.concatenate(parts)
    if cfo_hz:
        x = x * np.exp(2j * np.pi * cfo_hz * np.arange(x.size) / fs)
    if snr_db is not None:
        x = x + amplitude * awgn(x.size, snr_db, rng)
    return x.astype(np.complex64)


def synth_symbols(values, sf: int, *, snr_db: float | None = None, seed: int = 0, bw: float = 125e3,
                  fs: float = 1e6) -> np.ndarray:
    """Aligned data symbols only (K1 parity inputs): chirp shift = value, optional AWGN."""
    x = modulate_shifts(values, sf, bw, fs)
    if snr_db is not None:
        x = x + awgn(x.size, snr_db, np.random.default_rng(seed))
    return x.astype(np.complex64)
