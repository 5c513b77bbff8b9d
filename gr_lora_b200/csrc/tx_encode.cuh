// tx_encode.cuh -- the LoRa frame encoder on the device: payload bytes -> chirp shifts of the data symbols (SURVEY 8(f) N3).
//
// The exact inverse of the integer decode chain of int_chain.cuh, and bit-identical to the host encoder
// gr_lora_b200/tx.py::encode_frame:
//   payload nibbles (low first; explicit header: 5 nibbles, high first, with its 5-bit checksum)
//   -> Hamming(8,4) -> XOR whitening -> bit shuffle -> mask to 8 bits (header block) or 4 + cr bits (payload blocks)
//   -> diagonal interleave of one block of ppm code words into 8 (header) or 4 + cr (payload) words
//   -> inverse Gray -> x4 for reduced-rate symbols -> +1 bin, since the gradient demodulator reports (bin - 1) mod N.
// Symbol i of a block depends on that block's ppm code words only, and each code word on one nibble, so every
// (frame, symbol) is computed independently: one thread per data symbol, no serial pass over a frame.
#pragma once
#include "int_chain.cuh"

namespace lb {

// what the encoder needs of a decoder configuration
struct TxCode {
    uint32_t sf, cr;          // SF7..12, CR 1..4 (4/5 .. 4/8)
    uint32_t explicit_hdr, crc, reduced_rate;
};

// 5-bit explicit-header checksum over (length, cr, crc): the reference never verifies it (include/lora/utilities.h:396-404),
// its README golden 04 90 40 carries it (README.md:67-71)
LB_HD uint32_t header_checksum(uint32_t length, uint32_t cr, uint32_t crc) {
    const uint32_t h0 = (length >> 4) & 15u, h1 = length & 15u, h2 = ((cr & 7u) << 1) | (crc & 1u);
    auto b = [](uint32_t v, int i) { return (v >> i) & 1u; };
    const uint32_t c4 = b(h0, 3) ^ b(h0, 2) ^ b(h0, 1) ^ b(h0, 0);
    const uint32_t c3 = b(h0, 3) ^ b(h1, 3) ^ b(h1, 2) ^ b(h1, 1) ^ b(h2, 0);
    const uint32_t c2 = b(h0, 2) ^ b(h1, 3) ^ b(h1, 0) ^ b(h2, 3) ^ b(h2, 1);
    const uint32_t c1 = b(h0, 1) ^ b(h1, 2) ^ b(h1, 0) ^ b(h2, 2) ^ b(h2, 1) ^ b(h2, 0);
    const uint32_t c0 = b(h0, 0) ^ b(h1, 1) ^ b(h2, 3) ^ b(h2, 2) ^ b(h2, 1) ^ b(h2, 0);
    return (c4 << 4) | (c3 << 3) | (c2 << 2) | (c1 << 1) | c0;
}

LB_HD uint8_t shuffle_byte(uint8_t v) {        // inverse of deshuffle_byte: bit j goes to pattern[j], {5,0,1,2,4,3,6,7}
    return (uint8_t)(((v & 1u) << 5) | ((v >> 1) & 1u) | (((v >> 2) & 1u) << 1) | (((v >> 3) & 1u) << 2) |
                     (((v >> 4) & 1u) << 4) | (((v >> 5) & 1u) << 3) | (v & 0xC0u));
}

LB_HD uint32_t rotr_bits(uint32_t bits, uint32_t count, uint32_t size) {
    const uint32_t mask = (1u << size) - 1u;
    count %= size;
    bits &= mask;
    return count ? ((bits >> count) | ((bits << (size - count)) & mask)) : bits;
}

LB_HD uint32_t gray_decode(uint32_t w) {       // inverse of gray_encode
    uint32_t b = 0;
    for (; w; w >>= 1) b ^= w;
    return b;
}

// a payload length the encoder accepts: at most 255 bytes plus the two CRC bytes, and an explicit header with CRC needs them
LB_HD bool tx_length_ok(const TxCode &c, uint32_t len) {
    return len <= 255u + 2u * c.crc && !(c.explicit_hdr && c.crc && len < 2u);
}

LB_HD uint32_t tx_spare(const TxCode &c) { return c.sf - 2u - (c.explicit_hdr ? 5u : 0u); }   // payload code words in the header block
LB_HD uint32_t tx_ppm(const TxCode &c) { return c.reduced_rate ? c.sf - 2u : c.sf; }

// payload blocks: enough for the code words, and at least what the receiver reads after an explicit header (:842-847)
LB_HD uint32_t tx_payload_blocks(const TxCode &c, uint32_t len) {
    const uint32_t spare = tx_spare(c), ppm = tx_ppm(c), need = 2u * len;
    uint32_t blocks = need > spare ? (need - spare + ppm - 1u) / ppm : 0u;
    if (c.explicit_hdr) {
        const uint32_t rx = (uint32_t)payload_symbols(len, c.cr, c.sf, (int)c.reduced_rate) / (c.cr + 4u);
        if (rx > blocks) blocks = rx;
    }
    return blocks;
}

// data symbols of one frame: the 8-symbol header block and the payload blocks
LB_HD uint32_t tx_data_symbols(const TxCode &c, uint32_t len) { return 8u + tx_payload_blocks(c, len) * (c.cr + 4u); }

// the nibble the payload puts in payload code word p (p counts from the first payload nibble; past the payload: nibble 0)
LB_HD uint32_t tx_payload_nibble(const uint8_t *payload, uint32_t len, uint32_t p) {
    return p < 2u * len ? (payload[p >> 1] >> ((p & 1u) * 4u)) & 15u : 0u;
}

// the whitened, shuffled code word of nibble s at payload slot p, masked to nbits bits
LB_HD uint32_t tx_payload_cw(const TxCode &c, uint32_t s, uint32_t p, uint32_t nbits) {
    const uint8_t w = (uint8_t)(hamming84_encode((uint8_t)s) ^ whitening_byte(0, c.cr, p));
    return shuffle_byte(w) & ((1u << nbits) - 1u);
}

// payload code word p of the frame carrying payload[0 .. len)
LB_HD uint32_t tx_payload_codeword(const TxCode &c, const uint8_t *payload, uint32_t len, uint32_t p, uint32_t nbits) {
    return tx_payload_cw(c, tx_payload_nibble(payload, len, p), p, nbits);
}

// the nibble of header-block slot x (x < sf - 2): the 5 header nibbles of an explicit header, then payload nibbles
LB_HD uint32_t tx_header_nibble(const TxCode &c, const uint8_t *payload, uint32_t len, uint32_t x) {
    if (c.explicit_hdr && x < 5u) {
        const uint32_t length = (len - 2u * c.crc) & 0xFFu, chk = header_checksum(length, c.cr, c.crc);
        const uint32_t h1 = ((c.cr & 7u) << 5) | ((c.crc & 1u) << 4) | (chk >> 4), h2 = (chk & 15u) << 4;
        const uint32_t nib[5] = {length >> 4, length & 15u, h1 >> 4, h1 & 15u, h2 >> 4};
        return nib[x];
    }
    return tx_payload_nibble(payload, len, x - (c.explicit_hdr ? 5u : 0u));
}

// the code word of nibble s at header-block slot x (8 bits; payload slots are whitened with c.cr's table)
LB_HD uint32_t tx_header_cw(const TxCode &c, uint32_t s, uint32_t x) {
    if (c.explicit_hdr && x < 5u) return shuffle_byte((uint8_t)(hamming84_encode((uint8_t)s) ^ whitening_byte(1, c.cr, x)));
    return tx_payload_cw(c, s, x - (c.explicit_hdr ? 5u : 0u), 8u);
}

// code word x of the header block of the frame carrying payload[0 .. len)
LB_HD uint32_t tx_header_codeword(const TxCode &c, const uint8_t *payload, uint32_t len, uint32_t x) {
    return tx_header_cw(c, tx_header_nibble(c, payload, len, x), x);
}

// chirp shift of symbol i of an interleaver block whose ppm code words are cw(0 .. ppm): the word whose bit x is bit i of
// code word x, rotated right by i, inverse Gray, x4 for reduced-rate symbols, +1 bin
template <class CW>
LB_HD uint32_t tx_block_shift(const CW &cw, uint32_t i, uint32_t ppm, bool reduced, uint32_t n_bins) {
    uint32_t v = 0;
    for (uint32_t x = 0; x < ppm; x++) v |= ((cw(x) >> i) & 1u) << x;
    uint32_t g = gray_decode(rotr_bits(v, i, ppm));
    if (reduced) g = (4u * g) % n_bins;
    return (g + 1u) % n_bins;
}

// chirp shift of data symbol i (< tx_data_symbols) of the frame carrying payload[0 .. len)
LB_HD uint32_t tx_symbol_shift(const TxCode &c, const uint8_t *payload, uint32_t len, uint32_t i) {
    const uint32_t n_bins = 1u << c.sf;
    if (i < 8u)                                            // header block: ppm = sf - 2, 8 words, always reduced rate
        return tx_block_shift([&](uint32_t x) { return tx_header_codeword(c, payload, len, x); }, i, c.sf - 2u, true, n_bins);
    const uint32_t spb = c.cr + 4u, ppm = tx_ppm(c), b = (i - 8u) / spb, j = (i - 8u) - b * spb;
    const uint32_t p0 = tx_spare(c) + b * ppm;
    return tx_block_shift([&](uint32_t x) { return tx_payload_codeword(c, payload, len, p0 + x, spb); }, j, ppm, c.reduced_rate != 0u,
                          n_bins);
}

#ifdef __CUDACC__
// one thread = one (frame, data symbol); frame f = payloads[frames[f].x .. + frames[f].y); shifts[f * max_symbols + i]
__global__ void tx_encode_kernel(TxCode code, const uint8_t *__restrict__ payloads, const uint2 *__restrict__ frames, size_t n_frames,
                                 uint32_t max_symbols, uint32_t *__restrict__ shifts) {
    const size_t total = n_frames * max_symbols;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const size_t f = g / max_symbols;
        const uint32_t i = (uint32_t)(g - f * max_symbols);
        const uint2 fr = frames[f];
        if (i >= tx_data_symbols(code, fr.y)) continue;
        shifts[g] = tx_symbol_shift(code, payloads + fr.x, fr.y, i);
    }
}
#endif

}  // namespace lb
