// lora_crc.h -- the LoRa payload CRC as published by the decode chain, shared by the host (lora_b200_frames_crc_last, the
// CPU emulation) and the device (rs_crc_list_kernel, rx_sync.cuh).
//
// Semtech's payload CRC of a payload of L >= 2 bytes: CRC-16, polynomial 0x1021, initial value 0, no reflection, no final
// XOR, over payload[0 .. L-2), XORed with payload[L-1] | payload[L-2] << 8.  The radio appends it low byte first and does not
// whiten it, but the decode chain (K8, bit-exact to the reference) dewhitens every payload nibble, the CRC's too: the two
// published bytes are crc ^ W(L), W(L) being what the chain makes of all-zero code words at nibbles 2L .. 2L+3 (the data
// projection of the whitening bytes there: Hamming decode for CR 3-4, the data bits for CR 1-2).  Both the CRC and W are
// fixed linear maps, so a published frame checks iff
//     crc16(payload[0 .. L-2)) ^ (payload[L-1] | payload[L-2] << 8) ^ (c0 | c1 << 8) ^ W(L) == 0.
// The reference's own known answer: de ad be ef (L = 4) -> CRC 0xEC80, published 70 0d.
#pragma once
#include "int_chain.cuh"

#define LORA_CRC_NONE 0u       // no CRC in the header (or the implicit configuration), or L < 2
#define LORA_CRC_OK 1u
#define LORA_CRC_BAD 2u
#define LORA_CRC_RECOVERED 3u  // OK after CRC-aided list decoding (rs_crc_list_kernel)

namespace lb {

LB_HD uint32_t lb_crc16_byte(uint32_t crc, uint32_t byte) {
    crc ^= (byte & 0xFFu) << 8;
    for (int k = 0; k < 8; k++) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x1021u) & 0xFFFFu : (crc << 1) & 0xFFFFu;
    return crc;
}

// CRC-16 (0x1021, init 0) over b[0 .. n)
LB_HD uint32_t lb_crc16(const uint8_t *b, uint32_t n) {
    uint32_t crc = 0;
    for (uint32_t i = 0; i < n; i++) crc = lb_crc16_byte(crc, b[i]);
    return crc;
}

// the payload CRC of payload[0 .. L), L >= 2
LB_HD uint32_t lb_payload_crc(const uint8_t *payload, uint32_t L) {
    return lb_crc16(payload, L - 2u) ^ (payload[L - 1u] | ((uint32_t)payload[L - 2u] << 8));
}

// the decode chain's nibble of an all-zero code word at payload nibble p of a frame with coding rate cr (decode_byte)
LB_HD uint32_t lb_crc_white_nibble(uint32_t cr, uint32_t p) {
    const uint8_t w = whitening_byte(0, cr, p);
    return cr >= 3u ? hamming84_decode(w) : extract_data(w);
}

// W(L): the fixed XOR the chain puts on the CRC bytes of an L-byte payload, published bytes c0 | c1 << 8
LB_HD uint32_t lb_crc_whitening(uint32_t cr, uint32_t L) {
    uint32_t w = 0;
    for (uint32_t k = 0; k < 4u; k++) w |= lb_crc_white_nibble(cr, 2u * L + k) << (4u * k);
    return w;
}

// the syndrome of published bytes b[0 .. L + 2): 0 iff the frame checks
LB_HD uint32_t lb_crc_syndrome(const uint8_t *b, uint32_t L, uint32_t cr) {
    return lb_payload_crc(b, L) ^ b[L] ^ ((uint32_t)b[L + 1u] << 8) ^ lb_crc_whitening(cr, L);
}

// status of the published payload b[0 .. n) (CRC bytes included when crc != 0) of a frame with coding rate cr
LB_HD uint32_t lb_crc_check(const uint8_t *b, uint32_t n, uint32_t cr, uint32_t crc) {
    if (!crc || n < 4u) return LORA_CRC_NONE;
    return lb_crc_syndrome(b, n - 2u, cr) == 0u ? LORA_CRC_OK : LORA_CRC_BAD;
}

// ... of a published record loratap (15 B) | phy header (3 B) | payload, len bytes in all: the header's has_mac_crc and cr,
// the payload length from len, as message_socket_sink strips it
LB_HD uint32_t lb_crc_record_status(const uint8_t *rec, uint32_t len) {
    if (len < 18u) return LORA_CRC_NONE;
    return lb_crc_check(rec + 18, len - 18u, (uint32_t)rec[16] >> 5, ((uint32_t)rec[16] >> 4) & 1u);
}

}  // namespace lb
