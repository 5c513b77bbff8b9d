"""Host-side view of a published frame (SURVEY.md §8f N4).

The reference publishes ``loratap (15 B, zero except rssi.snr) | loraphy header (3 B) | payload`` and never verifies
the explicit header's 5-bit checksum (``include/lora/utilities.h:396-404``: the check is commented out) nor the payload CRC
(``README.md:12``).  This module adds both checks WITHOUT touching what is published: `parse_frame` and `crc_status` only
read the blob.  The payload CRC (tx.payload_crc) is Semtech's CRC-16; the radio does not whiten it but the
decode chain dewhitens it like every payload nibble, so a published frame carries crc ^ W(L) (tx.crc_whitening) -- the
reference's own golden frame ``de ad be ef`` -> ``70 0d`` (README.md:67-71): CRC 0xEC80, W(4) = 0xE1F0.
"""
from __future__ import annotations

from dataclasses import dataclass

from .tx import crc_whitening, header_checksum, payload_crc

CRC_NONE, CRC_OK, CRC_BAD = 0, 1, 2        # lora_b200_frames_crc_last (CRC_RECOVERED = 3 comes from the list decoder only)

LORATAP_LEN = 15       # include/lora/loratap.h:48-55 (packed), all zero except rssi.snr (lib/decoder_impl.cc:597)
PHY_LEN = 3            # include/lora/loraphy.h:25-32


@dataclass(frozen=True)
class Frame:
    snr: int                 # loratap rssi.snr byte
    length: int              # PHY header: payload length without the MAC CRC
    cr: int                  # coding rate 1..4 (the reference clamps > 4 to 4, lib/decoder_impl.cc:837-839)
    has_mac_crc: bool
    checksum: int            # the 5 received checksum bits
    header_ok: bool          # checksum == header_checksum(length, cr, has_mac_crc)
    payload: bytes           # everything after the PHY header (payload + 2 CRC bytes when has_mac_crc)


def parse_frame(blob: bytes) -> Frame:
    """Split a frame blob as published on port ``frames`` (lib/decoder_impl.cc:588-609)."""
    if len(blob) < LORATAP_LEN + PHY_LEN:
        raise ValueError(f"frame of {len(blob)} bytes is shorter than loratap + phy header")
    snr = blob[13]                                   # loratap_header_t.rssi.snr (byte 13; byte 14 is sync_word)
    b0, b1, b2 = blob[LORATAP_LEN:LORATAP_LEN + PHY_LEN]
    # LSB-first bit fields of loraphy_header_t: length:8 | crc_msn:4 has_mac_crc:1 cr:3 | reserved:4 crc_lsn:4
    length, crc_msn, has_crc, cr = b0, b1 & 0x0F, (b1 >> 4) & 1, (b1 >> 5) & 7
    crc_lsn = (b2 >> 4) & 0x0F
    chk = ((crc_msn & 1) << 4) | crc_lsn
    return Frame(snr=snr, length=length, cr=cr, has_mac_crc=bool(has_crc), checksum=chk,
                 header_ok=chk == header_checksum(length, cr, has_crc), payload=bytes(blob[LORATAP_LEN + PHY_LEN:]))


def crc_status(blob: bytes) -> int:
    """The payload CRC status of a published frame blob: CRC_NONE when its PHY header has no CRC flag (has_mac_crc, the
    configured flag for implicit headers) or its payload has fewer than 2 bytes, else CRC_OK or CRC_BAD.  The payload is what
    follows the PHY header without the last two bytes, as message_socket_sink strips it (LORAMAC)."""
    f = parse_frame(blob)
    if not f.has_mac_crc or len(f.payload) < 4:
        return CRC_NONE
    pay, c = f.payload[:-2], f.payload[-2] | f.payload[-1] << 8
    return CRC_OK if c ^ crc_whitening(len(pay), f.cr) == payload_crc(pay) else CRC_BAD
