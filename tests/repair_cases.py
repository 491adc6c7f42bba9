"""Erasure repair of one framing candidate (include/wmbus_b200_framer.h, wmb_frame_repair), restated in plain Python.

The decoder's verdict on a candidate -- a line and its CRC_OK column, or where it stopped -- comes from the oracle's
per-bit state machines (tests/orc.py, restating t1_c1_packet_decoder.h / s1_packet_decoder.h).  The repair is the
definition applied to the bit list; nothing here calls the product's framers."""
import ctypes as C
import itertools

import numpy as np

NONE, REPAIRED, AMBIGUOUS, TOO_MANY, UNREPAIRABLE, TRUNCATED = range(6)
OUTCOMES = ["none", "repaired", "ambiguous", "too_many", "unrepairable", "truncated"]

# EN 13757-4 3-out-of-6: nibble -> code word
ENC_3OF6 = [0x16, 0x0D, 0x0E, 0x0B, 0x1C, 0x19, 0x1A, 0x13, 0x2C, 0x25, 0x26, 0x23, 0x34, 0x31, 0x32, 0x29]
DEC_3OF6 = {w: v for v, w in enumerate(ENC_3OF6)}
CAPTURE_THRESHOLD = 5


def _crc_table():
    tab = []
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x3D65) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        tab.append(c)
    return tab


CRC_TAB = _crc_table()


def crc16(data) -> int:
    """CRC-16, polynomial 0x3D65, complemented."""
    crc = 0
    for b in data:
        crc = CRC_TAB[(b ^ (crc >> 8)) & 0xFF] ^ ((crc << 8) & 0xFFFF)
    return crc ^ 0xFFFF


def block_ok(q) -> bool:
    return len(q) >= 2 and crc16(q[:-2]) == (q[-2] << 8 | q[-1])


def tlg_len_a(L: int) -> int:
    """bytes on air of a frame-A telegram with L-field L (CRCs included)"""
    return 1 + L + 2 * (1 + ((L - 9 + 15) // 16 if L > 9 else 0))


def blocks_a(n: int):
    """(offset, length) of the CRC blocks of frame format A: 12 bytes, then 18 (the last one shorter)"""
    out, off = [(0, 12)], 12
    while off < n:
        out.append((off, min(18, n - off)))
        off += 18
    return out


def fillings_3of6(w: int):
    """nibbles of the code words at Hamming distance 1 from the 6-bit word w, lowest flipped bit first"""
    return [DEC_3OF6[w ^ (1 << k)] for k in range(6) if (w ^ (1 << k)) in DEC_3OF6]


def oracle_verdict(orc_mod, chain, bits, rssi):
    """(chips consumed, line or None) of the oracle's per-bit decoder on one candidate"""
    L = orc_mod.lib()
    out = C.create_string_buffer(4096)
    got = C.c_int(0)
    fn = L.orc_frame_t1c1 if chain == 0 else L.orc_frame_s1
    consumed = fn(np.ascontiguousarray(bits, np.uint8), np.ascontiguousarray(rssi, np.uint8), len(bits), b"",
                  out, 4096, C.byref(got))
    return consumed, (out.value.decode().rstrip("\n") if got.value else None)


def repair(orc_mod, chain, bits, rssi, offsets, sync_sample, e_max):
    """The repair of one candidate: dict(outcome, erasures, blocks, had_line) plus, when repaired, the line's fields
    (mode, crc_ok, ok_3of6, packet_rssi, current_rssi, serial, datagram, consumed, end_sample)."""
    bits = [int(x) & 1 for x in bits]
    n = len(bits)
    r = dict(outcome=NONE, erasures=0, blocks=0, had_line=0)
    if e_max == 0 or n == 0:
        return r
    consumed, line = oracle_verdict(orc_mod, chain, bits, rssi)
    if line is not None:
        mode, crc_ok = line.split(";")[:2]
        if crc_ok != "0":
            return r
        r["had_line"] = 1
        if mode == "C1":
            r["outcome"] = UNREPAIRABLE
            return r
    else:
        pos = consumed - 1
        if chain == 0 or pos < 18 or pos % 2 or bits[pos] != bits[pos - 1]:
            return r                       # not an abort on a Manchester violation after the L-field byte

    def word(first, k):
        v = 0
        for x in bits[first:first + k]:
            v = v << 1 | x
        return v

    t1 = chain == 0
    L = (DEC_3OF6[word(1, 6)] << 4 | DEC_3OF6[word(7, 6)]) if t1 else word2(bits, 2, 8)
    length = tlg_len_a(L)
    P = 1 + (12 if t1 else 16) * length
    if n < P:
        r["outcome"] = TRUNCATED
        return r
    if length < 12 or any(int(x) < CAPTURE_THRESHOLD for x in rssi[:P - 1]):
        r["outcome"] = UNREPAIRABLE
        return r

    pkt = [0] * length
    pkt[0] = L
    erasures = []                          # (byte, shift, fillings) in chip order
    for l in range(1, length):
        v = 0
        if t1:
            for s, shift in ((0, 4), (1, 0)):
                w = word(1 + 12 * l + 6 * s, 6)
                if w in DEC_3OF6:
                    v |= DEC_3OF6[w] << shift
                else:
                    f = fillings_3of6(w)
                    if not f:
                        r["outcome"] = UNREPAIRABLE
                        return r
                    erasures.append((l, shift, f))
        else:
            for k in range(8):
                a, c = bits[1 + 16 * l + 2 * k], bits[2 + 16 * l + 2 * k]
                if a != c:
                    v |= c << (7 - k)
                else:
                    erasures.append((l, 7 - k, [0, 1]))
        pkt[l] = v
    blocks = blocks_a(length)
    per_block = [[e for e in erasures if off <= e[0] < off + blk] for off, blk in blocks]
    if any(len(es) > e_max for es in per_block):
        r["outcome"] = TOO_MANY
        return r
    n_erasures = n_blocks = 0
    for (off, blk), es in zip(blocks, per_block):
        passing = []
        for fill in itertools.product(*[e[2] for e in es]):
            q = pkt[off:off + blk]
            for (byte, shift, _), v in zip(es, fill):
                q[byte - off] |= v << shift
            if block_ok(q):
                passing.append(fill)
        if len(passing) != 1:
            r["outcome"] = AMBIGUOUS if passing else UNREPAIRABLE
            return r
        for (byte, shift, _), v in zip(es, passing[0]):
            pkt[byte] |= v << shift
        n_erasures += len(es)
        n_blocks += 1 if es else 0
    if n_erasures == 0:
        r["outcome"] = UNREPAIRABLE
        return r
    datagram = pkt[:10] + [x for off, blk in blocks[1:] for x in pkt[off:off + blk - 2]]
    r.update(outcome=REPAIRED, erasures=n_erasures, blocks=n_blocks, mode="T1" if t1 else "S1", crc_ok=1, ok_3of6=1, packet_rssi=int(rssi[1]),
             current_rssi=int(rssi[P - 1]), serial=int.from_bytes(bytes(pkt[4:8]), "little"), datagram=bytes(datagram),
             consumed=P, end_sample=sync_sample + int(offsets[P - 1]))
    return r


def word2(bits, first, k):
    """k Manchester data bits: the second chip of each pair from index `first` on"""
    v = 0
    for i in range(k):
        v = v << 1 | bits[first + 2 * i]
    return v
