"""Synthetic Wireless M-Bus captures (cu8) for parity tests and the benchmark.

Deterministic generator of rtl_sdr-style interleaved unsigned-8-bit IQ with planted
T1 / C1 (frame A and B) / S1 telegrams in Gaussian noise, following the transmitter
side of EN 13757-4 as the reference's own TX helpers describe it
(reference include/mode_t_util.h:38-40 3-of-6 table, include/mode_s_util.h Manchester
table, t1_c1_packet_decoder.h:39-41 C1 mode words, rtl_wmbus.c:97-103 access codes).

The generator is only trusted because the compiled reference / CPU oracle decode what it
plants (tests/test_synth.py).  Works on CPU and CUDA torch devices; the noise is drawn
slab by slab from a generator seeded with (seed, slab index) so a capture of any size is
reproducible on the device type that made it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

_ENC_3OF6 = [0x16, 0x0D, 0x0E, 0x0B, 0x1C, 0x19, 0x1A, 0x13, 0x2C, 0x25, 0x26, 0x23, 0x34, 0x31, 0x32, 0x29]

SYNC_T1C1 = "0000111101"            # last 16 chips of preamble+sync = 0x543D (rtl_wmbus.c:97)
SYNC_S1 = "000111011010010110"      # last 24 chips of preamble+sync = 0x547696 (rtl_wmbus.c:101)
C1_MODE_A = "0101010011001101"      # 0x54C + 0xD (t1_c1_packet_decoder.h:39,41)
C1_MODE_B = "0101010000111101"      # 0x543 + 0xD (t1_c1_packet_decoder.h:40,41)


def crc16(data: bytes) -> int:
    """CRC-16 poly 0x3D65, init 0, complemented (t1_c1_packet_decoder.h:463-469)."""
    crc = 0
    for b in data:
        crc ^= b << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x3D65) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return crc ^ 0xFFFF


def frame_a(payload: bytes) -> bytes:
    """payload = L-field + L bytes (no CRCs) -> wire bytes with a CRC after block 1 (10 B) and
    after every following 16-byte block (format A)."""
    assert payload[0] == len(payload) - 1 and len(payload) >= 10
    out = bytearray()
    blocks = [payload[:10]] + [payload[i:i + 16] for i in range(10, len(payload), 16)]
    for blk in blocks:
        out += blk + crc16(blk).to_bytes(2, "big")
    return bytes(out)


def frame_b(payload: bytes) -> bytes:
    """Same logical payload as frame_a() but format B: L counts the CRC bytes too; one CRC
    over the first 126 bytes (blocks 1+2), one over the rest (t1_c1_packet_decoder.h:508-536)."""
    body = bytearray(payload)
    n_crc = 1 if len(payload) + 2 <= 128 else 2
    body[0] = len(payload) - 1 + 2 * n_crc
    out = bytearray()
    if n_crc == 1:
        out += body + crc16(bytes(body)).to_bytes(2, "big")
    else:
        first, rest = bytes(body[:126]), bytes(body[126:])
        out += first + crc16(first).to_bytes(2, "big") + rest + crc16(rest).to_bytes(2, "big")
    return bytes(out)


def _bits_msb(data: bytes) -> str:
    return "".join(f"{b:08b}" for b in data)


def chips_t1(wire: bytes, preamble_pairs: int = 24, post_pairs: int = 4) -> np.ndarray:
    s = "01" * preamble_pairs + SYNC_T1C1
    for b in wire:
        s += f"{_ENC_3OF6[b >> 4]:06b}{_ENC_3OF6[b & 15]:06b}"
    s += "01" * post_pairs
    return np.frombuffer(s.encode(), np.uint8) - 48


def chips_c1(wire: bytes, frame_b_: bool = False, preamble_pairs: int = 24, post_pairs: int = 4) -> np.ndarray:
    s = "01" * preamble_pairs + SYNC_T1C1 + (C1_MODE_B if frame_b_ else C1_MODE_A) + _bits_msb(wire)
    s += "01" * post_pairs
    return np.frombuffer(s.encode(), np.uint8) - 48


def chips_s1(wire: bytes, preamble_pairs: int = 40, post_pairs: int = 4) -> np.ndarray:
    s = "01" * preamble_pairs + SYNC_S1
    s += "".join("01" if c == "1" else "10" for c in _bits_msb(wire))   # s1_packet_decoder.h:35-37
    s += "01" * post_pairs
    return np.frombuffer(s.encode(), np.uint8) - 48


def fsk_burst(chips: np.ndarray, chip_rate: float, fs: float, dev_hz: float, offset_hz: float,
              amp: float, chip_dev: np.ndarray | None = None) -> np.ndarray:
    """Phase-continuous 2-FSK, chip 1 = +deviation (chip_dev: a factor on chip i's deviation).  Returns float32 array
    [n, 2] (I, Q)."""
    n = int(math.ceil(len(chips) * fs / chip_rate))
    idx = np.minimum((np.arange(n, dtype=np.float64) * (chip_rate / fs)).astype(np.int64), len(chips) - 1)
    f = offset_hz + dev_hz * (2.0 * chips[idx].astype(np.float64) - 1.0)
    if chip_dev is not None:
        f = offset_hz + (f - offset_hz) * np.asarray(chip_dev, np.float64)[idx]
    phase = 2.0 * math.pi * np.cumsum(f) / fs
    return np.stack([amp * np.cos(phase), amp * np.sin(phase)], axis=1).astype(np.float32)


@dataclass
class Emitter:
    mode: str                    # "T1", "C1A", "C1B", "S1"
    ident: int                   # 8 BCD digits as printed in LINK_LAYER_IDENT_NO
    amp: float = 90.0
    offset_hz: float = 0.0
    dev_hz: float = 50e3
    l_field: int = 0x19          # logical L (format A meaning)
    period_s: float = 0.5
    start_s: float = 0.01
    manufacturer: int = 0x5068
    seed: int = 1
    sync_flips: tuple = ()       # chips of the access code sent inverted in every telegram, counted back from its last chip
    data_flips: tuple = ()       # chips after the access code sent inverted in every telegram (0: the L-field's first chip)
    weak_flips: tuple = ()       # chips after the access code sent on the wrong tone at weak_dev of the deviation (0: as data_flips)
    weak_dev: float = 0.2        # the low-reliability error noise makes; data_flips is the full-swing one
    chip_rate: float = field(init=False)

    def __post_init__(self):
        self.chip_rate = 32768.0 if self.mode == "S1" else 100e3

    def payload(self, k: int) -> bytes:
        """Logical telegram k (L, C, M, A(6), data...) without CRC bytes."""
        rng = np.random.default_rng([self.seed, self.ident & 0xFFFF, k])
        L = self.l_field
        p = bytearray(1 + L)
        p[0] = L
        p[1] = 0x44
        p[2:4] = self.manufacturer.to_bytes(2, "little")
        p[4:8] = self.ident.to_bytes(4, "little")
        p[8] = 0x71
        p[9] = 0x07
        if L > 9:
            data = rng.integers(0, 256, L - 9, dtype=np.uint8).tobytes()
            p[10:] = data
            if L >= 13:
                p[10:14] = (k & 0xFFFFFFFF).to_bytes(4, "little")      # telegram counter
        return bytes(p)

    def chips(self, k: int) -> np.ndarray:
        c = self._chips(k)
        end = 2 * 40 + len(SYNC_S1) if self.mode == "S1" else 2 * 24 + len(SYNC_T1C1)
        if self.sync_flips:      # a receiver accepts these only with access-code errors allowed (wmb_set_receiver)
            c = c.copy()
            c[end - 1 - np.asarray(self.sync_flips)] ^= 1
        if self.data_flips:      # T1 symbols / S1 chip pairs that lose a chip: erasures for wmb_frame_repair
            c = c.copy()
            c[end + np.asarray(self.data_flips)] ^= 1
        return c

    def chip_dev(self):
        """per chip, the fraction of dev_hz it is sent at (None: all at full deviation): -weak_dev at weak_flips"""
        if not self.weak_flips:
            return None
        end = 2 * 40 + len(SYNC_S1) if self.mode == "S1" else 2 * 24 + len(SYNC_T1C1)
        dev = np.ones(len(self._chips(0)))
        dev[end + np.asarray(self.weak_flips)] = -self.weak_dev
        return dev

    def _chips(self, k: int) -> np.ndarray:
        p = self.payload(k)
        if self.mode == "T1":
            return chips_t1(frame_a(p))
        if self.mode == "C1A":
            return chips_c1(frame_a(p), False)
        if self.mode == "C1B":
            return chips_c1(frame_b(p), True)
        if self.mode == "S1":
            return chips_s1(frame_a(p))
        raise ValueError(self.mode)

    def expected_fields(self, k: int):
        """(MODE, IDENT string, datagram hex) the reference prints for telegram k when decoded
        without errors.  C1-B prints with L rewritten to the format-A value."""
        p = self.payload(k)
        return (self.mode[:2], f"{self.ident:08X}", "0x" + p.hex())


@dataclass
class Planted:
    emitter: int
    k: int
    start_iq: int
    n_iq: int


def default_emitters(config: str = "t1x2"):
    """Emitter sets for the BASELINE.json configs."""
    if config == "t1x2":       # config 2: two T1 emitters, strong + weak (SURVEY 8d)
        return [Emitter("T1", 0x71200023, amp=95.0, offset_hz=8e3, l_field=0x29, period_s=0.50, start_s=0.020, seed=11),
                Emitter("T1", 0x64700082, amp=40.0, offset_hz=-12e3, l_field=0x66, period_s=0.73, start_s=0.170, seed=12)]
    if config == "s1":         # config 3
        return [Emitter("S1", 0x20338739, amp=70.0, offset_hz=3e3, l_field=0x19, period_s=0.41, start_s=0.015, seed=13),
                Emitter("S1", 0x02717473, amp=45.0, offset_hz=-6e3, l_field=0x2E, period_s=0.67, start_s=0.120, seed=14)]
    if config == "mixed":      # every telegram type; used by the parity tests
        return [Emitter("T1", 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x29, period_s=0.11, start_s=0.004, seed=21),
                Emitter("C1A", 0x20338739, amp=60.0, offset_hz=-5e3, l_field=0x19, period_s=0.13, start_s=0.030, seed=22),
                Emitter("C1B", 0x20210116, amp=60.0, offset_hz=4e3, l_field=0x19, period_s=0.17, start_s=0.055, seed=23),
                Emitter("S1", 0x19131290, amp=70.0, offset_hz=2e3, l_field=0x19, period_s=0.19, start_s=0.080, seed=24)]
    raise ValueError(config)


def plan_bursts(emitters, n_iq: int, fs: float):
    plan = []
    for ei, e in enumerate(emitters):
        k = 0
        while True:
            start = int(round((e.start_s + k * e.period_s) * fs))
            n = int(math.ceil(len(e.chips(0)) * fs / e.chip_rate))
            if start + n + 64 > n_iq:
                break
            plan.append(Planted(ei, k, start, n))
            k += 1
    plan.sort(key=lambda p: p.start_iq)
    return plan


def synth_capture(n_bytes: int, fs: float = 1.6e6, emitters=None, seed: int = 0xB2000000,
                  noise_sigma: float = 8.0, mean: float = 127.4, device="cpu",
                  center_shift_hz: float = 0.0, slab_iq: int = 1 << 24, out: torch.Tensor | None = None):
    """Returns (uint8 tensor [n_bytes] on `device`, list[Planted]).

    center_shift_hz shifts T1/C1 emitters by +shift and S1 emitters by -shift (the `-s`
    scenario: capture centred on 868.625 MHz, shift 325 kHz)."""
    assert n_bytes % 4096 == 0
    emitters = default_emitters() if emitters is None else emitters
    n_iq = n_bytes // 2
    dev = torch.device(device)
    buf = out if out is not None else torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    plan = plan_bursts(emitters, n_iq, fs)
    burst_cache = {}
    for s_idx, s0 in enumerate(range(0, n_iq, slab_iq)):
        s1 = min(n_iq, s0 + slab_iq)
        g = torch.Generator(device=dev)
        g.manual_seed((seed + 7919 * s_idx) & 0x7FFFFFFFFFFFFFFF)
        x = torch.randn((s1 - s0, 2), generator=g, device=dev, dtype=torch.float32)
        x.mul_(noise_sigma).add_(mean)
        for p in plan:
            if p.start_iq >= s1 or p.start_iq + p.n_iq <= s0:
                continue
            key = (p.emitter, p.k)
            if key not in burst_cache:
                e = emitters[p.emitter]
                shift = center_shift_hz if e.mode != "S1" else -center_shift_hz
                b = fsk_burst(e.chips(p.k), e.chip_rate, fs, e.dev_hz, e.offset_hz + shift, e.amp, e.chip_dev())
                burst_cache[key] = torch.from_numpy(b).to(dev)
            b = burst_cache[key]
            a0, a1 = max(s0, p.start_iq), min(s1, p.start_iq + b.shape[0])
            x[a0 - s0:a1 - s0] += b[a0 - p.start_iq:a1 - p.start_iq]
            if p.start_iq + b.shape[0] <= s1:
                burst_cache.pop(key, None)
        buf[2 * s0:2 * s1] = x.round_().clamp_(0, 255).to(torch.uint8).reshape(-1)
        del x
    return buf, plan
