"""The reference's receiver with other receiver constants -- TEST INFRASTRUCTURE ONLY.

Built on the CPU oracle (oracle/wmbus_oracle.c through tests/orc.py), which states the reference with its constants:
clock-lock threshold 2 (opts_CLOCK_LOCK_THRESHOLD_*, rtl_wmbus.c:865-866) and no access-code errors
(ACCESS_CODE_*_ERRORS, :99, :103).  Neither constant changes anything in front of the bit sync, so the oracle's stages
(slicer bits, clock signs, rssi) and its run-length events (bits, resets) hold for any setting.  What depends on them is
restated here:
  * time2 strobes: sample m iff the clock read low at m-L-1 and high at m-L..m (the lock counter of :1092-1111; the
    clock reads low before the first sample);
  * the access-code flag: count_set_bits((bitstream & MASK) ^ CODE) <= E (:688, :773, :822, :846) over the bits since
    the last run-length reset (the reset clears the register, :717-726; time2 never resets);
  * the decoder calls: per stream a candidate starts the oracle's framer (orc_frame_t1c1 / orc_frame_s1) only when the
    decoder is idle (t1_c1_packet_decoder.h:272-278), a run-length reset ends a telegram in flight, and lines come out in
    the reference's order (sample of the last bit, then T1/C1 rla, T1/C1 t2a, S1 rla, S1 t2a; :1354-1355).
With the default settings this reproduces orc.run_lines exactly; with others it is pinned against reference builds with
the constants changed (tests/golden/reference_runs_receiver.json)."""
import ctypes as C

import numpy as np

import orc

CODES = {0: (0x543D, 0xFFFF, 16), 1: (0x547696, 0xFFFFFF, 24)}     # access code, mask, register bits per chain


def strobes(clk, lock):
    """time2 strobes of clock signs `clk` (0/1 per sample) at clock-lock threshold `lock`"""
    c = np.asarray(clk).astype(bool)
    idx = np.arange(len(c), dtype=np.int64)
    last_low = np.maximum.accumulate(np.where(c, -1, idx))         # -1: low before the first sample
    return ((idx - last_low) == lock + 1).astype(np.uint8)         # exactly L+1 high samples up to m


def access_code_flags(bits, resets, chain, errors):
    """the flag of every bit of one stream: the register holds the bits since the last reset"""
    code, mask, nb = CODES[chain]
    bits = np.asarray(bits).astype(np.uint64)
    n = len(bits)
    idx = np.arange(n, dtype=np.int64)
    start = np.maximum.accumulate(np.where(np.asarray(resets) != 0, idx, 0))
    sr = np.zeros(n, np.uint64)
    for k in range(nb):
        j = idx - k
        sr |= np.where(j >= start, bits[np.maximum(j, 0)], np.uint64(0)) << np.uint64(k)
    return (np.bitwise_count((sr & np.uint64(mask)) ^ np.uint64(code)) <= errors).astype(np.uint8)


def runlength_events(st, chain):
    """orc.events(st, chain, 0) without its cap of M/2 events (a run-length tracker whose bit length has collapsed
    under an in-channel tone emits more): the oracle reports how many there are, and a second call takes them all"""
    L = orc.lib()
    cap = st["M"] // 2 + 64
    while True:
        ev = np.zeros(cap, orc.EVENT_DTYPE)
        n = L.orc_runlength_events(st["bit"], st["rssi"], st["M"], chain, ev.ctypes.data, cap)
        if n <= cap:
            return ev[:n]
        cap = n


def stream_events(st, chain, algo, lock, errors):
    """the decoder calls of one (chain, algorithm) stream: dict of arrays m, bit, sync, reset, rssi"""
    if algo == 1:
        m = np.nonzero(strobes(st["clk"], lock))[0].astype(np.uint64)
        ev = dict(m=m, bit=st["bit"][m].astype(np.uint8), reset=np.zeros(len(m), np.uint8),
                  rssi=st["rssi"][m].astype(np.uint32).astype(np.uint8))
    else:
        e = runlength_events(st, chain)
        ev = {f: np.ascontiguousarray(e[f]) for f in ("m", "bit", "reset", "rssi")}
    ev["sync"] = access_code_flags(ev["bit"], ev["reset"], chain, errors)
    return ev


def stream_lines(ev, chain, algo):
    """[(sample of the last bit, chain, algo, line)] of one stream"""
    L = orc.lib()
    frame = L.orc_frame_t1c1 if chain == 0 else L.orc_frame_s1
    prefix = b"rla;" if algo == 0 else b"t2a;"
    bits, rssi = np.ascontiguousarray(ev["bit"], np.uint8), np.ascontiguousarray(ev["rssi"], np.uint8)
    n = len(bits)
    resets = np.nonzero(ev["reset"])[0]
    buf = C.create_string_buffer(4096)
    got = C.c_int(0)
    out, busy = [], 0
    for c in np.nonzero(ev["sync"])[0]:
        if c < busy:
            continue                                               # the decoder is receiving: the flag is ignored
        end = n
        if algo == 0:                                              # a run-length reset resets the decoder too
            r = np.searchsorted(resets, c, side="right")
            if r < len(resets):
                end = int(resets[r])
        used = frame(bits[c:end], rssi[c:end], end - c, prefix, buf, len(buf), C.byref(got))
        if got.value:
            out.append((int(ev["m"][c + used - 1]), chain, algo, buf.value.decode().rstrip("\n")))
        busy = c + used
    return out


def run_lines(cu8, flags, lock=(2, 2), errors=(0, 0)):
    """the reference's lines (TIMESTAMP blanked) for a capture, reference-style flags and receiver settings
    lock = (T1/C1, S1) clock-lock thresholds, errors = (T1/C1, S1) access-code errors"""
    return run_lines_many(cu8, flags, [(lock, errors)])[0]


def run_lines_many(cu8, flags, settings):
    """run_lines for several (lock, errors) settings of one capture; the oracle's stages are computed once"""
    o = orc.opts_from_flags(flags)
    cu8 = np.ascontiguousarray(cu8, np.uint8)
    found = [[] for _ in settings]
    for chain, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)):
        if not on:
            continue
        st = orc.stages(cu8, o, chain)
        for algo, alg_on in ((0, o.rla_enabled), (1, o.t2_enabled)):
            if alg_on:
                for f, (lock, errors) in zip(found, settings):
                    f += stream_lines(stream_events(st, chain, algo, lock[chain], errors[chain]), chain, algo)
        del st
    out = []
    for f in found:
        f.sort(key=lambda x: (x[0], x[1], x[2]))
        lines = [l for _, _, _, l in f]
        if not o.show_algorithm:
            lines = [l[4:] for l in lines]
        out.append([orc.blank_ts(l) for l in lines])
    return out
