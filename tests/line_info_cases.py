"""Per-line carrier offsets (wmb_take_lines_info, wmb_line_info): the restatement on the CPU oracle and the checks shared
by the CPU-simulation tests (test_line_info.py) and the GPU tests (test_line_info_gpu.py).

The restatement: for each line the oracle prints, its access-code match is bit c of its stream (receiver_oracle), on
decimated sample s = m[c].  The window is [s - 384, s - 128) for T1/C1 and [s - 1367, s - 586) for S1, clipped at the
stream's first sample; sum = sum of rint(fir * 2^24) over it in float64, fir the oracle's post-FIR discriminator output
before the DC block.  The library must give the same (sync_sample, n, sum) for every line, exactly."""
import ctypes as C
import importlib

import numpy as np

import orc
import receiver_cases as rc
import receiver_oracle as ro

WINDOW = {0: (384, 128), 1: (1367, 586)}       # samples before the match: [s - lo, s - hi)
SCALE = float(1 << 24)

# Offsets planted by the synthetic emitters come back within this bound (Hz), both algorithms.  Worst case measured on
# the CPU build over the captures of PLANTED (t1x2, mixed, mixed -o, mixed at 2.4 MS/s with -d 3 -s): 75 Hz, a weak
# T1 emitter (amp 40) at -12 kHz; the bound leaves twice that.  The two algorithms report a match a few samples apart,
# so their windows sit at different phases of the chip pattern; S1's 781 samples are 31.99 chips, not a whole number,
# which leaves a phase-dependent residue of tens of Hz (measured: rla +32 Hz, t2a -2 Hz mean on the same S1 emitter).
# Lines whose window overlaps another emitter's burst are left out (collided()): there the discriminator follows the
# stronger telegram, or neither (measured up to 11.8 kHz off).
BOUND_HZ = 150.0

# (emitter config, flags, bytes, fs, seed, center shift)
PLANTED = [("t1x2", "-v", 16 << 20, 1.6e6, 0xB2000071, 0.0), ("mixed", "-v", 8 << 20, 1.6e6, 0xB2000072, 0.0),
           ("mixed", "-v -d 3 -s", 12 << 20, 2.4e6, 0xB2000073, 325e3), ("mixed", "-v -o", 8 << 20, 1.6e6, 0xB2000074, 0.0)]


def window_sum(fir, s, chain, first=0):
    a, b = WINDOW[chain]
    lo = max(s - a, first)
    hi = max(s - b, lo)
    return hi - lo, int(np.rint(fir[lo:hi].astype(np.float64) * SCALE).sum())


def _stream_info(ev, chain, algo, fir):
    """receiver_oracle.stream_lines, plus each line's (sync sample, n, sum)"""
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
            continue
        end = n
        if algo == 0:
            r = np.searchsorted(resets, c, side="right")
            if r < len(resets):
                end = int(resets[r])
        used = frame(bits[c:end], rssi[c:end], end - c, prefix, buf, len(buf), C.byref(got))
        if got.value:
            s = int(ev["m"][c])
            out.append((int(ev["m"][c + used - 1]), chain, algo, buf.value.decode().rstrip("\n"), s) + window_sum(fir, s, chain))
        busy = c + used
    return out


def oracle_info(cu8, flags, lock=(2, 2), errors=(0, 0), prefilter=0):
    """[(line with TS blanked, sync_sample, n, sum, chain, algo)] in print order"""
    o = orc.opts_from_flags(flags)
    o.prefilter = prefilter
    cu8 = np.ascontiguousarray(cu8, np.uint8)
    found = []
    for chain, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)):
        if not on:
            continue
        st = orc.stages(cu8, o, chain)
        for algo, alg_on in ((0, o.rla_enabled), (1, o.t2_enabled)):
            if alg_on:
                found += _stream_info(ro.stream_events(st, chain, algo, lock[chain], errors[chain]), chain, algo, st["fir"])
        del st
    found.sort(key=lambda x: (x[0], x[1], x[2]))
    out = []
    for _, chain, algo, line, s, n, sm in found:
        if not o.show_algorithm:
            line = line[4:]
        out.append((orc.blank_ts(line), s, n, sm, chain, algo))
    return out


def product_info(pkg, lib, cu8, flags, lock=(2, 2), errors=(0, 0), pushes=None, **tuning):
    """the library's lines and records for a capture: pushes = list of byte counts (None: one process call)"""
    with pkg.WmbusB200(flags, lib=lib, clock_lock=lock, access_code_errors=errors, **tuning) as ctx:
        if pushes is None:
            lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
        else:
            off = 0
            for n in pushes + [len(cu8)]:
                n = min(n, len(cu8) - off)
                ctx.push(cu8.ctypes.data + off, n)
                off += n
            ctx.poll_flush()
            lines, recs = ctx.take_lines(info=True)
        st = ctx.stats()
    return [orc.blank_ts(l) for l in lines], recs, st


def check_parity(pkg, lib, cu8, flags, lock=(2, 2), errors=(0, 0), pushes=None, **tuning):
    """every line's (sync_sample, n, sum), in order, equals the restatement exactly"""
    want = oracle_info(cu8, flags, lock, errors, tuning.get("prefilter", 0))
    lines, recs, st = product_info(pkg, lib, cu8, flags, lock, errors, pushes, **tuning)
    assert lines == [w[0] for w in want], (flags, tuning, len(lines), len(want))
    assert len(recs) == len(lines)
    a_flag = "-a" in flags.split()
    for i, (w, r) in enumerate(zip(want, recs)):
        got = (int(r["sync_sample"]), int(r["n"]), int(r["sum"]), int(r["chain"]), int(r["algo"]))
        assert got == w[1:], (flags, tuning, i, w[0], got, w[1:])
        assert int(r["valid"]) == (0 if a_flag or w[2] == 0 else 1)
        assert int(r["crc_ok"]) == int(w[0].split(";")[2 if w[0][:4] in ("rla;", "t2a;") else 1])
    assert st.overflow_batches == 0
    return want, recs


def offset_hz(rec, gain):
    """offset_hz of a record from its sum, restated (gain: the chain's FIR DC gain)"""
    return rec["sum"] / rec["n"] / SCALE * 400e3 / gain


def fir_gains():
    """sum of the post-demod FIR taps, in double, per chain (wmb_chain.cuh c_fir_t1c1 / c_fir_s1, float literals)"""
    import re
    import os
    src = open(os.path.join(rc.ROOT, "rtl-wmbus_b200", "csrc", "wmb_chain.cuh")).read()
    out = []
    for name in ("c_fir_t1c1", "c_fir_s1"):
        body = re.search(name + r"\[\d+\] = \{([^}]*)\}", src).group(1)
        taps = np.array([float(t) for t in body.replace("\n", " ").split(",") if t.strip()], np.float32)
        out.append(float(taps.astype(np.float64).sum()))
    return out


def ident_of(line):
    f = line.split(";")
    if f[0] in ("rla", "t2a"):
        f = f[1:]
    return int(f[6], 16)


def collided(plan, emitters, ident, m, d):
    """the window of the match at decimated sample m (of emitter `ident`) overlaps another emitter's burst"""
    ei = [e.ident for e in emitters].index(ident)
    lo, hi = (m - 1400) * d, m * d
    return any(p.emitter != ei and p.start_iq < hi and p.start_iq + p.n_iq > lo for p in plan)


def planted_errors(lines, recs, emitters, plan, d, shift_hz=0.0):
    """({(ident, algo): [offset_hz - planted]}, lines left out) of the CRC-ok lines whose window holds no other
    emitter's burst (two telegrams on the air at once: the discriminator follows the stronger one, or neither);
    shift_hz as synth_capture's center_shift_hz"""
    by_id = {}
    for e in emitters:
        by_id[e.ident] = e
    out, skipped = {}, 0
    for l, r in zip(lines, recs):
        if not r["crc_ok"]:
            continue
        e = by_id[ident_of(l)]
        assert r["valid"] == 1
        if collided(plan, emitters, e.ident, int(r["sync_sample"]), d):
            skipped += 1
            continue
        shift = shift_hz if e.mode != "S1" else -shift_hz
        planted = e.offset_hz + shift - r["carrier_hz"]
        out.setdefault((e.ident, int(r["algo"])), []).append(float(r["offset_hz"]) - planted)
    return out, skipped


def synth_mod():
    return importlib.import_module("rtl-wmbus_b200.synth")


def check_planted(pkg, lib, config, flags, n_bytes, fs, seed, shift_hz=0.0, bound=BOUND_HZ, **kw):
    """every CRC-ok line's offset lies within `bound` of its emitter's planted offset, for both algorithms;
    returns the worst error"""
    synth = synth_mod()
    em = synth.default_emitters(config)
    buf, plan = synth.synth_capture(n_bytes, fs=fs, emitters=em, seed=seed, center_shift_hz=shift_hz)
    cu8 = np.ascontiguousarray(buf.numpy())
    with pkg.WmbusB200(flags, lib=lib, **kw) as ctx:
        lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    errs, skipped = planted_errors(lines, recs, em, plan, int(round(fs / 800e3)), shift_hz)
    assert skipped <= len(lines) // 5, (skipped, len(lines))
    assert {a for _, a in errs} == {0, 1}, errs.keys()
    assert len({i for i, _ in errs}) == len(em), (config, sorted(errs))
    worst = max(abs(x) for v in errs.values() for x in v)
    assert worst <= bound, (config, flags, worst, {k: (min(v), max(v)) for k, v in errs.items()})
    if shift_hz:
        for l, r in zip(lines, recs):
            want = 325e3 if (l.split(";")[1] if l[:4] in ("rla;", "t2a;") else l.split(";")[0]) != "S1" else -325e3
            assert r["carrier_hz"] == want
    return worst
