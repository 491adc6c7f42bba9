"""Signal quality (wmb_set_line_quality, wmb_take_lines_quality, wmb_take_bursts_quality): the restatement on the CPU
oracle's stages and the checks shared by the CPU-simulation tests (test_line_quality.py) and the GPU tests
(test_line_quality_gpu.py).

The restatement follows the definition in include/wmbus_b200.h with one array operation per step, on the oracle's
post-FIR discriminator output `fir` over a line's or a burst's offset window [lo, hi) (line_info_cases.WINDOW,
burst_cases.CONST): x = rint(fir * 2^24); high = x n >= sum; a sample of [lo + 1, hi - 1) counts when it and both
neighbours share a class; per class the count, sum of x and sum of x^2.  bits is the number of bit events the oracle's
framer consumed from the access-code bit on.  The library must give the same six sums and bits for every line and every
burst, exactly, in order."""
import ctypes as C

import numpy as np

import burst_cases as bc
import line_info_cases as lc
import orc
import receiver_oracle as ro

SCALE = float(1 << 24)
SUMS = ("n_hi", "n_lo", "s1_hi", "s1_lo", "s2_hi", "s2_lo")

# Planted-signal bounds (DESIGN.md §8), from the CPU build on synth.py T1 / S1 emitters at amp 90, noise sigma 8:
# deviation_hz / planted deviation measured 0.787 .. 0.804 at 40, 50 and 60 kHz -- the post-demod FIR's ISI keeps the
# tones from their full swing inside a chip;
DEV_RATIO = (0.77, 0.82)
# chip_rate_hz against a planted chip clock scaled by 0.98 / 1.02, measured -2450 .. +264 ppm (T1) and -2100 .. 0 ppm
# (S1): the end sample is the last bit's decision, up to a chip after its start, over a telegram of ~400 bits;
CHIP_PPM = 3000.0
# the eye SNR of a noiseless T1 telegram, measured 13.58 .. 13.59 dB: the ceiling the FIR's ISI sets.
SNR_CEILING_DB = 13.59


def class_sums(fir, lo, hi):
    """(n_hi, n_lo, s1_hi, s1_lo, s2_hi, s2_lo) over the window [lo, hi) of fir"""
    x = np.rint(np.asarray(fir[lo:hi], np.float64) * SCALE).astype(np.int64)
    n, s = len(x), int(x.sum())
    high = x * n >= s                                          # 1. class, no division
    mid = x[1:-1]
    hi_c = high[:-2] & high[1:-1] & high[2:]                   # 1. the sample and both neighbours high ...
    lo_c = ~high[:-2] & ~high[1:-1] & ~high[2:]                # ... or all three low
    return (int(hi_c.sum()), int(lo_c.sum()), int(mid[hi_c].sum()), int(mid[lo_c].sum()),
            int((mid[hi_c] ** 2).sum()), int((mid[lo_c] ** 2).sum()))    # 2. (x^2 < 2^52, sums < 2^63)


def derive(q, gain):
    """3. (valid, deviation_hz, eye_snr_db) from a record's sums, in double"""
    nh, nl = float(q["n_hi"]), float(q["n_lo"])
    if nh < 2 or nl < 2:
        return 0, np.nan, np.nan
    mh, ml = float(q["s1_hi"]) / nh, float(q["s1_lo"]) / nl
    var = (float(q["s2_hi"]) - nh * mh * mh + float(q["s2_lo"]) - nl * ml * ml) / (nh + nl - 2.0)
    if not var > 0:
        return 0, np.nan, np.nan
    half = (mh - ml) / 2.0
    return 1, half / SCALE * 400e3 / gain, 10.0 * np.log10(half * half / var)


def _stream(ev, chain, algo, fir):
    """line_info_cases._stream_info with the framer's consumed bits and the class sums of each line"""
    L = orc.lib()
    frame = L.orc_frame_t1c1 if chain == 0 else L.orc_frame_s1
    prefix = b"rla;" if algo == 0 else b"t2a;"
    bits, rssi = np.ascontiguousarray(ev["bit"], np.uint8), np.ascontiguousarray(ev["rssi"], np.uint8)
    n = len(bits)
    resets = np.nonzero(ev["reset"])[0]
    buf = C.create_string_buffer(4096)
    got = C.c_int(0)
    out, busy = [], 0
    a, b = lc.WINDOW[chain]
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
            lo = max(s - a, 0)
            hi = max(s - b, lo)
            out.append((int(ev["m"][c + used - 1]), chain, algo, buf.value.decode().rstrip("\n"), s, int(used))
                       + class_sums(fir, lo, hi))
        busy = c + used
    return out


def oracle_quality(cu8, flags, lock=(2, 2), errors=(0, 0)):
    """[(line with TS blanked, sync_sample, end_sample, bits, chain, algo, n_hi, n_lo, s1_hi, s1_lo, s2_hi, s2_lo)] in
    print order"""
    o = orc.opts_from_flags(flags)
    cu8 = np.ascontiguousarray(cu8, np.uint8)
    found = []
    for chain, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)):
        if not on:
            continue
        st = orc.stages(cu8, o, chain)
        for algo, alg_on in ((0, o.rla_enabled), (1, o.t2_enabled)):
            if alg_on:
                found += _stream(ro.stream_events(st, chain, algo, lock[chain], errors[chain]), chain, algo, st["fir"])
        del st
    found.sort(key=lambda x: (x[0], x[1], x[2]))
    out = []
    for x in found:
        end, chain, algo, line, s, used = x[:6]
        if not o.show_algorithm:
            line = line[4:]
        out.append((orc.blank_ts(line), s, end, used, chain, algo) + tuple(x[6:]))
    return out


def oracle_burst_quality(cu8, flags, level, m0=0):
    """burst_cases.oracle_bursts with the class sums of each piece's offset window: [(start, chain, six sums)]"""
    o = orc.opts_from_flags(flags)
    cu8 = np.ascontiguousarray(cu8, np.uint8)
    out = []
    for chain, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)):
        if not on or not level[chain]:
            continue
        st = orc.stages(cu8, o, chain)
        rssi = st["rssi"].astype(np.uint32).astype(np.uint8)
        g0 = bc.CONST[chain]["g0"]
        for p in bc.pieces(rssi, st["fir"], chain, level[chain], m0):
            lo = p[0] - m0 + g0
            out.append((p[0], chain) + class_sums(st["fir"], lo, lo + p[4]))
        del st
    out.sort(key=lambda x: (x[0], x[1]))
    return out


def product(pkg, lib, cu8, flags, lock=(2, 2), errors=(0, 0), pushes=None, level=None, **tuning):
    """(lines, line quality records, bursts, burst quality records, stats) of the library with the report on"""
    with pkg.WmbusB200(flags, lib=lib, clock_lock=lock, access_code_errors=errors, burst_level=level, quality=True,
                       **tuning) as ctx:
        bursts, bq = [], []

        def take_b():
            if level is not None:
                b, q = ctx.take_bursts(quality=True)
                bursts.append(b)
                bq.append(q)
        off = 0
        for n in (pushes or []) + [len(cu8)]:
            n = min(n, len(cu8) - off)
            ctx.push(cu8.ctypes.data + off, n)
            take_b()
            off += n
        ctx.poll_flush()
        take_b()
        lines, quals = ctx.take_lines(quality=True)
        st = ctx.stats()
    if level is not None:
        bursts, bq = np.concatenate(bursts), np.concatenate(bq)
    return [orc.blank_ts(l) for l in lines], quals, bursts, bq, st


def sums_of(r):
    return tuple(int(r[f]) for f in SUMS)


def check_parity(pkg, lib, cu8, flags, lock=(2, 2), errors=(0, 0), pushes=None, level=None, **tuning):
    """every line's (sync_sample, end_sample, bits, chain, algo, six sums) and every burst's (start, chain, six sums), in
    order, equal the restatement exactly; the derived values follow from the sums"""
    want = oracle_quality(cu8, flags, lock, errors)
    lines, quals, bursts, bq, st = product(pkg, lib, cu8, flags, lock, errors, pushes, level, **tuning)
    assert lines == [w[0] for w in want], (flags, tuning, len(lines), len(want))
    assert len(quals) == len(lines)
    a_flag = "-a" in flags.split()
    gains = lc.fir_gains()
    for i, (w, r) in enumerate(zip(want, quals)):
        got = (int(r["sync_sample"]), int(r["end_sample"]), int(r["bits"]), int(r["chain"]), int(r["algo"])) + sums_of(r)
        exp = w[1:6] + ((0,) * 6 if a_flag else w[6:])
        assert got == exp, (flags, tuning, i, w[0], got, exp)
        check_derived(r, gains[int(r["chain"])], a_flag)
        rate = 800e3 * (int(r["bits"]) - 1) / (int(r["end_sample"]) - int(r["sync_sample"]))
        assert abs(float(r["chip_rate_hz"]) - rate) <= 1e-9 * rate
    if level is not None:
        wb = oracle_burst_quality(cu8, flags, level)
        gotb = [(int(q["start_sample"]), int(q["chain"])) + sums_of(q) for q in bq]
        expb = [x[:2] + ((0,) * 6 if a_flag else x[2:]) for x in wb]
        assert gotb == expb, (flags, tuning, len(gotb), len(expb), bc.first_diff(gotb, expb))
        assert np.array_equal(bq["start_sample"], bursts["start_sample"]) and np.array_equal(bq["chain"], bursts["chain"])
        for q in bq:
            check_derived(q, gains[int(q["chain"])], a_flag)
    assert st.overflow_batches == 0
    return want, quals, bq


def check_derived(r, gain, a_flag):
    valid, dev, snr = derive(r, gain)
    if a_flag:
        valid = 0
    assert int(r["valid"]) == valid, (r, valid)
    if valid:
        assert abs(float(r["deviation_hz"]) - dev) <= 1e-9 * abs(dev) + 1e-9
        assert abs(float(r["eye_snr_db"]) - snr) <= 1e-9 * abs(snr) + 1e-9
    else:
        assert np.isnan(r["deviation_hz"]) and np.isnan(r["eye_snr_db"])


# ---- planted signals (synth.py) ---------------------------------------------------------------------------------------

def planted_quality(pkg, lib, emitters, n_bytes=8 << 20, seed=0xB20000A1, noise_sigma=8.0, fs=1.6e6, flags="-v"):
    """{emitter index: (deviation_hz list, eye_snr_db list, chip_rate_hz list)} of the CRC-ok lines, by LINK_LAYER_IDENT_NO"""
    synth = lc.synth_mod()
    buf, plan = synth.synth_capture(n_bytes, fs=fs, emitters=emitters, seed=seed, noise_sigma=noise_sigma)
    cu8 = np.ascontiguousarray(buf.numpy())
    with pkg.WmbusB200(flags, lib=lib, quality=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        lines, quals = ctx.take_lines(quality=True)
    ids = [e.ident for e in emitters]
    out = {}
    for l, q in zip(lines, quals):
        if not q["crc_ok"] or not q["valid"]:
            continue
        ei = ids.index(lc.ident_of(l))
        if lc.collided(plan, emitters, ids[ei], int(q["sync_sample"]), int(round(fs / 800e3))):
            continue
        d = out.setdefault(ei, ([], [], []))
        d[0].append(float(q["deviation_hz"])); d[1].append(float(q["eye_snr_db"])); d[2].append(float(q["chip_rate_hz"]))
    return out
