"""The burst report (wmb_set_bursts / wmb_take_bursts): the restatement on the CPU oracle's stages and the checks shared
by the CPU-simulation tests (test_bursts.py) and the GPU tests (test_bursts_gpu.py).

The restatement follows the definition in include/wmbus_b200.h sample by sample, in numpy, on the oracle's (unsigned)rssi
and post-FIR discriminator output: above = rssi >= level; runs of above samples joined across fewer than G below ones;
cut at multiples of P = 2^16 at least Q = 2^17 after the run start; pieces of at least Lmin samples reported with their
rssi sum, peak and the sum of rint(fir * 2^24) over [start + g0, min(end, start + g0 + w)).  A run whose end the input
does not confirm (fewer than G samples after its last above sample) is closed there at end of input, flagged at_end."""
import importlib

import numpy as np

import orc

Q, P = 1 << 17, 1 << 16
CONTINUED, CUT, AT_END = 1, 2, 4
CONST = {0: dict(G=64, Lmin=256, g0=64, w=256), 1: dict(G=196, Lmin=782, g0=196, w=781)}
SCALE = float(1 << 24)

# the CLI's default levels (T1/C1, S1), DESIGN.md §8
DEFAULT_LEVEL = (14, 14)

FIELDS = ("start_sample", "end_sample", "peak", "rssi_sum", "n", "sum", "chain", "flags")


def pieces(rssi, fir, chain, level, m0=0):
    """[(start, end, peak, rssi_sum, n, sum, chain, flags)] of one chain, absolute sample indices (stream sample 0 is
    decimated sample m0)"""
    c = CONST[chain]
    G, Lmin, g0, w = c["G"], c["Lmin"], c["g0"], c["w"]
    rssi = np.asarray(rssi)
    M = len(rssi)
    idx = np.nonzero(rssi >= level)[0]
    if not len(idx):
        return []
    brk = np.nonzero(np.diff(idx) - 1 >= G)[0]
    starts = idx[np.r_[0, brk + 1]]
    lasts = idx[np.r_[brk, len(idx) - 1]]
    r64 = rssi.astype(np.uint64)
    out = []
    for k, (s, la) in enumerate(zip(starts.tolist(), lasts.tolist())):
        e = la + 1
        at_end = k == len(starts) - 1 and la + G > M - 1
        S, E = m0 + s, m0 + e
        c0 = -(-(S + Q) // P) * P
        bounds = [S] + list(range(c0, E, P)) + [E]
        for j in range(len(bounds) - 1):
            a, b = bounds[j], bounds[j + 1]
            if b - a < Lmin:
                continue
            fl = (CONTINUED if j > 0 else 0) | (CUT if j < len(bounds) - 2 else 0) | (AT_END if at_end and j == len(bounds) - 2 else 0)
            lo, hi = a - m0, b - m0
            wlo, whi = lo + g0, min(hi, lo + g0 + w)
            n = max(0, whi - wlo)
            sm = int(np.rint(fir[wlo:wlo + n].astype(np.float64) * SCALE).sum()) if n else 0
            seg = r64[lo:hi]
            out.append((a, b, int(seg.max()), int(seg.sum()), n, sm, chain, fl))
    return out


def oracle_bursts(cu8, flags, level, prefilter=0, m0=0):
    """the restatement for a capture: pieces of every enabled chain, ordered by (start, chain)"""
    o = orc.opts_from_flags(flags)
    o.prefilter = prefilter
    cu8 = np.ascontiguousarray(cu8, np.uint8)
    out = []
    for chain, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)):
        if not on or not level[chain]:
            continue
        st = orc.stages(cu8, o, chain)
        rssi = st["rssi"].astype(np.uint32).astype(np.uint8)
        out += pieces(rssi, st["fir"], chain, level[chain], m0)
        del st
    out.sort(key=lambda x: (x[0], x[6]))
    return out


def as_tuples(recs):
    return [tuple(int(r[f]) for f in FIELDS) for r in recs]


def product_bursts(pkg, lib, cu8, flags, level, pushes=None, **tuning):
    """(lines, burst records, stats) of the library for a capture; pushes: byte counts (None: one process call)"""
    with pkg.WmbusB200(flags, lib=lib, burst_level=level, **tuning) as ctx:
        if pushes is None:
            lines = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
            recs = ctx.take_bursts()
        else:
            off, got = 0, []
            for n in pushes + [len(cu8)]:
                n = min(n, len(cu8) - off)
                ctx.push(cu8.ctypes.data + off, n)
                got.append(ctx.take_bursts())
                off += n
            ctx.poll_flush()
            got.append(ctx.take_bursts())
            lines = ctx.take_lines()
            recs = np.concatenate(got)
        st = ctx.stats()
    return lines, recs, st


def check_parity(pkg, lib, cu8, flags, level=DEFAULT_LEVEL, pushes=None, **tuning):
    """every record's (start, end, peak, rssi_sum, n, sum, chain, flags) equals the restatement, in order"""
    want = oracle_bursts(cu8, flags, level, tuning.get("prefilter", 0))
    _, recs, st = product_bursts(pkg, lib, cu8, flags, level, pushes, **tuning)
    got = as_tuples(recs)
    assert got == want, (flags, tuning, len(got), len(want), first_diff(got, want))
    a_flag = "-a" in flags.split()
    for r in recs:
        assert int(r["valid"]) == (0 if a_flag or r["n"] == 0 else 1)
        assert np.isnan(r["offset_hz"]) == (not r["valid"])
    return want, recs


def first_diff(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return i, x, y
    return min(len(a), len(b)), a[len(b):len(b) + 1], b[len(a):len(a) + 1]


def synth_mod():
    return importlib.import_module("rtl-wmbus_b200.synth")


def cw_capture(n_bytes, fs=1.6e6, seed=0xB2000091, tone_hz=20e3, amp=40.0, on=(0.2, 0.8), emitters=None):
    """noise + an in-band CW carrier over the fraction `on` of the capture (several 2^17 spans long)"""
    synth = synth_mod()
    buf, plan = synth.synth_capture(n_bytes, fs=fs, emitters=emitters or [], seed=seed)
    iq = buf.numpy().astype(np.float32).reshape(-1, 2) - 127.5
    n = len(iq)
    a, b = int(n * on[0]), int(n * on[1])
    t = np.arange(a, b, dtype=np.float64)
    ph = 2 * np.pi * tone_hz / fs * t
    iq[a:b, 0] += (amp * np.cos(ph)).astype(np.float32)
    iq[a:b, 1] += (amp * np.sin(ph)).astype(np.float32)
    return np.ascontiguousarray(np.clip(np.rint(iq + 127.5), 0, 255).astype(np.uint8).reshape(-1)), plan


# Planted offsets come back within these bounds (Hz).  Measured on the CPU build with planted_capture() (a T1 emitter at
# +8 kHz, an S1 emitter at +2 kHz, a T1 emitter at +-60 kHz that nothing decodes): in-tune worst 106 Hz (S1: its 781-sample
# window is 31.99 chips, a phase-dependent residue), the far emitter's worst 55 Hz.  The bounds leave about twice that.
BOUND_HZ = 220.0
BOUND_FAR_HZ = 120.0


def planted_emitters(far_hz=60e3):
    """two in-tune emitters and one T1 emitter far_hz off (returned second)"""
    E = synth_mod().Emitter
    far = E("T1", 0x55500001, amp=90.0, offset_hz=far_hz, l_field=0x19, period_s=0.13, start_s=0.050, seed=25)
    return [E("T1", 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x29, period_s=0.11, start_s=0.004, seed=21),
            E("S1", 0x19131290, amp=70.0, offset_hz=2e3, l_field=0x19, period_s=0.19, start_s=0.080, seed=24), far], far


def planted_capture(emitters, n_bytes=8 << 20, seed=0xB2000092, center_shift_hz=0.0):
    buf, plan = synth_mod().synth_capture(n_bytes, fs=1.6e6, emitters=emitters, seed=seed, center_shift_hz=center_shift_hz)
    return np.ascontiguousarray(buf.numpy()), plan


def planted_errors(recs, emitters, plan, d=2):
    """({emitter index: [offset_hz - planted]}, bursts left out): the bursts of an emitter's chain that overlap one of
    its telegrams and no other emitter's"""
    errs, skipped = {}, 0
    for ei, e in enumerate(emitters):
        ch = 1 if e.mode == "S1" else 0
        for r in recs[recs["chain"] == ch]:
            s, t = int(r["start_sample"]) * d, int(r["end_sample"]) * d
            if not any(p.emitter == ei and p.start_iq < t and p.start_iq + p.n_iq > s for p in plan):
                continue
            if any(p.emitter != ei and p.start_iq < t and p.start_iq + p.n_iq > s for p in plan):
                skipped += 1
                continue
            errs.setdefault(ei, []).append(float(r["offset_hz"]) - (e.offset_hz - r["carrier_hz"]))
    return errs, skipped


def check_planted(pkg, lib, cu8, emitters, plan, far, **kw):
    """every emitter's bursts within the bounds; returns (errors, left out, the far emitter's mean reported offset)"""
    with pkg.WmbusB200("-v", lib=lib, burst_level=DEFAULT_LEVEL, **kw) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        recs = ctx.take_bursts()
    errs, skipped = planted_errors(recs, emitters, plan)
    fi = emitters.index(far)
    assert set(errs) == set(range(len(emitters))), sorted(errs)
    for ei, v in errs.items():
        bound = BOUND_FAR_HZ if ei == fi else BOUND_HZ
        assert len(v) >= 5 and max(abs(x) for x in v) <= bound, (ei, min(v), max(v))
    return errs, skipped, far.offset_hz + float(np.mean(errs[fi]))
