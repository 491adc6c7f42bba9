"""Soft-decision repair of S1 telegrams (wmbus_b200_framer.h, wmb_frame_repair_s1_soft), restated in plain Python: the
soft value per S1 chip on the CPU oracle's stages, and the pair rule on top of repair_cases (the erasure rule, which runs
first); with the helpers shared by the CPU-simulation tests (test_s1_soft_repair.py) and the GPU tests
(test_s1_soft_repair_gpu.py).

Soft value of bit event e of an S1 stream at decimated sample m: chip centre c = m - D_T2 (t2a) or
c = m - D_RL - 24 (n - 1 - i) (rla, the i-th of the n events at sample m); v = floor(sum of rint(fir * 2^24) over
[c - 8, c + 8) / 2^SHIFT), clamped to +-32767; -32768 when the window starts before the first sample or n - 1 - i > 31.

S1 frame: bit 0 the flagged bit, byte l at bits [1 + 16 l, 17 + 16 l); pair p = 8 l + b (data bit b, MSB first) is
bits (1 + 2 p, 2 + 2 p), "01" = 1.  d = v2 - v1 (0 when a chip has no value); ML = d > 0, or for d = 0 the received bit of a
valid pair, else 0; key (has a value, |d|, p).  In a failing block every searchable pair takes its ML bit and the
min(s_max, pairs) of lowest key are searched; exactly one of the 2^K patterns (0: pure ML) must pass."""
import ctypes as C

import numpy as np

import orc
import receiver_oracle as ro
import repair_cases as rc
import soft_repair_cases as sc
import t1_soft_cases as tc

SCALE = float(1 << 24)
NONE = sc.NONE
D_T2, D_RL, SHIFT = 7, 13, 14      # include/wmbus_b200_framer.h WMB_SOFT_S1_D_T2 / _D_RL / _SHIFT (DESIGN.md section 8)
D_RANGE = range(7, 49)             # D >= 7: the window [c - 8, c + 8) ends at the event's own sample
S_MAX = 6


# ---- the soft value per chip --------------------------------------------------------------------------------------------

def soft_values(fir, ev, algo, d_t2=D_T2, d_rl=D_RL, shift=SHIFT):
    """int16 soft value of every event of one S1 stream (events since the start of fir)"""
    m = ev["m"].astype(np.int64)
    n = len(m)
    after = np.zeros(n, np.int64)
    if algo == 0 and n:
        starts = np.r_[True, m[1:] != m[:-1]]
        run_id = np.cumsum(starts) - 1
        run_end = np.r_[np.nonzero(starts)[0][1:], n]
        after = run_end[run_id] - 1 - np.arange(n)
        c = m - d_rl - 24 * after
    else:
        c = m - d_t2
    x = np.rint(np.asarray(fir, np.float64) * SCALE).astype(np.int64)
    cs = np.r_[0, np.cumsum(x)]
    lo, hi = c - 8, c + 8
    ok = (lo >= 0) & (after <= 31) & (hi <= len(x))
    s = np.zeros(n, np.int64)
    s[ok] = cs[hi[ok]] - cs[lo[ok]]
    raw = np.floor_divide(s, 1 << shift)
    v = np.clip(raw, -32767, 32767)
    v[~ok] = NONE
    return v.astype(np.int16), raw, ok


def oracle_streams(cu8, flags, lock=(2, 2), errors=(0, 0)):
    """{algo: (events, soft values)} of the S1 chain"""
    o = orc.opts_from_flags(flags)
    st = orc.stages(np.ascontiguousarray(cu8, np.uint8), o, 1)
    out = {}
    for algo, on in ((0, o.rla_enabled), (1, o.t2_enabled)):
        if on:
            ev = ro.stream_events(st, 1, algo, lock[1], errors[1])
            out[algo] = (ev, soft_values(st["fir"], ev, algo)[0])
    return out


def d_scores(cu8, flags="", lock=(2, 2)):
    """{algo: {D: mean of (2 chip - 1) v over the chips [17, P) of every CRC-clean S1 line}} for D in D_RANGE, and the
    largest |unclamped value| over those chips at the constants' delays"""
    o = orc.opts_from_flags(flags)
    st = orc.stages(np.ascontiguousarray(cu8, np.uint8), o, 1)
    L = orc.lib()
    buf = C.create_string_buffer(4096)
    got = C.c_int(0)
    out, peak = {}, 0
    for algo in (0, 1):
        ev = ro.stream_events(st, 1, algo, lock[1], 0)
        bits, rssi = np.ascontiguousarray(ev["bit"], np.uint8), np.ascontiguousarray(ev["rssi"], np.uint8)
        resets = np.nonzero(ev["reset"])[0]
        sel, busy = [], 0
        for c in np.nonzero(ev["sync"])[0]:
            if c < busy:
                continue
            end = len(bits)
            if algo == 0:
                r = np.searchsorted(resets, c, side="right")
                if r < len(resets):
                    end = int(resets[r])
            used = L.orc_frame_s1(bits[c:end], rssi[c:end], end - c, b"", buf, len(buf), C.byref(got))
            if got.value and buf.value.startswith(b"S1;1;"):
                sel.append(np.arange(c + 17, c + used))
            busy = c + used
        idx = np.concatenate(sel)
        sign = 2 * bits[idx].astype(np.int64) - 1
        scores = {}
        for d in D_RANGE:
            v, raw, ok = soft_values(st["fir"], ev, algo, d, d)
            v, raw, ok = v[idx].astype(np.int64), raw[idx], ok[idx]
            scores[d] = float((sign[ok] * v[ok]).mean())
            if d == (D_RL if algo == 0 else D_T2):
                peak = max(peak, int(np.abs(raw[ok]).max()))
        out[algo] = scores
    return out, peak


def polled_soft(pkg, lib, cu8, flags, batching="1mib", batch_mib=1):
    """{(chain, algo, ordinal): soft values or None} of every frame a manual_frames context with S1 values polls"""
    import repair_stream_cases as rsc
    out = {}
    with pkg.WmbusB200(flags, lib=lib, manual_frames=1, soft_bits=True, soft_bits_s1=True, max_batch_mib=batch_mib) as ctx:
        def take(flush):
            arr, k = ctx.poll(flush=flush)
            for i in range(k):
                out[(arr[i].chain, arr[i].algo, arr[i].ordinal)] = ctx.frame_soft(arr[i])
        for lo, hi in rsc.pushes(len(cu8), batching):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
            take(False)
        take(True)
    return out


def check_polled_soft(got, want_s1, want_t1c1):
    """every frame's values equal the restatement's at its ordinals; returns the S1 values checked"""
    n = 0
    for (chain, algo, ordinal), v in got.items():
        assert v is not None
        ref = (want_s1 if chain == 1 else want_t1c1)[algo][1][ordinal:ordinal + len(v)]
        assert np.array_equal(v, ref), (chain, algo, ordinal, np.nonzero(v != ref)[0][:5])
        n += len(v) if chain == 1 else 0
    return n


# ---- the S1 soft repair rule ---------------------------------------------------------------------------------------------

def s1_length(bits):
    L = rc.word2([int(x) & 1 for x in bits[:17]], 2, 8)
    return L, rc.tlg_len_a(L)


def pair(bits, soft, p):
    """(ML bit, key, hard bit or None for a violation) of pair p"""
    a, c = int(bits[1 + 2 * p]) & 1, int(bits[2 + 2 * p]) & 1
    v1, v2 = int(soft[1 + 2 * p]), int(soft[2 + 2 * p])
    has = v1 != NONE and v2 != NONE
    d = v2 - v1 if has else 0
    ml = 1 if d > 0 else 0 if d < 0 else (c if a != c else 0)
    return ml, (int(has), abs(d), p), (c if a != c else None)


def repair_soft_s1(bits, rssi, soft, s_max, had_line):
    """the soft rule on an S1 candidate (the caller checks that it is one): a dict like repair_cases.repair's"""
    L, n = s1_length(bits)
    P = 1 + 16 * n
    ml, key, hard = {}, {}, {}
    for p in range(8, 8 * n):
        ml[p], key[p], hard[p] = pair(bits, soft, p)
    cur = {p: (hard[p] if hard[p] is not None else 0) for p in hard}

    def byte(l, src):
        return sum(src[8 * l + b] << (7 - b) for b in range(8))

    out = dict(outcome=rc.UNREPAIRABLE, erasures=0, blocks=0, had_line=had_line)
    changed = blocks = 0
    for off, blk in rc.blocks_a(n):
        pairs = list(range(8 * max(off, 1), 8 * (off + blk)))
        q = [L if l == 0 else byte(l, cur) for l in range(off, off + blk)]
        if all(hard[p] is not None for p in pairs) and rc.block_ok(q):
            continue
        for p in pairs:
            cur[p] = ml[p]
        sel = sorted(pairs, key=lambda p: key[p])[:min(s_max, len(pairs))]
        passing = []
        for x in range(1 << len(sel)):
            trial = dict(cur)
            for t, p in enumerate(sel):
                if x >> t & 1:
                    trial[p] ^= 1
            q = [L if l == 0 else byte(l, trial) for l in range(off, off + blk)]
            if rc.block_ok(q):
                passing.append(x)
        if len(passing) != 1:
            out["outcome"] = rc.AMBIGUOUS if passing else rc.UNREPAIRABLE
            return out
        for t, p in enumerate(sel):
            if passing[0] >> t & 1:
                cur[p] ^= 1
        changed += sum(1 for p in pairs if hard[p] != cur[p])
        blocks += 1
    pkt = [L] + [byte(l, cur) for l in range(1, n)]
    datagram = pkt[:10] + [x for off, blk in rc.blocks_a(n)[1:] for x in pkt[off:off + blk - 2]]
    out.update(outcome=rc.REPAIRED, erasures=min(changed, 255), blocks=blocks, mode="S1", crc_ok=1, ok_3of6=1,
               packet_rssi=int(rssi[1]), current_rssi=int(rssi[P - 1]), serial=int.from_bytes(bytes(pkt[4:8]), "little"),
               datagram=bytes(datagram), consumed=P)
    return out


def restated(orc_mod, c, f, e_max, s_max):
    """wmb_frame_repair_s1_soft of one corpus case, restated: the erasure rule, then the soft rule on its candidates"""
    w = np.ctypeslib.as_array(f.bits, (f.nbits,))
    r = rc.repair(orc_mod, c["chain"], w & 1, (w >> 1) & 0xFF, w >> 9, f.sync_sample, e_max)
    if not s_max or c.get("soft") is None or c["chain"] != 1 or r["outcome"] not in (rc.TOO_MANY, rc.UNREPAIRABLE):
        return r
    bits = [int(x) & 1 for x in c["bits"]]
    L, n = s1_length(bits)
    P = 1 + 16 * n
    if n < 12 or any(int(x) < rc.CAPTURE_THRESHOLD for x in c["rssi"][:P - 1]):
        return r
    r = repair_soft_s1(bits, c["rssi"], c["soft"], s_max, r["had_line"])
    if r["outcome"] == rc.REPAIRED:
        r["end_sample"] = f.sync_sample + int(w[r["consumed"] - 1] >> 9)
    return r


# ---- the corpus ---------------------------------------------------------------------------------------------------------

def s1_bits(synth, L, k):
    """the frame bits of a clean S1 telegram (flagged bit first, 8 idle pairs after it) and its datagram"""
    from test_repair import telegram_chips
    return telegram_chips(synth, "S1", L, k)


def pair_chips(p):
    return [1 + 2 * p, 2 + 2 * p]


def corpus(synth, s_max, seed=13):
    """S1 telegrams with 0 .. s_max + 1 wrong pairs per block -- one chip flipped (a violation, weak or full swing), both
    chips flipped (a valid wrong bit), weak pairs (both chips on the wrong tone at a fifth of the deviation) -- some chips
    without a value, RSSI drop-outs, truncated lists"""
    rng = np.random.default_rng(seed)
    cases = []
    for L in (9, 0x0E, 0x19, 0x2E, 0x44, 0x7F, 0xB3, 0xFF):
        for k in range(3):
            bits, p = s1_bits(synth, L, k)
            n = rc.tlg_len_a(L)
            P = 1 + 16 * n
            soft = tc.clean_soft(rng, bits)
            strong = bool(rng.integers(0, 4) == 0)
            for off, blk in rc.blocks_a(n):
                pairs = np.arange(8 * max(off, 1), 8 * (off + blk))
                for q in rng.choice(pairs, min(int(rng.integers(0, s_max + 4)), len(pairs)), replace=False):
                    chips = pair_chips(int(q))
                    kind = int(rng.integers(0, 3))
                    pick = [chips[int(rng.integers(0, 2))]] if kind == 0 else chips
                    for j in pick:
                        bits[j] ^= 1
                        mag = rng.integers(2000, 6000) if strong and kind != 2 else rng.integers(10, 600)
                        soft[j] = (2 * int(bits[j]) - 1) * mag
            for j in rng.choice(np.arange(17, P), int(rng.integers(0, 3)), replace=False):
                soft[j] = NONE
            rssi = np.full(len(bits), 100, np.uint8)
            tail = int(rng.integers(0, 12))
            if tail == 0:
                rssi[int(rng.integers(17, P - 1))] = 2               # an RSSI drop-out
            elif tail == 1:
                bits, rssi, soft = bits[:P - 5], rssi[:P - 5], soft[:P - 5]      # a truncated list
            cases.append(dict(chain=1, bits=bits, rssi=rssi, soft=soft, sent=p, wire=synth.frame_a(p)))
    return cases


def ambiguous_cases(synth):
    """a block where a weight-6 code word of the shortened CRC code (the least weight there is) lies on six data pairs:
    three of its pairs are received flipped (both chips, a valid wrong bit) and all six are the least reliable, so from
    K = 6 on two patterns pass (the three received ones flipped back, or the other three flipped) and the block is
    AMBIGUOUS; below, it is REPAIRED or UNREPAIRABLE"""
    out = []
    bits0, p = s1_bits(synth, 0x19, 0)
    # the first block's searchable bits are its last 88, a later block's all 144: a word of the 88-bit code is one of
    # the first block's after the L byte (the syndrome of a bit depends only on its distance from the block's end)
    for nbits, first_pair in ((88, 8), (144, 8 * 12)):
        bits = bits0.copy()
        pos = [first_pair + x for x in sc.min_weight_word(nbits, 6)]
        soft = ((2 * bits.astype(np.int64) - 1) * 4000).astype(np.int16)
        for t, q in enumerate(sorted(pos)):
            a, c = pair_chips(q)
            if t < 3:
                bits[a] ^= 1; bits[c] ^= 1
            soft[a] = (2 * int(bits[a]) - 1) * 3
            soft[c] = (2 * int(bits[c]) - 1) * 3
        out.append(dict(chain=1, bits=bits, rssi=np.full(len(bits), 100, np.uint8), soft=soft, sent=p,
                        wire=synth.frame_a(p), weight=6))
    return out


def soft_ptrs(cases):
    arrs = [np.ascontiguousarray(c["soft"], np.int16) if c.get("soft") is not None else None for c in cases]
    return arrs, (C.c_void_p * len(cases))(*[None if a is None else a.ctypes.data for a in arrs])


def run_rule(lib, pkg, cases, e_max, s_max, chunk=1000):
    """host twin and device (K4, K4R, K4S) on every case"""
    from test_repair import make_frames
    frames, keep = make_frames(pkg, cases)
    arrs, ptrs = soft_ptrs(cases)
    host = (pkg.WmbRepaired * len(cases))()
    for i in range(len(cases)):
        assert lib.wmb_frame_repair_s1_soft(C.addressof(frames[i]), ptrs[i], e_max, s_max, C.addressof(host[i])) == 0
    dev = (pkg.WmbRepaired * len(cases))()
    fs, rs, ps = C.sizeof(pkg.WmbFrame), C.sizeof(pkg.WmbRepaired), C.sizeof(C.c_void_p)
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        for lo in range(0, len(cases), chunk):
            n = min(chunk, len(cases) - lo)
            assert lib.wmb_frame_repair_s1_soft_device(ctx._ctx, C.addressof(frames) + lo * fs, C.addressof(ptrs) + lo * ps,
                                                       n, e_max, s_max, C.addressof(dev) + lo * rs) == 0, lib.wmb_last_error()
    return (frames, keep, arrs), host, dev


def within_k(c, s_max):
    """the wrong bits of a corpus telegram lie among its K searched pairs, block by block (and it has some): every pair
    whose ML bit is not the sent one is searched, and the L byte is intact"""
    bits = c["bits"]
    L, n = s1_length(bits)
    P = 1 + 16 * n
    if len(bits) < P or n < 12 or (c["rssi"][:P - 1] < rc.CAPTURE_THRESHOLD).any() or L != c["wire"][0]:
        return False
    sent = [c["wire"][l] >> (7 - b) & 1 for l in range(n) for b in range(8)]
    wrong_any = False
    for off, blk in rc.blocks_a(n):
        pairs = list(range(8 * max(off, 1), 8 * (off + blk)))
        info = {q: pair(bits, c["soft"], q) for q in pairs}
        wrong = {q for q in pairs if info[q][0] != sent[q]}
        wrong_any |= bool(wrong)
        if not wrong <= set(sorted(pairs, key=lambda q: info[q][1])[:s_max]):
            return False
    return wrong_any


# ---- the streaming path -------------------------------------------------------------------------------------------------

def s1_emitters(synth):
    """S1 emitters whose telegrams each lose a bit to a weak pair (both chips of pair 2 of byte 3 on the wrong tone: a
    valid wrong bit, UNREPAIRABLE for the erasure rule) or four bits of one block to a weak chip each (TOO_MANY), beside a
    clean S1 one, the T1 / S1 emitters with flipped chips of tests/test_repair.py and a C1 emitter with weak bits (chip 0:
    the L-field's first chip; byte l of an S1 telegram is chips 16 l .. 16 l + 15)"""
    from test_repair import flipped_emitters
    return [synth.Emitter("S1", 0x55001122, amp=70.0, offset_hz=-5e3, l_field=0x19, period_s=0.17, start_s=0.020, seed=71,
                          weak_flips=(16 * 3 + 4, 16 * 3 + 5)),
            synth.Emitter("S1", 0x55003344, amp=70.0, offset_hz=4e3, l_field=0x2E, period_s=0.19, start_s=0.075, seed=72,
                          weak_flips=(16 * 13 + 2, 16 * 15 + 9, 16 * 17 + 6, 16 * 20 + 11)),
            synth.Emitter("S1", 0x55005566, amp=70.0, offset_hz=1e3, l_field=0x2E, period_s=0.23, start_s=0.130, seed=73),
            ] + flipped_emitters(synth)[:2] + sc.weak_emitters(synth)[:1]


def s1_capture(n=8 << 20):
    import importlib
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = s1_emitters(synth)
    cu8, plan = synth.synth_capture(n, emitters=ems, seed=0xB200000D)
    return np.ascontiguousarray(cu8.numpy()), plan, ems


def record_tuple(r):
    import repair_stream_cases as rs
    return rs.record_tuple(r) + (r.soft_t1, r.soft_s1)


def stream(pkg, lib, cu8, flags, e_max, batching="1mib", batch_mib=1, quality=False, burst_level=None, **ctx_kw):
    """the streaming run: (records with soft_t1, soft_s1 last, lines, line info, quality, bursts, stats)"""
    import repair_stream_cases as rs
    with pkg.WmbusB200(flags, lib=lib, repair=e_max, quality=quality, burst_level=burst_level,
                       max_batch_mib=batch_mib, **ctx_kw) as ctx:
        recs = []
        for lo, hi in rs.pushes(len(cu8), batching):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
            recs += ctx.take_repairs()
        ctx.poll_flush()
        recs += ctx.take_repairs()
        if quality:
            lines, info, qual = ctx.take_lines(1, info=True, quality=True)
        else:
            (lines, info), qual = ctx.take_lines(1, info=True), None
        bursts = ctx.take_bursts() if burst_level else None
        return [record_tuple(r) for r in recs], lines, info, qual, bursts, ctx.stats()


def restated_stream(pkg, lib, cu8, flags, e_max, s_maxes, **ctx_kw):
    """{s_max: sorted record tuples} from manual framing with S1 soft values: repair_stream_cases.restated with
    wmb_frame_repair_s1_soft in place of wmb_frame_repair; soft_s1 = 1 where the S1 rule ran (an S1 candidate of the
    erasure rule that ended TOO_MANY or UNREPAIRABLE, len >= 12, no rssi drop before P - 1, soft values)"""
    import repair_stream_cases as rs
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    with pkg.WmbusB200(flags, lib=lib, manual_frames=1, soft_bits_s1=True, **ctx_kw) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True, cap=1 << 20)
        frames = sorted((arr[i] for i in range(k)), key=lambda f: (f.chain, f.algo, f.ordinal))
        busy, accepted = {}, []
        for f in frames:
            s = (f.chain, f.algo)
            if f.ordinal <= busy.get(s, -1):
                continue
            d = pkg.WmbDecoded()
            lib.wmb_frame_decode(C.addressof(f), C.addressof(d))
            busy[s] = f.ordinal + d.consumed - 1
            accepted.append((f, d, ctx.frame_soft(f)))
        out = {}
        for s_max in s_maxes:
            recs = []
            for f, d, soft in accepted:
                r, r0 = pkg.WmbRepaired(), pkg.WmbRepaired()
                sp = None if soft is None else soft.ctypes.data
                assert lib.wmb_frame_repair_s1_soft(C.addressof(f), sp, e_max, s_max, C.addressof(r)) == 0
                if r.outcome in (rc.NONE, rc.TRUNCATED):
                    continue
                assert lib.wmb_frame_repair(C.addressof(f), e_max, C.addressof(r0)) == 0
                w = np.ctypeslib.as_array(f.bits, (f.nbits,))
                soft_s1 = 0
                if s_max and soft is not None and f.chain == 1 and r0.outcome in (rc.TOO_MANY, rc.UNREPAIRABLE):
                    L, n = s1_length(w & 1)
                    P = 1 + 16 * n
                    soft_s1 = int(n >= 12 and not (((w[:P - 1] >> 1) & 0xFF) < rc.CAPTURE_THRESHOLD).any())
                if d.status == 1 and d.mode == b"C1":
                    end = d.end_sample
                else:
                    end = f.sync_sample + int(w[rs.telegram_bits(f) - 1] >> 9)
                rec = pkg.WmbRepairRecord()
                rec.sync_sample = f.sync_sample; rec.end_sample = end; rec.chain = f.chain; rec.algo = f.algo
                rec.repair = r
                rec.soft_s1 = soft_s1
                recs.append(record_tuple(rec))
            out[s_max] = sorted(recs, key=rs.key)
    return out

