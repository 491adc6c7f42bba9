"""Soft-decision repair of T1 telegrams (wmbus_b200_framer.h, wmb_frame_repair_t1_soft), restated in plain Python on top of
repair_cases (the erasure rule, which runs first) and soft_repair_cases (the soft values per chip), and the helpers shared
by the CPU-simulation tests (test_t1_soft_repair.py) and the GPU tests (test_t1_soft_repair_gpu.py).

T1 frame: bit 0 the flagged bit, byte l at bits [1 + 12 l, 13 + 12 l), its high-nibble symbol first, MSB first; symbol i
= 2 l + s covers bits [1 + 6 i, 7 + 6 i).  Centring over [13, P): y_j = v_j 2 n0 n1 - (S1 n0 + S0 n1) (or v_j when
n0 n1 = 0; 0 without a value); C(w) = sum (2 w_j - 1) y_j; ML = argmax C (ties: lower nibble), runner-up the argmax of the
other 15; delta = C(ML) - C(runner-up).  In a failing block every searchable symbol takes its ML value and the
min(s_max, symbols) of key (all chips have values, delta, index) are searched; exactly one of the 2^K patterns passes."""
import ctypes as C
import itertools

import numpy as np

import repair_cases as rc
import soft_repair_cases as sc

S_MAX = 6
NONE = sc.NONE


def word(bits, first, k):
    v = 0
    for x in bits[first:first + k]:
        v = v << 1 | int(x)
    return v


def t1_length(bits):
    L = rc.DEC_3OF6[word(bits, 1, 6)] << 4 | rc.DEC_3OF6[word(bits, 7, 6)]
    return L, rc.tlg_len_a(L)


def centred(bits, soft, P):
    """y_j for the chips [0, P) (0 before chip 13 and for a chip without a value), as Python ints"""
    b = [int(x) & 1 for x in bits[:P]]
    v = [int(x) for x in soft[:P]]
    ok = [j >= 13 and v[j] != NONE for j in range(P)]
    n1 = sum(1 for j in range(P) if ok[j] and b[j]); n0 = sum(1 for j in range(P) if ok[j] and not b[j])
    S1 = sum(v[j] for j in range(P) if ok[j] and b[j]); S0 = sum(v[j] for j in range(P) if ok[j] and not b[j])
    y = [0] * P
    for j in range(13, P):
        if ok[j]:
            y[j] = v[j] if n0 * n1 == 0 else v[j] * 2 * n0 * n1 - (S1 * n0 + S0 * n1)
    return y, ok


def symbol_scores(y6):
    """(ML, runner-up, delta) of one symbol from its six centred chip values"""
    score = [sum((2 * (rc.ENC_3OF6[n] >> (5 - j) & 1) - 1) * y6[j] for j in range(6)) for n in range(16)]
    ml = max(range(16), key=lambda n: (score[n], -n))
    ru = max((n for n in range(16) if n != ml), key=lambda n: (score[n], -n))
    return ml, ru, score[ml] - score[ru]


def repair_soft_t1(bits, rssi, soft, s_max):
    """the soft rule on a T1 candidate (the caller checks that it is one): a dict like repair_cases.repair's"""
    L, n = t1_length(bits)
    P = 1 + 12 * n
    y, ok = centred(bits, soft, P)
    hard, ml, ru, key = {}, {}, {}, {}
    for i in range(2, 2 * n):
        first = 1 + 6 * i
        hard[i] = rc.DEC_3OF6.get(word(bits, first, 6))            # None: invalid
        ml[i], ru[i], delta = symbol_scores(y[first:first + 6])
        key[i] = (int(all(ok[first:first + 6])), delta, i)
    nib = {i: (hard[i] if hard[i] is not None else 0) for i in hard}

    def byte(l):
        return nib[2 * l] << 4 | nib[2 * l + 1]

    out = dict(outcome=rc.UNREPAIRABLE, erasures=0, blocks=0, had_line=1)
    changed = blocks = 0
    for off, blk in rc.blocks_a(n):
        syms = list(range(2 * max(off, 1), 2 * (off + blk)))
        q = [L if l == 0 else byte(l) for l in range(off, off + blk)]
        if all(hard[i] is not None for i in syms) and rc.block_ok(q):
            continue
        for i in syms:
            nib[i] = ml[i]
        sel = sorted(syms, key=lambda i: key[i])[:min(s_max, len(syms))]
        passing = []
        for x in range(1 << len(sel)):
            trial = dict(nib)
            for t, i in enumerate(sel):
                if x >> t & 1:
                    trial[i] = ru[i]
            q = [L if l == 0 else trial[2 * l] << 4 | trial[2 * l + 1] for l in range(off, off + blk)]
            if rc.block_ok(q):
                passing.append(x)
        if len(passing) != 1:
            out["outcome"] = rc.AMBIGUOUS if passing else rc.UNREPAIRABLE
            return out
        for t, i in enumerate(sel):
            if passing[0] >> t & 1:
                nib[i] = ru[i]
        changed += sum(1 for i in syms if hard[i] != nib[i])
        blocks += 1
    pkt = [L] + [byte(l) for l in range(1, n)]
    datagram = pkt[:10] + [x for off, blk in rc.blocks_a(n)[1:] for x in pkt[off:off + blk - 2]]
    out.update(outcome=rc.REPAIRED, erasures=min(changed, 255), blocks=blocks, mode="T1", crc_ok=1, ok_3of6=1,
               packet_rssi=int(rssi[1]), current_rssi=int(rssi[P - 1]), serial=int.from_bytes(bytes(pkt[4:8]), "little"),
               datagram=bytes(datagram), consumed=P)
    return out


def restated(orc_mod, c, f, e_max, s_max):
    """wmb_frame_repair_t1_soft of one corpus case, restated: the erasure rule, then the soft rule on its candidates"""
    w = np.ctypeslib.as_array(f.bits, (f.nbits,))
    r = rc.repair(orc_mod, c["chain"], w & 1, (w >> 1) & 0xFF, w >> 9, f.sync_sample, e_max)
    if not s_max or c.get("soft") is None or c["chain"] != 0 or r["outcome"] not in (rc.TOO_MANY, rc.UNREPAIRABLE):
        return r
    _, line = rc.oracle_verdict(orc_mod, 0, c["bits"], c["rssi"])
    if line is None or not line.startswith("T1;0;") or t1_length(c["bits"])[1] < 12:
        return r
    r = repair_soft_t1(c["bits"], c["rssi"], c["soft"], s_max)
    if r["outcome"] == rc.REPAIRED:
        r["end_sample"] = f.sync_sample + int(w[r["consumed"] - 1] >> 9)
    return r


# ---- distance of the block codes in nibble substitutions ----------------------------------------------------------------

def substitution_syndromes(nbytes, first_byte):
    """{(symbol, mask): syndrome} of every non-zero nibble substitution of the symbols of bytes [first_byte, nbytes) of a
    block of nbytes (data, then its two CRC bytes); symbol 2 l is byte l's high nibble"""
    cols = sc.syndrome_columns(8 * nbytes)
    out = {}
    for l in range(first_byte, nbytes):
        for s in (0, 1):
            for m in range(1, 16):
                bm = m << 4 if s == 0 else m
                syn = 0
                for b in range(8):
                    if bm & (0x80 >> b):
                        syn ^= cols[8 * l + b]
                out[(2 * l + s, m)] = syn
    return out


def min_substitutions(nbytes, first_byte, max_w=4):
    """a least set of nibble substitutions (distinct symbols) whose syndromes cancel, by meeting in the middle over pairs
    of (symbol, mask); None when there is none up to max_w (<= 4)"""
    subs = substitution_syndromes(nbytes, first_byte)
    items = sorted(subs.items())
    by_syn = {}
    for k, s in items:
        by_syn.setdefault(s, []).append(k)
    if 0 in by_syn:
        return [by_syn[0][0]]
    for s, ks in by_syn.items():                                  # two: equal syndromes at two symbols
        for a, b in itertools.combinations(ks, 2):
            if a[0] != b[0]:
                return [a, b]
    if max_w < 3:
        return None
    pairs = {}
    for (a, sa), (b, sb) in itertools.combinations(items, 2):
        if a[0] != b[0]:
            pairs.setdefault(sa ^ sb, []).append((a, b))
    for (k, s) in items:                                          # three: a pair and a third symbol
        for a, b in pairs.get(s, ()):
            if k[0] not in (a[0], b[0]):
                return [a, b, k]
    if max_w < 4:
        return None
    for ps in pairs.values():                                     # four: two pairs on four symbols
        for (a, b), (c, d) in itertools.combinations(ps, 2):
            if len({a[0], b[0], c[0], d[0]}) == 4:
                return [a, b, c, d]
    return None


def min_words(nbytes, first_byte, limit=200):
    """up to `limit` sets of three nibble substitutions on distinct symbols whose syndromes cancel (the least number,
    min_substitutions says)"""
    items = sorted(substitution_syndromes(nbytes, first_byte).items())
    pairs = {}
    for (a, sa), (b, sb) in itertools.combinations(items, 2):
        if a[0] != b[0]:
            pairs.setdefault(sa ^ sb, []).append((a, b))
    out = []
    for k, s in items:
        for a, b in pairs.get(s, ()):
            if k[0] > b[0] > a[0]:
                out.append((a, b, k))
                if len(out) >= limit:
                    return out
    return out


# ---- the corpus ---------------------------------------------------------------------------------------------------------

def t1_bits(synth, L, k):
    """the frame bits of a clean T1 telegram (flagged bit first, 8 idle pairs after it) and its datagram"""
    e = synth.Emitter("T1", 0x12345678 + L, l_field=L, seed=60 + L)
    p = e.payload(k)
    return synth.chips_t1(synth.frame_a(p), 0, 8)[9:].astype(np.uint8), p


def clean_soft(rng, bits, lo=2000, hi=6000):
    return ((2 * bits.astype(np.int64) - 1) * rng.integers(lo, hi, len(bits))).astype(np.int16)


def symbol_chips(i):
    return list(range(1 + 6 * i, 7 + 6 * i))


def corpus(synth, s_max, seed=11):
    """T1 telegrams with wrong chips in 0 .. s_max + 1 symbols per block -- single flips (weak or full swing), a 1-chip and
    a 0-chip of one symbol (often another valid code word), two or three flips in one symbol (weight 0 / 1 / 5 / 6 or an
    invalid weight 3) -- some chips without a value, RSSI drop-outs and truncated lists"""
    rng = np.random.default_rng(seed)
    cases = []
    for L in (9, 0x0E, 0x19, 0x2E, 0x44, 0x7F, 0xB3, 0xFF):
        for k in range(3):
            bits, p = t1_bits(synth, L, k)
            n = rc.tlg_len_a(L)
            P = 1 + 12 * n
            soft = clean_soft(rng, bits)
            strong = bool(rng.integers(0, 4) == 0)
            for off, blk in rc.blocks_a(n):
                syms = np.arange(2 * max(off, 1), 2 * (off + blk))
                for i in rng.choice(syms, min(int(rng.integers(0, s_max + 2)), len(syms)), replace=False):
                    chips = symbol_chips(int(i))
                    kind = int(rng.integers(0, 4))
                    if kind == 0:                                    # one chip
                        pick = [chips[int(rng.integers(0, 6))]]
                    elif kind == 1:                                  # a 1-chip and a 0-chip: often a valid wrong word
                        ones = [j for j in chips if bits[j]]; zeros = [j for j in chips if not bits[j]]
                        pick = [ones[int(rng.integers(0, len(ones)))], zeros[int(rng.integers(0, len(zeros)))]]
                    else:                                            # two or three chips of one kind or mixed
                        pick = list(rng.choice(chips, kind, replace=False))
                    for j in pick:
                        bits[j] ^= 1
                        mag = rng.integers(2000, 6000) if strong else rng.integers(10, 600)
                        soft[j] = (2 * int(bits[j]) - 1) * mag
            for j in rng.choice(np.arange(13, P), int(rng.integers(0, 3)), replace=False):
                soft[j] = NONE
            rssi = np.full(len(bits), 100, np.uint8)
            tail = int(rng.integers(0, 12))
            if tail == 0:
                rssi[int(rng.integers(13, P - 1))] = 2               # an RSSI drop-out: the decode aborts
            elif tail == 1:
                bits, rssi, soft = bits[:P - 5], rssi[:P - 5], soft[:P - 5]      # a truncated list
            cases.append(dict(chain=0, bits=bits, rssi=rssi, soft=soft, sent=p, wire=synth.frame_a(p)))
    return cases


def ambiguous_cases(synth, rng=None):
    """a block where three nibble substitutions cancel in the CRC (the least number there is): the first of the three
    symbols is received as its substitute, and all three are the least confident, with ML and runner-up the two values
    (so they must lie at chip distance 2).  From K = 3 on two patterns pass -- the first symbol's, and the other two's --
    so the block is AMBIGUOUS; below, it is REPAIRED or UNREPAIRABLE"""
    rng = rng or np.random.default_rng(3)
    out = []
    for nbytes, first, block_byte in ((12, 1, 0), (18, 0, 12)):
        words = min_words(nbytes, first)
        for k in range(60):
            bits, p = t1_bits(synth, 0x19, k)
            pkt = [rc.DEC_3OF6[word(bits, 1 + 6 * i, 6)] for i in range(2 * rc.tlg_len_a(0x19))]
            good = []
            for wd in words:
                ok = True
                for (i, m) in wd:
                    a = pkt[2 * block_byte + i]
                    ok &= bin(rc.ENC_3OF6[a] ^ rc.ENC_3OF6[a ^ m]).count("1") == 2
                if ok:
                    good.append(wd)
            if good:
                break
        wd = good[int(rng.integers(0, len(good)))]
        soft = clean_soft(rng, bits, 4000, 4001)
        for t, (i, m) in enumerate(wd):
            sym = 2 * block_byte + i
            a = pkt[sym]
            got = a ^ m if t == 0 else a                              # the first symbol received as its alternative
            ca, cg = rc.ENC_3OF6[a], rc.ENC_3OF6[got]
            other = ca if t == 0 else rc.ENC_3OF6[a ^ m]
            for c, j in enumerate(symbol_chips(sym)):
                bit = cg >> (5 - c) & 1
                bits[j] = bit
                differs = (cg ^ other) >> (5 - c) & 1
                soft[j] = (2 * bit - 1) * (3 if differs else 4000)
        out.append(dict(chain=0, bits=bits, rssi=np.full(len(bits), 100, np.uint8), soft=soft, sent=p,
                        wire=synth.frame_a(p), weight=3))
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
        assert lib.wmb_frame_repair_t1_soft(C.addressof(frames[i]), ptrs[i], e_max, s_max, C.addressof(host[i])) == 0
    dev = (pkg.WmbRepaired * len(cases))()
    fs, rs, ps = C.sizeof(pkg.WmbFrame), C.sizeof(pkg.WmbRepaired), C.sizeof(C.c_void_p)
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        for lo in range(0, len(cases), chunk):
            n = min(chunk, len(cases) - lo)
            assert lib.wmb_frame_repair_t1_soft_device(ctx._ctx, C.addressof(frames) + lo * fs, C.addressof(ptrs) + lo * ps,
                                                       n, e_max, s_max, C.addressof(dev) + lo * rs) == 0, lib.wmb_last_error()
    return (frames, keep, arrs), host, dev


def within_k(c, s_max):
    """the wrong symbols of a corpus telegram lie among its K searched symbols, block by block (and it has some), and the
    L byte is intact"""
    bits = c["bits"]
    L, n = t1_length(bits)
    P = 1 + 12 * n
    if len(bits) < P or n < 12 or (c["rssi"][:P - 1] < rc.CAPTURE_THRESHOLD).any():
        return False
    if L != c["wire"][0]:
        return False
    y, ok = centred(bits, c["soft"], P)
    sent = [x for l in range(n) for x in (c["wire"][l] >> 4, c["wire"][l] & 15)]
    wrong_any = False
    for off, blk in rc.blocks_a(n):
        syms = list(range(2 * max(off, 1), 2 * (off + blk)))
        key = {}
        wrong = set()
        for i in syms:
            first = 1 + 6 * i
            ml, ru, delta = symbol_scores(y[first:first + 6])
            key[i] = (int(all(ok[first:first + 6])), delta, i)
            if ml != sent[i]:
                if ru != sent[i]:
                    return False                                      # the soft values do not point at the sent value
                wrong.add(i)
        wrong_any |= bool(wrong)
        if not wrong <= set(sorted(syms, key=lambda i: key[i])[:s_max]):
            return False
    return wrong_any


# ---- the streaming path -------------------------------------------------------------------------------------------------

def t1_emitters(synth):
    """T1 emitters whose telegrams each lose a symbol to two weak chips (chips 0 and 1 of byte 3's high symbol: another
    code word or one with no filling, UNREPAIRABLE for the erasure rule) or four symbols of one block to a weak chip each
    (TOO_MANY), beside a clean T1 one, the T1 / S1 emitters with flipped chips of tests/test_repair.py and a C1 emitter
    with weak bits (chip 0: the L-field's first chip; byte l of a T1 telegram is chips 12 l .. 12 l + 11)"""
    from test_repair import flipped_emitters
    return [synth.Emitter("T1", 0x44001122, amp=70.0, offset_hz=-5e3, l_field=0x19, period_s=0.17, start_s=0.020, seed=51,
                          weak_flips=(12 * 3, 12 * 3 + 1)),
            synth.Emitter("T1", 0x44003344, amp=70.0, offset_hz=4e3, l_field=0x2E, period_s=0.19, start_s=0.075, seed=52,
                          weak_flips=(12 * 13 + 2, 12 * 15 + 8, 12 * 17 + 3, 12 * 20 + 10)),
            synth.Emitter("T1", 0x44005566, amp=70.0, offset_hz=1e3, l_field=0x2E, period_s=0.23, start_s=0.130, seed=53),
            ] + flipped_emitters(synth)[:2] + sc.weak_emitters(synth)[:1]


def t1_capture(n=8 << 20):
    import importlib
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = t1_emitters(synth)
    cu8, plan = synth.synth_capture(n, emitters=ems, seed=0xB200000B)
    return np.ascontiguousarray(cu8.numpy()), plan, ems


def record_tuple(r):
    import repair_stream_cases as rs
    return rs.record_tuple(r) + (r.soft_t1,)


def stream(pkg, lib, cu8, flags, e_max, batching="1mib", batch_mib=1, quality=False, burst_level=None, **ctx_kw):
    """the streaming run: (records with soft_t1 last, lines, line info, quality, bursts, stats)"""
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


def restated_stream(pkg, lib, cu8, flags, e_max, settings, **ctx_kw):
    """{(k_max, s_max): sorted record tuples} from manual framing with soft values: repair_stream_cases.restated with
    wmb_frame_repair_soft on the C1 lines with CRC errors (k_max) and wmb_frame_repair_t1_soft on every other frame (s_max);
    soft_t1 = 1 where the T1 rule ran (a T1 line with CRC errors, len >= 12, soft values, the erasure rule TOO_MANY or
    UNREPAIRABLE)"""
    import repair_stream_cases as rs
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    with pkg.WmbusB200(flags, lib=lib, manual_frames=1, soft_bits=True, **ctx_kw) as ctx:
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
        for k_max, s_max in settings:
            recs = []
            for f, d, soft in accepted:
                r, r0 = pkg.WmbRepaired(), pkg.WmbRepaired()
                sp = None if soft is None else soft.ctypes.data
                c1_line = d.status == 1 and d.mode == b"C1" and not d.crc_ok
                if c1_line and k_max:
                    assert lib.wmb_frame_repair_soft(C.addressof(f), sp, e_max, k_max, C.addressof(r)) == 0
                else:
                    assert lib.wmb_frame_repair_t1_soft(C.addressof(f), sp, e_max, s_max, C.addressof(r)) == 0
                if r.outcome in (rc.NONE, rc.TRUNCATED):
                    continue
                assert lib.wmb_frame_repair(C.addressof(f), e_max, C.addressof(r0)) == 0
                w = np.ctypeslib.as_array(f.bits, (f.nbits,))
                soft_t1 = int(bool(s_max) and soft is not None and d.status == 1 and d.mode == b"T1" and not d.crc_ok
                              and r0.outcome in (rc.TOO_MANY, rc.UNREPAIRABLE) and t1_length(w & 1)[1] >= 12)
                if d.status == 1 and d.mode == b"C1":
                    end = d.end_sample
                else:
                    end = f.sync_sample + int(w[rs.telegram_bits(f) - 1] >> 9)
                rec = pkg.WmbRepairRecord()
                rec.sync_sample = f.sync_sample; rec.end_sample = end; rec.chain = f.chain; rec.algo = f.algo
                rec.repair = r
                rec.soft_t1 = soft_t1
                recs.append(record_tuple(rec))
            out[(k_max, s_max)] = sorted(recs, key=rs.key)
    return out
