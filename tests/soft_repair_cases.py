"""Soft-decision repair of C1 telegrams (wmbus_b200_framer.h): the restatement of the soft value per bit on the CPU
oracle's stages, of the C1 soft repair rule in plain Python, and the helpers shared by the CPU-simulation tests
(test_soft_repair.py) and the GPU tests (test_soft_repair_gpu.py).

Soft value of bit event e of a T1/C1 stream at decimated sample m: chip centre c = m - D_T2 (t2a) or
c = m - D_RL - 8 (n - 1 - i) (rla, the i-th of the n events at sample m); v = floor(sum of rint(fir * 2^24) over
[c - 2, c + 3) / 2^12), clamped to +-32767; -32768 when the window starts before the first sample or n - 1 - i > 63."""
import ctypes as C
import importlib

import numpy as np

import orc
import receiver_oracle as ro
import repair_cases as rc

SCALE = float(1 << 24)
NONE = -32768
D_T2, D_RL = 2, 7              # include/wmbus_b200_framer.h WMB_SOFT_D_T2 / WMB_SOFT_D_RL (DESIGN.md section 8)
D_RANGE = range(2, 16)         # D >= 2: the window ends at the event's own sample, which the event's batch holds
K_MAX = 6
MODE_A, MODE_B = 0x54C, 0x543


# ---- the soft value per bit ------------------------------------------------------------------------------------------

def soft_values(fir, ev, algo, d_t2=D_T2, d_rl=D_RL):
    """int16 soft value of every event of one T1/C1 stream (events since the start of fir)"""
    m = ev["m"].astype(np.int64)
    n = len(m)
    after = np.zeros(n, np.int64)                  # n - 1 - i: later events at the same sample
    if algo == 0 and n:
        starts = np.r_[True, m[1:] != m[:-1]]
        run_id = np.cumsum(starts) - 1
        run_end = np.r_[np.nonzero(starts)[0][1:], n]          # one past each run's last event
        after = run_end[run_id] - 1 - np.arange(n)
        c = m - d_rl - 8 * after
    else:
        c = m - d_t2
    x = np.rint(np.asarray(fir, np.float64) * SCALE).astype(np.int64)
    cs = np.r_[0, np.cumsum(x)]
    lo, hi = c - 2, c + 3
    ok = (lo >= 0) & (after <= 63) & (hi <= len(x))         # (the last: only for D < 2, which d_scores tries)
    s = np.zeros(n, np.int64)
    s[ok] = cs[hi[ok]] - cs[lo[ok]]
    v = np.clip(np.floor_divide(s, 1 << 12), -32767, 32767)
    v[~ok] = NONE
    return v.astype(np.int16)


def oracle_streams(cu8, flags, lock=(2, 2), errors=(0, 0)):
    """{algo: (events, soft values)} of the T1/C1 chain"""
    o = orc.opts_from_flags(flags)
    st = orc.stages(np.ascontiguousarray(cu8, np.uint8), o, 0)
    out = {}
    for algo, on in ((0, o.rla_enabled), (1, o.t2_enabled)):
        if on:
            ev = ro.stream_events(st, 0, algo, lock[0], errors[0])
            out[algo] = (ev, soft_values(st["fir"], ev, algo))
    return out


def d_scores(cu8, flags="", lock=(2, 2)):
    """{algo: [mean of (2 bit - 1) v over the bits [17, P) of every CRC-clean C1 line, for D = 0 .. 15]}"""
    o = orc.opts_from_flags(flags)
    st = orc.stages(np.ascontiguousarray(cu8, np.uint8), o, 0)
    L = orc.lib()
    buf = C.create_string_buffer(4096)
    got = C.c_int(0)
    out = {}
    for algo in (0, 1):
        ev = ro.stream_events(st, 0, algo, lock[0], 0)
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
            used = L.orc_frame_t1c1(bits[c:end], rssi[c:end], end - c, b"", buf, len(buf), C.byref(got))
            if got.value and buf.value.startswith(b"C1;1;"):
                sel.append(np.arange(c + 17, c + used))
            busy = c + used
        idx = np.concatenate(sel)
        sign = 2 * bits[idx].astype(np.int64) - 1
        scores = []
        for d in range(16):
            v = soft_values(st["fir"], ev, algo, d, d)[idx].astype(np.int64)
            ok = v != NONE
            scores.append(float((sign[ok] * v[ok]).mean()))
        out[algo] = scores
    return out


# ---- the C1 soft repair rule -------------------------------------------------------------------------------------------

def blocks_b(n):
    """frame B: 128-byte blocks from byte 0, the last one shorter"""
    return [(off, min(128, n - off)) for off in range(0, n, 128)]


def c1_layout(bits):
    """(frame B, len) of a C1 frame's bit list (flagged bit first)"""
    mode = int("".join(str(int(b)) for b in bits[1:13]), 2)
    L = int("".join(str(int(b)) for b in bits[17:25]), 2)
    fb = mode == MODE_B
    return fb, (1 + L if fb else rc.tlg_len_a(L))


def reliabilities(bits, soft, P):
    """r_j for the bits [17, P); a sentinel bit ranks lowest: (0, 0) before every (1, r)"""
    b = np.asarray(bits[17:P], np.int64)
    v = np.asarray(soft[17:P], np.int64)
    ok = v != NONE
    n1 = int((ok & (b == 1)).sum()); n0 = int((ok & (b == 0)).sum())
    S1 = int(v[ok & (b == 1)].sum()); S0 = int(v[ok & (b == 0)].sum())
    sign = 2 * b - 1
    if n0 * n1 == 0:
        r = sign * v
    else:
        r = sign * (v * 2 * n0 * n1 - (S1 * n0 + S0 * n1))
    return [(1, int(r[i])) if ok[i] else (0, 0) for i in range(len(b))]


def crc_ok(q):
    return len(q) >= 2 and rc.crc16(bytes(q[:-2])) == (q[-2] << 8 | q[-1])


def repair_soft_c1(bits, rssi, soft, k_max):
    """the rule for a C1 frame whose decode is a line with crc_ok = 0 (the caller checks that): a dict like
    repair_cases.repair's"""
    fb, n = c1_layout(bits)
    P = 17 + 8 * n
    out = dict(outcome=rc.UNREPAIRABLE, erasures=0, blocks=0, had_line=1)
    if n < 12:
        return out
    pkt = bytearray(int("".join(str(int(b)) for b in bits[17 + 8 * l:25 + 8 * l]), 2) for l in range(n))
    key = reliabilities(bits, soft, P)
    flips = blocks = 0
    for off, blk in (blocks_b(n) if fb else rc.blocks_a(n)):
        if crc_ok(pkt[off:off + blk]):
            continue
        cand = [j for j in range(17 + 8 * max(off, 1), 17 + 8 * (off + blk))]
        cand.sort(key=lambda j: (key[j - 17], j))
        sel = cand[:min(k_max, len(cand))]
        passing = []
        for x in range(1, 1 << len(sel)):
            q = bytearray(pkt[off:off + blk])
            for t, j in enumerate(sel):
                if x >> t & 1:
                    q[(j - 17) // 8 - off] ^= 0x80 >> ((j - 17) % 8)
            if crc_ok(q):
                passing.append(x)
        if len(passing) != 1:
            out["outcome"] = rc.AMBIGUOUS if passing else rc.UNREPAIRABLE
            return out
        for t, j in enumerate(sel):
            if passing[0] >> t & 1:
                pkt[(j - 17) // 8] ^= 0x80 >> ((j - 17) % 8)
                flips += 1
        blocks += 1
    if fb:
        nblk = len(blocks_b(n))
        data = bytearray()
        for off, blk in blocks_b(n):
            data += pkt[off:off + blk - 2]
        data[0] = (pkt[0] - 2 * nblk) & 0xFF
    else:
        data = bytearray()
        for off, blk in rc.blocks_a(n):
            data += pkt[off:off + blk - 2]
    out.update(outcome=rc.REPAIRED, erasures=flips, blocks=blocks, mode="C1", crc_ok=1, ok_3of6=1,
               packet_rssi=int(rssi[1]), current_rssi=int(rssi[P - 1]), serial=int.from_bytes(bytes(pkt[4:8]), "little"),
               datagram=bytes(data), consumed=P)
    return out


def load_pkg():
    return importlib.import_module("rtl-wmbus_b200")


# ---- polled soft values -------------------------------------------------------------------------------------------------

def polled_soft(pkg, lib, cu8, flags, batching="1mib", batch_mib=1):
    """{(chain, algo, ordinal): soft values or None} of every frame a manual_frames context polls (last delivery wins)"""
    import repair_stream_cases as rsc
    out = {}
    with pkg.WmbusB200(flags, lib=lib, manual_frames=1, soft_bits=True, max_batch_mib=batch_mib) as ctx:
        def take(flush):
            arr, k = ctx.poll(flush=flush)
            for i in range(k):
                out[(arr[i].chain, arr[i].algo, arr[i].ordinal)] = ctx.frame_soft(arr[i])
        for lo, hi in rsc.pushes(len(cu8), batching):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
            take(False)
        take(True)
    return out


def check_polled_soft(got, want):
    """every T1/C1 frame's values equal the restatement's at its ordinals; S1 frames have none"""
    n = 0
    for (chain, algo, ordinal), v in got.items():
        if chain != 0:
            assert v is None
            continue
        ref = want[algo][1][ordinal:ordinal + len(v)]
        assert np.array_equal(v, ref), (algo, ordinal, np.nonzero(v != ref)[0][:5])
        n += len(v)
    return n


# ---- minimum weight of the shortened CRC codes --------------------------------------------------------------------------

def syndrome_columns(nbits):
    """the CRC syndrome of each single flipped bit of a block of nbits (data, then the 16 CRC bits), MSB first"""
    nd = nbits // 8 - 2
    cols = []
    for q in range(nbits // 8):
        for b in range(8):
            mask = 0x80 >> b
            if q >= nd:
                cols.append(mask << 8 if q == nd else mask)
                continue
            crc = mask << 8
            for _ in range(8 * (nd - q)):
                crc = ((crc << 1) ^ 0x3D65) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
            cols.append(crc)
    return cols


def min_weight_word(nbits, max_w):
    """a lowest-weight code word (bit positions) of the shortened code up to weight max_w (<= 6), by meeting in the
    middle over pairs and triples; None when there is none up to max_w.  The triple loop can meet a weight-6 word before
    a weight-5 one; that cannot make the result wrong, because 0x13D65 is divisible by x + 1 and every code word has even
    weight: there is no weight 5 (nor 3)."""
    import itertools
    cols = syndrome_columns(nbits)
    n = len(cols)
    seen = {}
    for i, c in enumerate(cols):
        if c in seen:
            return (seen[c], i)
        seen[c] = i
    pairs = {}
    for i, j in itertools.combinations(range(n), 2):
        pairs.setdefault(cols[i] ^ cols[j], []).append((i, j))
    for s, v in pairs.items():                                   # weight 3: a pair and a third column
        if s in seen and seen[s] not in v[0]:
            return v[0] + (seen[s],)
    if max_w < 4:
        return None
    for v in pairs.values():                                     # weight 4: two disjoint pairs
        if len(v) > 1:
            return v[0] + v[1]
    if max_w < 5:
        return None
    triples = {}
    for t in itertools.combinations(range(n), 3):
        s = cols[t[0]] ^ cols[t[1]] ^ cols[t[2]]
        for p in pairs.get(s, ()):
            if not set(p) & set(t):
                return t + p
        if max_w >= 6:
            for u in triples.get(s, ()):
                if not set(u) & set(t):
                    return u + t
            triples.setdefault(s, []).append(t)
    return None


# ---- the streaming path -------------------------------------------------------------------------------------------------

def weak_emitters(synth):
    """C1A and C1B emitters whose telegrams each send two data chips on the wrong tone at a fifth of the deviation (chip 0:
    the first of the C1 mode word; C1 byte l is chips 16 + 8 l .. 23 + 8 l), beside clean C1 ones and the T1 / S1 emitters
    with flipped chips of tests/test_repair.py"""
    from test_repair import flipped_emitters
    return [synth.Emitter("C1A", 0x20338739, amp=70.0, offset_hz=-5e3, l_field=0x19, period_s=0.17, start_s=0.020, seed=41,
                          weak_flips=(16 + 8 * 3 + 2, 16 + 8 * 20 + 5)),
            synth.Emitter("C1B", 0x20210116, amp=70.0, offset_hz=4e3, l_field=0x2E, period_s=0.19, start_s=0.075, seed=42,
                          weak_flips=(16 + 8 * 7 + 4,)),
            synth.Emitter("C1A", 0x31415926, amp=70.0, offset_hz=1e3, l_field=0x2E, period_s=0.23, start_s=0.130, seed=43),
            ] + flipped_emitters(synth)[:2]


def weak_capture(n=8 << 20):
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = weak_emitters(synth)
    cu8, plan = synth.synth_capture(n, emitters=ems, seed=0xB2000009)
    return np.ascontiguousarray(cu8.numpy()), plan, ems


def restated_stream(pkg, lib, cu8, flags, e_max, k_maxes, **ctx_kw):
    """{k_max: sorted record tuples} from manual framing with soft values: repair_stream_cases.restated with
    wmb_frame_repair_soft in place of wmb_frame_repair"""
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
        for k_max in k_maxes:
            recs = []
            for f, d, soft in accepted:
                r = pkg.WmbRepaired()
                sp = None if soft is None else soft.ctypes.data
                assert lib.wmb_frame_repair_soft(C.addressof(f), sp, e_max, k_max, C.addressof(r)) == 0
                if r.outcome in (rc.NONE, rc.TRUNCATED):
                    continue
                if d.status == 1 and d.mode == b"C1":
                    end = d.end_sample                  # a C1 line: its last bit, bit P - 1
                else:
                    P = rs.telegram_bits(f)
                    end = f.sync_sample + int(np.ctypeslib.as_array(f.bits, (f.nbits,))[P - 1] >> 9)
                rec = pkg.WmbRepairRecord()
                rec.sync_sample = f.sync_sample; rec.end_sample = end; rec.chain = f.chain; rec.algo = f.algo
                rec.repair = r
                recs.append(rs.record_tuple(rec))
            out[k_max] = sorted(recs, key=rs.key)
    return out
