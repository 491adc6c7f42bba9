"""Erasure repair on the streaming path (wmb_set_repair, wmb_take_repairs): the records of a context that frames for
itself, and their restatement from manual framing -- wmb_poll(flush) frames, the stream-order rule of book_frames
restated in Python over the host twin's verdicts (wmb_frame_decode), wmb_frame_repair on the accepted candidates,
NONE and TRUNCATED dropped, the rest sorted by (end_sample, chain * 2 + (algo == t2a), sync_sample)."""
import ctypes as C
import importlib

import numpy as np

import repair_cases as rc

MIB = 1 << 20


def record_tuple(r):
    """one record, field by field (a WmbRepairRecord, or the restatement's tuple source)"""
    p = r.repair
    t = (r.sync_sample, r.end_sample, r.chain, r.algo, p.outcome, p.erasures, p.blocks, p.had_line)
    if p.outcome != rc.REPAIRED:
        return t
    d = p.line
    return t + (d.status, d.consumed, d.end_sample, d.mode, d.crc_ok, d.ok_3of6, d.packet_rssi, d.current_rssi,
                d.serial, bytes(d.datagram[:d.len]))


def key(t):
    return t[1], t[2] * 2 + (1 if t[3] == 1 else 0), t[0]


def telegram_bits(f):
    """P of a frame (from its L-field), or None when the list does not hold the L-field"""
    w = np.ctypeslib.as_array(f.bits, (f.nbits,)) & 1
    if f.chain == 0:
        if f.nbits < 13:
            return None
        a = int("".join(str(int(x)) for x in w[1:7]), 2)
        b = int("".join(str(int(x)) for x in w[7:13]), 2)
        if a not in rc.DEC_3OF6 or b not in rc.DEC_3OF6:
            return None
        return 1 + 12 * rc.tlg_len_a(rc.DEC_3OF6[a] << 4 | rc.DEC_3OF6[b])
    if f.nbits < 17:
        return None
    return 1 + 16 * rc.tlg_len_a(rc.word2(w, 2, 8))


def restated(pkg, lib, cu8, flags, e_maxes, **ctx_kw):
    """{e_max: sorted record tuples} from manual framing of cu8 (one push, poll with flush)"""
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    with pkg.WmbusB200(flags, lib=lib, manual_frames=1, **ctx_kw) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True, cap=1 << 20)
        frames = sorted((arr[i] for i in range(k)), key=lambda f: (f.chain, f.algo, f.ordinal))
        busy = {}
        accepted = []
        for f in frames:
            s = (f.chain, f.algo)
            if f.ordinal <= busy.get(s, -1):
                continue
            d = pkg.WmbDecoded()
            lib.wmb_frame_decode(C.addressof(f), C.addressof(d))
            assert d.status != 2 or f.truncated, "a final frame shorter than its header demands"
            busy[s] = f.ordinal + d.consumed - 1
            accepted.append((f, d))
        out = {}
        for e_max in e_maxes:
            recs = []
            for f, d in accepted:
                r = pkg.WmbRepaired()
                assert lib.wmb_frame_repair(C.addressof(f), e_max, C.addressof(r)) == 0
                if r.outcome in (rc.NONE, rc.TRUNCATED):
                    continue
                if d.status == 1 and d.mode == b"C1":
                    end = d.end_sample                  # a C1 line (never repaired): its last bit
                else:
                    P = telegram_bits(f)
                    end = f.sync_sample + int(np.ctypeslib.as_array(f.bits, (f.nbits,))[P - 1] >> 9)
                rec = pkg.WmbRepairRecord()
                rec.sync_sample = f.sync_sample; rec.end_sample = end; rec.chain = f.chain; rec.algo = f.algo
                rec.repair = r
                recs.append(record_tuple(rec))
            out[e_max] = sorted(recs, key=key)
    return out


def pushes(n, batching):
    """byte ranges of the pushes: "1mib" / "one" (one push of everything) / "uneven" (ragged sizes)"""
    if batching == "uneven":
        cuts, at, k = [], 0, 0
        sizes = (300_001, 1_500_000, 77_777, 2_900_000, 640_000)
        while at < n:
            nxt = min(n, at + sizes[k % len(sizes)])
            cuts.append((at, nxt))
            at, k = nxt, k + 1
        return cuts
    step = MIB if batching == "1mib" else n
    return [(lo, min(n, lo + step)) for lo in range(0, n, step)]


def stream(pkg, lib, cu8, flags, e_max, batching="1mib", batch_mib=1, quality=False, burst_level=None, device=False,
           **ctx_kw):
    """the streaming run: (records, lines, line info, quality, bursts, stats)"""
    with pkg.WmbusB200(flags, lib=lib, repair=e_max, quality=quality, burst_level=burst_level,
                       max_batch_mib=batch_mib, **ctx_kw) as ctx:
        recs = []
        for lo, hi in pushes(len(cu8), batching):
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


def flipped_capture(n=8 << 20):
    """the flipped-emitter capture of tests/test_repair.py and its plan"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    from test_repair import flipped_emitters
    ems = flipped_emitters(synth)
    cu8, plan = synth.synth_capture(n, emitters=ems, seed=0xB2000007)
    return np.ascontiguousarray(cu8.numpy()), plan, ems
