"""Erasure repair of T1 / S1 candidates (wmbus_b200_framer.h): the host twin wmb_frame_repair(), the device repair K4R
(wmb_frame_repair_device, here on the CPU build) and the plain-Python restatement (tests/repair_cases.py) agree frame by
frame, and planted telegrams with a few flipped chips per block come back with the datagram that was sent."""
import ctypes as C
import importlib

import numpy as np
import pytest

import repair_cases as rc

E_MAX = (1, 2, 3)
CHUNK = 1000                        # frames per device call: their datagrams fit one slot's pool


Repaired = importlib.import_module("rtl-wmbus_b200").WmbRepaired


def make_frames(pkg, cases):
    """wmb_frame per case; bit i lies 3 i samples after sync_sample"""
    frames = (pkg.WmbFrame * len(cases))()
    keep = []
    for i, c in enumerate(cases):
        k = len(c["bits"])
        words = (np.arange(k, dtype=np.uint32) * 3 << 9) | (c["rssi"].astype(np.uint32) << 1) | c["bits"].astype(np.uint32)
        words = np.ascontiguousarray(words, np.uint32)
        keep.append(words)
        f = frames[i]
        f.sync_sample = 1000 + 7 * i; f.ordinal = i; f.chain = c["chain"]; f.algo = i & 1; f.nbits = k
        f.bits = words.ctypes.data_as(C.POINTER(C.c_uint32))
    return frames, keep


def host_repair(lib, frames, e_max):
    out = (Repaired * len(frames))()
    for i in range(len(frames)):
        assert lib.wmb_frame_repair(C.addressof(frames[i]), e_max, C.addressof(out[i])) == 0
    return out


def device_repair(lib, pkg, frames, e_max):
    out = (Repaired * len(frames))()
    size = C.sizeof(pkg.WmbFrame)
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        for lo in range(0, len(frames), CHUNK):
            n = min(CHUNK, len(frames) - lo)
            rc_ = lib.wmb_frame_repair_device(ctx._ctx, C.addressof(frames) + lo * size, n, e_max,
                                              C.addressof(out) + lo * C.sizeof(Repaired))
            assert rc_ == 0, lib.wmb_last_error()
    return out


def as_tuple(r):
    t = (r.outcome, r.erasures, r.blocks, r.had_line)
    if r.outcome != rc.REPAIRED:
        return t
    d = r.line
    return t + (d.status, d.mode.decode(), d.crc_ok, d.ok_3of6, d.packet_rssi, d.current_rssi, d.serial,
                bytes(d.datagram[:d.len]), d.consumed, d.end_sample)


def restated_tuple(r):
    t = (r["outcome"], r["erasures"], r["blocks"], r["had_line"])
    if r["outcome"] != rc.REPAIRED:
        return t
    return t + (1, r["mode"], r["crc_ok"], r["ok_3of6"], r["packet_rssi"], r["current_rssi"], r["serial"],
                r["datagram"], r["consumed"], r["end_sample"])


# ---- candidates ------------------------------------------------------------------------------------------------------

SYNC_LEN = {"T1": 10, "S1": 18}


def telegram_chips(synth, mode, L, k):
    """chips from the access-code bit (the flagged one) to 8 idle pairs after the telegram, and the logical payload"""
    e = synth.Emitter(mode, 0x12345678 + L, l_field=L, seed=40 + L)
    p = e.payload(k)
    wire = synth.frame_a(p)
    chips = synth.chips_t1(wire, 0, 8) if mode == "T1" else synth.chips_s1(wire, 0, 8)
    return chips[SYNC_LEN[mode] - 1:].astype(np.uint8), p


def flip_data_chips(rng, mode, L, chips, per_block):
    """a copy of chips with one chip flipped in each of `per_block[j]` distinct T1 symbols / S1 pairs of block j (never
    in the L-field)"""
    n = rc.tlg_len_a(L)
    chips = chips.copy()
    for (off, blk), want in zip(rc.blocks_a(n), per_block):
        bytes_ = [l for l in range(off, off + blk) if l >= 1]
        if mode == "T1":
            units = [(l, s) for l in bytes_ for s in (0, 1)]
        else:
            units = [(l, s) for l in bytes_ for s in range(8)]
        for u in rng.choice(len(units), min(want, len(units)), replace=False):
            l, s = units[u]
            if mode == "T1":
                chips[1 + 12 * l + 6 * s + int(rng.integers(0, 6))] ^= 1
            else:
                chips[1 + 16 * l + 2 * s + int(rng.integers(0, 2))] ^= 1
    return chips


def planted_cases(synth, n_per, seed=7):
    """T1 and S1 telegrams of many lengths with 0..4 single-chip flips per block (`sent`: the payload; `planted`: the
    payload and the most erasures in a block), plus variants that cannot be repaired: two or three flips in one T1 symbol, both
    chips of an S1 pair, RSSI drop-outs, truncated lists."""
    rng = np.random.default_rng(seed)
    cases = []
    for mode in ("T1", "S1"):
        for L in (9, 0x0E, 0x19, 0x2E, 0x66, 0xFF):
            n = rc.tlg_len_a(L)
            nblk = len(rc.blocks_a(n))
            for k in range(n_per):
                chips, p = telegram_chips(synth, mode, L, k)
                per_block = [int(x) for x in rng.choice([0, 1, 1, 2, 2, 3, 4], nblk)]
                if sum(per_block) == 0:
                    per_block[int(rng.integers(0, nblk))] = 1
                bits = flip_data_chips(rng, mode, L, chips, per_block)
                rssi = rng.integers(20, 200, len(bits)).astype(np.uint8)
                variant = k % 8
                planted = dict(payload=p, worst=max(per_block))
                if variant == 5 and mode == "T1":           # a second / third chip in one symbol: weight 1, 3 or 5
                    l = int(rng.integers(1, n))
                    for c in rng.choice(6, int(rng.integers(2, 4)), replace=False):
                        bits[1 + 12 * l + int(c)] ^= 1
                    planted = None
                elif variant == 5:                          # both chips of a pair: a wrong bit, no erasure
                    l = int(rng.integers(1, n))
                    b0 = 1 + 16 * l + 2 * int(rng.integers(0, 8))
                    bits[b0:b0 + 2] ^= 1
                    planted = None
                elif variant == 6:                          # an RSSI drop-out somewhere in the telegram
                    rssi[int(rng.integers(1, len(bits) - 16))] = int(rng.integers(0, 5))
                    planted = None
                elif variant == 7:                          # the list ends before the telegram does
                    cut = int(rng.integers(1, len(bits) - 16))
                    bits, rssi = bits[:cut], rssi[:cut]
                    planted = None
                cases.append(dict(chain=0 if mode == "T1" else 1, bits=bits, rssi=rssi, planted=planted, sent=p))
    return cases


def random_cases(n, seed=19):
    """random bit lists; every other S1 one is valid Manchester up to one flipped chip after the L-field byte"""
    rng = np.random.default_rng(seed)
    cases = []
    for trial in range(n):
        chain = trial & 1
        m = int(rng.integers(1, 600))
        bits = rng.integers(0, 2, m).astype(np.uint8)
        if chain == 1 and trial % 4 == 1:
            v = rng.integers(0, 2, (m - 1) // 2).astype(np.uint8)
            bits[1:1 + 2 * len(v):2] = 1 - v
            bits[2:2 + 2 * len(v):2] = v
            j = 2 * int(rng.integers(9, max(10, m // 2))) - 1     # one chip flipped: a violation after the L-field
            if j < m:
                bits[j] ^= 1
        rssi = rng.integers(3, 60, m).astype(np.uint8)
        cases.append(dict(chain=chain, bits=bits, rssi=rssi, planted=None))
    return cases


def c1_cases(synth, n, seed=23):
    """C1 telegrams with flipped chips: lines whose CRCs fail, never repaired (NRZ has no erasures)"""
    rng = np.random.default_rng(seed)
    cases = []
    for k in range(n):
        e = synth.Emitter("C1A", 0x00112233, l_field=0x19, seed=3)
        chips = synth.chips_c1(synth.frame_a(e.payload(k)), False, 0, 8)[len(synth.SYNC_T1C1) - 1:].astype(np.uint8)
        chips[int(rng.integers(40, len(chips) - 20))] ^= 1
        cases.append(dict(chain=0, bits=chips, rssi=rng.integers(20, 200, len(chips)).astype(np.uint8), planted=None))
    return cases


def ambiguous_cases(synth, n=8, seed=29):
    """single-block T1 telegrams (L = 9) with three erased data symbols that two fillings repair.  The CRC is affine,
    so flipping nibble bits whose syndromes cancel leaves the block passing; such a flip pattern d1, d2, d3 is found
    by search, nibbles t_i are chosen so that the code words of t_i and t_i ^ d_i differ in two chips, and the
    received word is the weight-2 word between them: one chip flipped from what was sent."""
    rng = np.random.default_rng(seed)
    zero = rc.crc16(bytes(10))
    nib_syn = []                                     # syndrome of XOR-ing value d into data nibble q (bytes 1..9)
    for q in range(18):
        row = []
        for d in range(16):
            x = bytearray(10)
            x[1 + q // 2] = d << (4 if q % 2 == 0 else 0)
            row.append(rc.crc16(bytes(x)) ^ zero)
        nib_syn.append(np.array(row, np.int64))
    pair = {}                                        # d -> t with ENC[t], ENC[t ^ d] two chips apart
    for d in range(1, 16):
        for t in range(16):
            if bin(rc.ENC_3OF6[t] ^ rc.ENC_3OF6[t ^ d]).count("1") == 2:
                pair[d] = t
                break
    cases = []
    for q1 in range(18):
        for q2 in range(q1 + 1, 18):
            for q3 in range(q2 + 1, 18):
                syn = nib_syn[q1][:, None, None] ^ nib_syn[q2][None, :, None] ^ nib_syn[q3][None, None, :]
                hits = [h for h in zip(*np.nonzero(syn == 0)) if all(int(d) in pair for d in h)]
                if not hits or len(cases) >= n:
                    continue
                ds = [int(d) for d in hits[0]]
                p = bytearray([9]) + bytearray(rng.integers(0, 256, 9, dtype=np.uint8).tobytes())
                for q, d in zip((q1, q2, q3), ds):
                    sh = 4 if q % 2 == 0 else 0
                    p[1 + q // 2] = (p[1 + q // 2] & ~(15 << sh) & 0xFF) | pair[d] << sh
                chips = synth.chips_t1(synth.frame_a(bytes(p)), 0, 8)[len(synth.SYNC_T1C1) - 1:].astype(np.uint8)
                for q, d in zip((q1, q2, q3), ds):
                    t = pair[d]
                    w = rc.ENC_3OF6[t] & rc.ENC_3OF6[t ^ d]
                    first = 1 + 12 * (1 + q // 2) + (0 if q % 2 == 0 else 6)
                    chips[first:first + 6] = [(w >> (5 - k)) & 1 for k in range(6)]
                cases.append(dict(chain=0, bits=chips, rssi=rng.integers(20, 200, len(chips)).astype(np.uint8),
                                  planted=None))
    assert len(cases) == n
    return cases


def all_cases(synth):
    return planted_cases(synth, 450) + random_cases(4600) + c1_cases(synth, 40) + ambiguous_cases(synth)


def restated(orc_mod, cases, frames, e_max):
    return [restated_tuple(rc.repair(orc_mod, c["chain"], c["bits"], c["rssi"], np.arange(len(c["bits"])) * 3,
                                     frames[i].sync_sample, e_max))
            for i, c in enumerate(cases)]


@pytest.fixture(scope="module")
def cases():
    return all_cases(importlib.import_module("rtl-wmbus_b200.synth"))


def check_twins(lib, pkg, orc_mod, cases, device):
    """host twin == restatement (CPU only, it is the slow part) and device == host twin, at every e_max"""
    frames, _keep = make_frames(pkg, cases)
    seen = {}
    for e_max in E_MAX:
        host = [as_tuple(r) for r in host_repair(lib, frames, e_max)]
        if orc_mod is not None:
            want = restated(orc_mod, cases, frames, e_max)
            bad = [i for i in range(len(cases)) if host[i] != want[i]]
            assert not bad, (e_max, len(bad), bad[0], host[bad[0]][:4], want[bad[0]][:4])
        if device:
            dev = [as_tuple(r) for r in device_repair(lib, pkg, frames, e_max)]
            bad = [i for i in range(len(cases)) if dev[i] != host[i]]
            assert not bad, (e_max, len(bad), bad[0], dev[bad[0]][:4], host[bad[0]][:4])
        for t in host:
            seen[(e_max, t[0])] = seen.get((e_max, t[0]), 0) + 1
    return seen


def test_host_device_and_restatement_agree(hostsim_lib, pkg, orc_mod, cases):
    assert len(cases) >= 10000
    seen = check_twins(hostsim_lib, pkg, orc_mod, cases, device=True)
    for e_max in E_MAX:                               # every outcome occurs (two fillings passing: at 3 erasures)
        for o in range(6):
            assert seen.get((e_max, o), 0) > 0 or (o == rc.AMBIGUOUS and e_max < 3), (e_max, rc.OUTCOMES[o], seen)


def test_planted_telegrams_come_back_as_sent(hostsim_lib, pkg, cases):
    frames, _keep = make_frames(pkg, cases)
    for e_max in E_MAX:
        out = host_repair(hostsim_lib, frames, e_max)
        n_rep = 0
        for i, c in enumerate(cases):
            r = out[i]
            if r.outcome == rc.REPAIRED:              # no repaired datagram differs from the one sent
                assert bytes(r.line.datagram[:r.line.len]) == c.get("sent"), i
                n_rep += 1
            if c["planted"] is not None and c["planted"]["worst"] <= e_max:
                assert r.outcome == rc.REPAIRED, (e_max, i, rc.OUTCOMES[r.outcome])
            if c["planted"] is not None and c["planted"]["worst"] > e_max:
                assert r.outcome == rc.TOO_MANY, (e_max, i, rc.OUTCOMES[r.outcome])
        assert n_rep > 100, (e_max, n_rep)


def test_repaired_line_formats_as_a_good_line(hostsim_lib, pkg, cases):
    """the repaired line prints with CRC_OK = 1 and 3OUTOF6OK = 1, datagram as sent"""
    planted = [c for c in cases if c["planted"] is not None and c["planted"]["worst"] <= 3][:50]
    frames, _keep = make_frames(pkg, planted)
    with pkg.WmbusB200("-v", lib=hostsim_lib) as ctx:
        out = ctx.repair_frames(frames, len(planted), e_max=3, device=False)
        for i, c in enumerate(planted):
            assert out[i].outcome == rc.REPAIRED
            f = ctx.repaired_line(out[i], b"rla;").split(";")
            p = c["planted"]["payload"]
            assert f[:5] == ["rla", "T1" if c["chain"] == 0 else "S1", "1", "1", "TS"], f
            assert f[7] == p[4:8][::-1].hex().upper() and f[8] == "0x" + p.hex(), f


def test_e_max_range(hostsim_lib, pkg, cases):
    lib = hostsim_lib
    frames, _keep = make_frames(pkg, cases[:8])
    r = Repaired()
    assert lib.wmb_frame_repair(C.addressof(frames[0]), 4, C.addressof(r)) == -1          # WMB_E_INVAL
    assert lib.wmb_frame_repair(C.addressof(frames[0]), 0, C.addressof(r)) == 0 and r.outcome == rc.NONE
    out = (Repaired * 8)()
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_frame_repair_device(ctx._ctx, C.addressof(frames), 8, 4, C.addressof(out)) == -1
        assert lib.wmb_frame_repair_device(ctx._ctx, C.addressof(frames), 8, 0, C.addressof(out)) == 0
        assert all(o.outcome == rc.NONE for o in out)


# ---- from IQ samples: a capture decoded with manual framing, its candidates repaired -----------------------------------

def flipped_emitters(synth):
    """a T1 and an S1 emitter that lose one chip in block 0 and one in block 1 of every telegram (chip 0: the L-field's
    first chip; T1 byte l is chips 12 l .. 12 l + 11, S1 byte l chips 16 l .. 16 l + 15), beside clean T1 and S1 ones"""
    return [synth.Emitter("T1", 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x29, period_s=0.21, start_s=0.004, seed=31,
                          data_flips=(12 * 3 + 2, 12 * 14 + 8)),
            synth.Emitter("S1", 0x19131290, amp=80.0, offset_hz=2e3, l_field=0x19, period_s=0.29, start_s=0.050, seed=32,
                          data_flips=(16 * 5 + 1, 16 * 20 + 6)),
            synth.Emitter("T1", 0x64700082, amp=90.0, offset_hz=-5e3, l_field=0x19, period_s=0.23, start_s=0.100, seed=33),
            synth.Emitter("S1", 0x02717473, amp=80.0, offset_hz=-3e3, l_field=0x2E, period_s=0.31, start_s=0.150, seed=34)]


def check_capture_repair(lib, pkg, orc_mod=None, e_max=2):
    """manual framing (wmb_poll) of a capture with the flipped emitters: device repair == host twin (== restatement on
    the CPU build); every flipped telegram that no other one overlaps comes back as sent by at least one of its
    candidates (rla, t2a), and no repaired datagram differs from one that was sent"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = flipped_emitters(synth)
    cu8, plan = synth.synth_capture(8 << 20, emitters=ems, seed=0xB2000007)
    cu8 = cu8.numpy()
    flipped = {ems[p.emitter].payload(p.k): p for p in plan if ems[p.emitter].data_flips}
    alone = {d for d, p in flipped.items()                 # no other telegram on the air at the same time
             if not any(q is not p and q.start_iq < p.start_iq + p.n_iq and p.start_iq < q.start_iq + q.n_iq for q in plan)}
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        assert k > 0
        dev = ctx.repair_frames(arr, k, e_max, device=True)
        host = ctx.repair_frames(arr, k, e_max, device=False)
        assert [as_tuple(dev[i]) for i in range(k)] == [as_tuple(host[i]) for i in range(k)]
        if orc_mod is not None:
            for i in range(k):
                f = arr[i]
                w = np.ctypeslib.as_array(f.bits, (f.nbits,)).copy()
                want = rc.repair(orc_mod, f.chain, w & 1, (w >> 1) & 0xFF, w >> 9, f.sync_sample, e_max)
                assert as_tuple(host[i]) == restated_tuple(want), i
        got = {}
        for i in range(k):
            if dev[i].outcome == rc.REPAIRED:
                d = bytes(dev[i].line.datagram[:dev[i].line.len])
                assert d in flipped, d.hex()                  # no repaired datagram differs from one sent
                got[d] = got.get(d, 0) + 1
    assert len(alone) >= 15 and alone <= set(got), (len(alone), len(alone - set(got)))


def test_capture_with_flipped_chips_manual_framing(hostsim_lib, pkg, orc_mod):
    check_capture_repair(hostsim_lib, pkg, orc_mod)
