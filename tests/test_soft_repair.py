"""Soft values of the T1/C1 bits and the C1 soft repair (wmbus_b200_framer.h) on the CPU build: the values of every polled
frame equal the restatement on the oracle's stages (tests/soft_repair_cases.py); the host twin wmb_frame_repair_soft(),
the device repair K4S (wmb_frame_repair_soft_device) and the restatement agree frame by frame on a corpus of C1 telegrams
with weak and strong bit errors, sentinel bits and crafted ambiguous blocks."""
import ctypes as C
import importlib
import os

import numpy as np
import pytest

import orc
import repair_cases as rc
import soft_repair_cases as sc
from test_repair import as_tuple, make_frames, restated_tuple

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def golden(name):
    return np.fromfile(os.path.join(GOLDEN, name), np.uint8)


def c1_emitters(synth):
    return [synth.Emitter("C1A", 0x20338739, amp=60.0, offset_hz=-5e3, l_field=0x19, period_s=0.05, start_s=0.010, seed=31),
            synth.Emitter("C1B", 0x20210116, amp=60.0, offset_hz=4e3, l_field=0x2E, period_s=0.07, start_s=0.030, seed=32)]


def c1_capture(n=4 << 20, seed=0xC1C1):
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    cu8, _ = synth.synth_capture(n, emitters=c1_emitters(synth), seed=seed)
    return np.ascontiguousarray(cu8.numpy())


# ---- the soft value per bit ---------------------------------------------------------------------------------------------

def test_chip_centre_delays_are_the_argmax(orc_mod):
    """D_RL maximises the mean of (2 bit - 1) v over clean C1 telegrams over 0 .. 15; D_T2 over 2 .. 15 only, which departs
    from the plain argmax (D = 1 for t2a): a window reaching past the event's own sample would need a sample its batch
    may not hold"""
    s = sc.d_scores(c1_capture())
    assert max(range(16), key=lambda x: s[0][x]) == sc.D_RL
    assert max(range(16), key=lambda x: s[1][x]) == 1 and sc.D_T2 == 2
    for algo, d in ((0, sc.D_RL), (1, sc.D_T2)):
        best = max(sc.D_RANGE, key=lambda x: s[algo][x])
        assert best == d, (algo, [round(x) for x in s[algo]])
    pkg = importlib.import_module("rtl-wmbus_b200")
    hdr = open(os.path.join(os.path.dirname(pkg.__file__), "..", "include", "wmbus_b200_framer.h")).read()
    assert f"#define WMB_SOFT_D_T2  {sc.D_T2}\n" in hdr and f"#define WMB_SOFT_D_RL  {sc.D_RL}\n" in hdr


SOFT_CASES = [("synth_mixed_1m6.cu8", "", "1mib"), ("synth_mixed_1m6.cu8", "", "one"), ("synth_mixed_1m6.cu8", "", "uneven"),
              ("synth_mixed_1m6.cu8", "-o", "1mib"), ("synth_mixed_1m6.cu8", "-a", "1mib"),
              ("synth_mixed_2m4_shift.cu8", "-d 3 -s", "1mib"), ("c1", "", "1mib"), ("c1", "", "uneven")]


@pytest.mark.parametrize("name,flags,batching", SOFT_CASES)
def test_soft_values_equal_the_restatement(hostsim_lib, pkg, orc_mod, name, flags, batching):
    cu8 = c1_capture() if name == "c1" else golden(name)
    got = sc.polled_soft(pkg, hostsim_lib, cu8, flags, batching)
    want = sc.oracle_streams(cu8, flags)
    assert sc.check_polled_soft(got, want) > 1000
    if flags == "-a":                                        # the cross-product discriminator saturates the values
        assert any(v is not None and (np.abs(v.astype(np.int32)) == 32767).any() for v in got.values())


def test_soft_values_off_means_off(hostsim_lib, pkg):
    """soft values off: no values, and the polled frames, launches and copies are those of a context without them"""
    cu8 = golden("synth_mixed_1m6.cu8")
    runs = []
    for soft in (False, True):
        with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1, soft_bits=soft, max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, len(cu8))
            arr, k = ctx.poll(flush=True)
            frames = [(arr[i].chain, arr[i].algo, arr[i].ordinal, np.ctypeslib.as_array(arr[i].bits, (arr[i].nbits,)).tobytes())
                      for i in range(k)]
            soft_v = [ctx.frame_soft(arr[i]) for i in range(k)]
            runs.append((frames, soft_v, ctx.stats()))
    (f0, s0, st0), (f1, s1, st1) = runs
    assert f0 == f1 and all(v is None for v in s0) and any(v is not None for v in s1)
    assert st1.kernel_launches - st0.kernel_launches == st0.batches + 1      # k3_soft in every gather


def test_setter(hostsim_lib, pkg):
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1) as ctx:
        assert hostsim_lib.wmb_set_soft_bits(ctx._ctx, 2) == -1
        ctx.set_soft_bits(True)
        ctx.push_bytes(bytes(1 << 16))
        assert hostsim_lib.wmb_set_soft_bits(ctx._ctx, 0) != 0
        ctx.reset()
        ctx.set_soft_bits(False)


def test_minimum_weights_of_the_block_codes():
    """DESIGN.md section 8's table: w_min of the shortened CRC code of every block length the rule searches.  Every code
    word has even weight (0x13D65 is divisible by x + 1), so the first word min_weight_word finds has the least weight."""
    for nbits, w in ((96, 6), (88, 6), (144, 6), (1024, 2), (1016, 2)):
        word = sc.min_weight_word(nbits, 6)
        assert word is not None and len(word) == w, (nbits, word)
        cols = sc.syndrome_columns(nbits)
        acc = 0
        for j in word:
            acc ^= cols[j]
        assert acc == 0
    assert sc.min_weight_word(96, 5) is None and sc.min_weight_word(144, 5) is None


# ---- the rule -----------------------------------------------------------------------------------------------------------

def c1_bits(synth, fb, L, k):
    """the frame bits of a clean C1 telegram (flagged bit first, 8 idle pairs after it) and its datagram"""
    e = synth.Emitter("C1B" if fb else "C1A", 0x12345678 + L, l_field=L, seed=50 + L)
    p = e.payload(k)
    wire = synth.frame_b(p) if fb else synth.frame_a(p)
    return synth.chips_c1(wire, fb, 0, 8)[9:].astype(np.uint8), p


def byte_blocks(fb, n):
    return sc.blocks_b(n) if fb else rc.blocks_a(n)


def corpus(synth, k_max, seed=11):
    """C1A / C1B telegrams with 0 .. k_max + 1 flipped bits per block, weak (low |v|) or strong (full swing), some bits
    without a value, and blocks crafted from a minimum-weight code word so that two patterns pass"""
    rng = np.random.default_rng(seed)
    cases = []
    for fb in (False, True):
        for L in (9, 0x0E, 0x19, 0x2E, 0x66, 0x7F, 0xF0 if fb else 0xFF):      # (frame B: L + 4 <= 255)
            for k in range(3):
                bits, p = c1_bits(synth, fb, L, k)
                n = 1 + bits[17:25].dot(1 << np.arange(7, -1, -1)) if fb else rc.tlg_len_a(L)
                P = 17 + 8 * int(n)
                sign = 2 * bits.astype(np.int64) - 1
                soft = (sign * rng.integers(2000, 6000, len(bits))).astype(np.int16)
                strong = bool(rng.integers(0, 4) == 0)
                for off, blk in byte_blocks(fb, int(n)):
                    lo = 17 + 8 * max(off, 1)
                    want = int(rng.integers(0, k_max + 2))
                    for j in rng.choice(np.arange(lo, 17 + 8 * (off + blk)), want, replace=False):
                        bits[j] ^= 1
                        mag = rng.integers(2000, 6000) if strong else rng.integers(10, 600)
                        soft[j] = (2 * int(bits[j]) - 1) * mag
                for j in rng.choice(np.arange(17, P), int(rng.integers(0, 3)), replace=False):
                    soft[j] = sc.NONE
                cases.append(dict(chain=0, bits=bits, rssi=np.full(len(bits), 100, np.uint8), soft=soft, sent=p))
    cases += ambiguous_cases(synth)
    return cases


def ambiguous_cases(synth):
    """a block with half of a minimum-weight code word flipped and the word's bits least reliable: at K >= the word's
    weight both halves pass.  Frame A's blocks (96 and 144 bits) have weight 6; frame B's 1024-bit block weight 2 (here
    the words avoid the L byte: the shortened codes of 88 and 1016 bits)."""
    out = []
    for fb, L, nbits, block_byte in ((False, 0x19, 144, 12), (False, 0x19, 88, 1), (True, 0xC8, 1016, 1)):
        bits, p = c1_bits(synth, fb, L, 0)
        word = sc.min_weight_word(nbits, 6)
        first = 17 + 8 * block_byte
        pos = [first + w for w in word]
        soft = ((2 * bits.astype(np.int64) - 1) * 4000).astype(np.int16)
        for j in pos:
            soft[j] = 1 if bits[j] else -1
        for j in pos[:len(pos) // 2]:
            bits[j] ^= 1
            soft[j] = -soft[j]
        out.append(dict(chain=0, bits=bits, rssi=np.full(len(bits), 100, np.uint8), soft=soft, sent=p, weight=len(word)))
    return out


def soft_ptrs(cases):
    arrs = [np.ascontiguousarray(c["soft"], np.int16) if c.get("soft") is not None else None for c in cases]
    return arrs, (C.c_void_p * len(cases))(*[None if a is None else a.ctypes.data for a in arrs])


def run_rule(lib, pkg, cases, e_max, k_max):
    frames, keep = make_frames(pkg, cases)
    arrs, ptrs = soft_ptrs(cases)
    host = (pkg.WmbRepaired * len(cases))()
    for i in range(len(cases)):
        assert lib.wmb_frame_repair_soft(C.addressof(frames[i]), ptrs[i], e_max, k_max, C.addressof(host[i])) == 0
    dev = (pkg.WmbRepaired * len(cases))()
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_frame_repair_soft_device(ctx._ctx, C.addressof(frames), ptrs, len(cases), e_max, k_max,
                                                C.addressof(dev)) == 0, lib.wmb_last_error()
    return (frames, keep), host, dev


def restated(orc_mod, c, f, e_max, k_max):
    w = np.ctypeslib.as_array(f.bits, (f.nbits,))
    consumed, line = rc.oracle_verdict(orc_mod, c["chain"], c["bits"], c["rssi"])
    if k_max and c.get("soft") is not None and c["chain"] == 0 and line is not None and line.startswith("C1;0;"):
        r = sc.repair_soft_c1(c["bits"], c["rssi"], c["soft"], k_max)
        if r["outcome"] == rc.REPAIRED:
            r["end_sample"] = f.sync_sample + int(w[r["consumed"] - 1] >> 9)
        return r
    return rc.repair(orc_mod, c["chain"], w & 1, (w >> 1) & 0xFF, w >> 9, f.sync_sample, e_max)


@pytest.mark.parametrize("k_max", [1, 2, 4, 6])
def test_rule_host_device_restatement(hostsim_lib, pkg, orc_mod, k_max):
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    cases = corpus(synth, k_max)
    (frames, keep), host, dev = run_rule(hostsim_lib, pkg, cases, 2, k_max)
    seen, wrong = set(), 0
    for i, c in enumerate(cases):
        h = as_tuple(host[i])
        assert as_tuple(dev[i]) == h, i
        assert restated_tuple(restated(orc_mod, c, frames[i], 2, k_max)) == h, i
        seen.add(host[i].outcome)
        if "weight" in c:                                     # crafted: ambiguous exactly from the word's weight on
            assert (host[i].outcome == rc.AMBIGUOUS) == (k_max >= c["weight"]), (i, c["weight"])
        if host[i].outcome == rc.REPAIRED and bytes(host[i].line.datagram[:host[i].line.len]) != c["sent"]:
            wrong += 1                                        # a wrong repair needs an error outside the K bits searched
            assert not within_k(synth, c, k_max), i
    assert {rc.REPAIRED, rc.UNREPAIRABLE} | ({rc.AMBIGUOUS} if k_max >= 2 else set()) <= seen
    assert wrong <= 2, wrong


def within_k(synth, c, k_max):
    """the flipped bits of a corpus telegram lie among its K least reliable bits, block by block (and it has flips)"""
    fb, n_bytes = sc.c1_layout(c["bits"])
    P = 17 + 8 * n_bytes
    key = sc.reliabilities(c["bits"], c["soft"], P)
    sent_bits = np.unpackbits(np.frombuffer(sent_wire(synth, fb, c["sent"]), np.uint8))
    diff = np.nonzero(c["bits"][17:P] != sent_bits[:P - 17])[0] + 17
    ok = len(diff) > 0
    for off, blk in byte_blocks(fb, n_bytes):
        cand = sorted(range(17 + 8 * max(off, 1), 17 + 8 * (off + blk)), key=lambda j: (key[j - 17], j))[:k_max]
        ok &= {int(j) for j in diff if 17 + 8 * off <= j < 17 + 8 * (off + blk)} <= set(cand)
    return bool(ok)


def test_flips_among_the_least_reliable_come_back(hostsim_lib, pkg, orc_mod):
    """every corpus telegram whose flipped bits lie among its K least reliable bits, block by block, is REPAIRED as sent"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    k_max = 4
    cases = [c for c in corpus(synth, k_max, seed=5) if "weight" not in c]
    _, host, _ = run_rule(hostsim_lib, pkg, cases, 0, k_max)
    n = 0
    for i, c in enumerate(cases):
        if sc.c1_layout(c["bits"])[1] < 12 or not within_k(synth, c, k_max):
            continue
        n += 1
        assert host[i].outcome == rc.REPAIRED, i
        assert bytes(host[i].line.datagram[:host[i].line.len]) == c["sent"]
    assert n >= 5


def sent_wire(synth, fb, p):
    return synth.frame_b(p) if fb else synth.frame_a(p)


def test_other_frames_and_k_max_zero_are_wmb_frame_repair(hostsim_lib, pkg):
    """T1 and S1 candidates, and every frame at k_max = 0 or without soft values, repair exactly as wmb_frame_repair"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    from test_repair import planted_cases
    cases = planted_cases(synth, 2) + corpus(synth, 3)[:40]
    frames, keep = make_frames(pkg, cases)
    arrs, ptrs = soft_ptrs(cases)
    for e_max, k_max, use_soft in ((2, 0, True), (3, 4, True), (1, 6, False)):
        for i in range(len(cases)):
            a, b = pkg.WmbRepaired(), pkg.WmbRepaired()
            assert hostsim_lib.wmb_frame_repair(C.addressof(frames[i]), e_max, C.addressof(a)) == 0
            assert hostsim_lib.wmb_frame_repair_soft(C.addressof(frames[i]), ptrs[i] if use_soft else None, e_max, k_max,
                                                     C.addressof(b)) == 0
            if cases[i]["chain"] == 0 and use_soft and k_max and "soft" in cases[i]:
                continue                                      # C1 with values: the soft rule
            assert as_tuple(a) == as_tuple(b), (i, e_max, k_max)
    r = pkg.WmbRepaired()
    assert hostsim_lib.wmb_frame_repair_soft(C.addressof(frames[0]), ptrs[0], 2, 7, C.addressof(r)) == -1


def test_capture_soft_repair_manual_framing(hostsim_lib, pkg, orc_mod):
    """a C1 capture decoded with manual framing and soft values: K4S equals the host twin on every polled candidate, and
    no repaired datagram differs from a sent one"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = c1_emitters(synth)
    cu8, plan = synth.synth_capture(4 << 20, emitters=ems, seed=0xC1C2, noise_sigma=34.0)
    cu8 = np.ascontiguousarray(cu8.numpy())
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1, soft_bits=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        dev = ctx.repair_frames(arr, k, 2, device=True, k_max=6)
        host = ctx.repair_frames(arr, k, 2, device=False, k_max=6)
    assert [as_tuple(dev[i]) for i in range(k)] == [as_tuple(host[i]) for i in range(k)]
    for i in range(k):
        if host[i].outcome == rc.REPAIRED:
            assert bytes(host[i].line.datagram[:host[i].line.len]) in sent
