"""The S1 soft repair (wmb_frame_repair_s1_soft; wmbus_b200_framer.h) on the CPU build: the soft value of every S1 chip
equals the restatement on the oracle's stages (tests/s1_soft_cases.py); the delays are the argmax; ML decoding of clean S1
lines gives their hard bits; the distance of the blocks; the host twin, the device repair K4S
(wmb_frame_repair_s1_soft_device) and the restatement agree frame by frame on a corpus of S1 telegrams with weak and strong
chip errors; and on the streaming path the records equal the restatement from manual framing, the lines and statistics do
not move, time chunks merge, and setter, boundary state and CLI behave."""
import ctypes as C
import hashlib
import importlib

import numpy as np
import pytest

import repair_cases as rc
import repair_stream_cases as rs
import s1_soft_cases as s1c
import soft_repair_cases as sc
from test_repair import as_tuple, make_frames, planted_cases, restated_tuple
from test_repair_stream import blank_ts, cli

S_MAXES = (1, 2, 3, 4, 5, 6)


def synth_mod():
    return importlib.import_module("rtl-wmbus_b200.synth")


def s1_clean_capture(n=4 << 20, sigma=8.0, ls=(0x19, 0x2E)):
    synth = synth_mod()
    ems = [synth.Emitter("S1", 0x20338739, amp=60.0, offset_hz=-5e3, l_field=ls[0], period_s=0.05, start_s=0.010, seed=31),
           synth.Emitter("S1", 0x20210116, amp=60.0, offset_hz=4e3, l_field=ls[1], period_s=0.07, start_s=0.030, seed=32)]
    cu8, _ = synth.synth_capture(n, emitters=ems, seed=0x5151, noise_sigma=sigma)
    return np.ascontiguousarray(cu8.numpy())


# ---- soft values --------------------------------------------------------------------------------------------------------

def mixed_capture():
    import receiver_cases as rcs
    return rcs.cached_capture("synth_mixed_1m6.cu8")


@pytest.fixture(scope="module")
def mixed():
    """S1 and T1/C1 telegrams on one committed capture"""
    return mixed_capture()


def check_soft_values(pkg, lib, cu8):
    """every S1 event's value on both algorithms, and every T1/C1 one, equals the restatement, in one batch, 1 MiB
    batches and ragged pushes"""
    want_s1, want_t1c1 = s1c.oracle_streams(cu8, "-v"), sc.oracle_streams(cu8, "-v")
    for batching in ("one", "1mib", "uneven"):
        got = s1c.polled_soft(pkg, lib, cu8, "-v", batching, batch_mib=8 if batching == "one" else 1)
        assert s1c.check_polled_soft(got, want_s1, want_t1c1) > 1000


def test_soft_values_equal_the_restatement(hostsim_lib, pkg, mixed):
    check_soft_values(pkg, hostsim_lib, mixed)


@pytest.mark.parametrize("order", ["1", "2"])
def test_soft_values_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled (read once per process: a subprocess)"""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, test_s1_soft_repair as t;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200');"
            "t.check_soft_values(pkg, pkg.load_library(HOSTSIM_SO), t.mixed_capture())" % (root, here))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, WMB_HOSTSIM_ORDER=order),
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


def test_soft_none_at_a_seek_and_past_the_run_cap(hostsim_lib, pkg, mixed):
    """after a seek, the first events' windows start before the first sample; an rla run's events past the cap of 31
    later ones have no value -- in the restatement and in the polled values alike"""
    ev = dict(m=np.full(40, 2000, np.uint64))
    v, _, _ = s1c.soft_values(np.zeros(4000, np.float32), ev, 0)
    assert (v[:8] == sc.NONE).all() and (v[8:] != sc.NONE).all()
    half = np.ascontiguousarray(mixed[len(mixed) // 2 // 4096 * 4096:])
    got = s1c.polled_soft(pkg, hostsim_lib, half, "-v")
    want = s1c.oracle_streams(half, "-v")
    s1c.check_polled_soft(got, want, sc.oracle_streams(half, "-v"))
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1, soft_bits=True, soft_bits_s1=True) as ctx:
        ctx.push(mixed.ctypes.data, len(mixed))
        ctx.poll(flush=True)
        ctx.seek(0)
        ctx.push(half.ctypes.data, len(half))
        arr, k = ctx.poll(flush=True)
        after_seek = {(arr[i].chain, arr[i].algo, arr[i].ordinal): ctx.frame_soft(arr[i]) for i in range(k)}
    assert after_seek.keys() == got.keys()
    assert all(np.array_equal(after_seek[key], got[key]) for key in got)
    assert any((v[:8] == sc.NONE).any() for v in (want[0][1], want[1][1]))


def test_s1_setter_off_changes_nothing(hostsim_lib, pkg, mixed):
    """without wmb_set_soft_bits_s1: T1/C1 values unchanged and wmb_frame_soft(S1) is NULL; the setter's rules"""
    off = sc.polled_soft(pkg, hostsim_lib, mixed, "-v")
    sc.check_polled_soft(off, sc.oracle_streams(mixed, "-v"))
    lib = hostsim_lib
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_set_soft_bits_s1(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        assert lib.wmb_set_soft_bits_s1(ctx._ctx, 2) == -1
        assert lib.wmb_set_soft_bits_s1(ctx._ctx, 1) == 0
        ctx.push(mixed.ctypes.data, 1 << 20)
        assert lib.wmb_set_soft_bits_s1(ctx._ctx, 0) != 0 and b"after samples were pushed" in lib.wmb_last_error()
        ctx.reset()
        assert lib.wmb_set_soft_bits_s1(ctx._ctx, 0) == 0
    assert lib.wmb_set_soft_bits(None, 2) == -1


# ---- calibration and ML -------------------------------------------------------------------------------------------------

def test_chip_centre_delays_are_the_argmax():
    """WMB_SOFT_S1_D_RL / _D_T2 are the argmax over 7..48 of the mean signed value over the chips [17, P) of the clean S1
    lines of the calibration capture, and no chip of those lines clamps at WMB_SOFT_S1_SHIFT"""
    s, peak = s1c.d_scores(s1_clean_capture())
    print("S1 chip-centre scores rla:", {d: round(v) for d, v in s[0].items()})
    print("S1 chip-centre scores t2a:", {d: round(v) for d, v in s[1].items()})
    assert max(s[0], key=lambda d: s[0][d]) == s1c.D_RL
    assert max(s[1], key=lambda d: s[1][d]) == s1c.D_T2
    assert peak <= 32767, peak


def test_ml_gives_the_hard_bits_of_clean_lines(hostsim_lib, pkg):
    """every pair of every CRC-ok S1 line of a clean capture: its ML bit is its hard bit"""
    cu8 = s1_clean_capture()
    lib = hostsim_lib
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    n = 0
    with pkg.WmbusB200("", lib=lib, manual_frames=1, soft_bits_s1=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        for i in range(k):
            f = arr[i]
            d = pkg.WmbDecoded()
            lib.wmb_frame_decode(C.addressof(f), C.addressof(d))
            if f.chain != 1 or d.status != 1 or not d.crc_ok:
                continue
            w = np.ctypeslib.as_array(f.bits, (f.nbits,)) & 1
            soft = ctx.frame_soft(f)
            for p in range(8, (int(d.consumed) - 1) // 2):
                ml, _, hard = s1c.pair(w, soft, p)
                assert ml == hard, (i, p)
                n += 1
    assert n > 5000


# ---- distance -----------------------------------------------------------------------------------------------------------

def test_distance_of_the_blocks():
    """the least weight of the shortened CRC code on S1's blocks (88 searchable bits in the first, 144 in a later one)
    is 6, so no block can be AMBIGUOUS below K = 6"""
    for nbits in (88, 144):
        assert sc.min_weight_word(nbits, 5) is None
        w = sc.min_weight_word(nbits, 6)
        assert w is not None and len(w) == 6


# ---- the rule -----------------------------------------------------------------------------------------------------------

def full_corpus(s_max):
    """S1 telegrams (the corpus and crafted AMBIGUOUS blocks), S1 ones without soft values, random bit lists, and T1 and
    C1 telegrams (left to the erasure rule)"""
    from test_repair import random_cases
    synth = synth_mod()
    s1 = s1c.corpus(synth, s_max)
    no_soft = [dict(c, soft=None) for c in s1[::4]]
    others = [dict(c, soft=np.zeros(len(c["bits"]), np.int16)) for c in planted_cases(synth, 2) if c["chain"] == 0]
    rnd = [dict(c, soft=np.random.default_rng(i).integers(-3000, 3000, len(c["bits"])).astype(np.int16))
           for i, c in enumerate(random_cases(60))]
    return s1 + s1c.ambiguous_cases(synth) + no_soft + others + rnd


@pytest.mark.parametrize("e_max", [1, 3])
@pytest.mark.parametrize("s_max", S_MAXES)
def test_rule_host_device_restatement(hostsim_lib, pkg, orc_mod, s_max, e_max):
    cases = full_corpus(s_max)
    (frames, keep, arrs), host, dev = s1c.run_rule(hostsim_lib, pkg, cases, e_max, s_max)
    seen = set()
    for i, c in enumerate(cases):
        h = as_tuple(host[i])
        assert as_tuple(dev[i]) == h, i
        assert restated_tuple(s1c.restated(orc_mod, c, frames[i], e_max, s_max)) == h, i
        if c["chain"] == 1 and "wire" in c:
            seen.add(host[i].outcome)
        if "weight" in c:                                     # crafted: AMBIGUOUS exactly from the distance on
            assert (host[i].outcome == rc.AMBIGUOUS) == (s_max >= c["weight"]), (i, s_max)
    assert {rc.REPAIRED, rc.UNREPAIRABLE} <= seen
    if s_max >= 6:
        assert rc.AMBIGUOUS in seen


def test_every_outcome_occurs(hostsim_lib, pkg):
    seen = set()
    for s_max in (1, 6):
        for e_max in (1, 3):
            cases = full_corpus(s_max)
            _, host, _ = s1c.run_rule(hostsim_lib, pkg, cases, e_max, s_max)
            seen |= {host[i].outcome for i in range(len(cases))}
    assert seen == set(range(6)), seen


@pytest.mark.parametrize("s_max", [1, 3, 6])
def test_wrong_bits_among_the_searched_come_back(hostsim_lib, pkg, s_max):
    """every corpus telegram whose wrong bits lie among its K searched pairs, block by block, comes back as sent --
    unless the erasure rule repaired it first or found it AMBIGUOUS, which stands; no repaired datagram was not sent"""
    synth = synth_mod()
    cases = [c for seed in (5, 6) for c in s1c.corpus(synth, s_max, seed=seed)]
    _, host, _ = s1c.run_rule(hostsim_lib, pkg, cases, 1, s_max)
    frames, keep = make_frames(pkg, cases)
    sent = {c["sent"] for c in cases}
    n = 0
    for i, c in enumerate(cases):
        if host[i].outcome == rc.REPAIRED:
            assert bytes(host[i].line.datagram[:host[i].line.len]) in sent, i
        if not s1c.within_k(c, s_max):
            continue
        r0 = pkg.WmbRepaired()
        assert hostsim_lib.wmb_frame_repair(C.addressof(frames[i]), 1, C.addressof(r0)) == 0
        if r0.outcome == rc.AMBIGUOUS:
            continue
        n += 1
        assert host[i].outcome == rc.REPAIRED, (i, host[i].outcome)
        assert bytes(host[i].line.datagram[:host[i].line.len]) == c["sent"], i
    assert n >= (1 if s_max == 1 else 5), n


def test_erasure_outcomes_stand_and_other_frames_are_wmb_frame_repair(hostsim_lib, pkg):
    synth = synth_mod()
    cases = full_corpus(4) + planted_cases(synth, 2)
    frames, keep = make_frames(pkg, cases)
    arrs, ptrs = s1c.soft_ptrs([dict(c, soft=c.get("soft", np.zeros(len(c["bits"]), np.int16))) for c in cases])
    n_stand = 0
    for e_max, s_max, use_soft in ((1, 0, True), (3, 4, True), (2, 6, False), (1, 6, True)):
        for i in range(len(cases)):
            a, b = pkg.WmbRepaired(), pkg.WmbRepaired()
            assert hostsim_lib.wmb_frame_repair(C.addressof(frames[i]), e_max, C.addressof(a)) == 0
            assert hostsim_lib.wmb_frame_repair_s1_soft(C.addressof(frames[i]), ptrs[i] if use_soft else None, e_max,
                                                        s_max, C.addressof(b)) == 0
            if cases[i]["chain"] == 1 and use_soft and s_max and a.outcome in (rc.TOO_MANY, rc.UNREPAIRABLE):
                continue                                      # possibly the soft rule
            n_stand += a.outcome in (rc.REPAIRED, rc.AMBIGUOUS, rc.TRUNCATED)
            assert as_tuple(a) == as_tuple(b), (i, e_max, s_max)
    assert n_stand >= 20
    r = pkg.WmbRepaired()
    assert hostsim_lib.wmb_frame_repair_s1_soft(C.addressof(frames[0]), ptrs[0], 2, 7, C.addressof(r)) == -1
    assert hostsim_lib.wmb_frame_repair_s1_soft(C.addressof(frames[0]), ptrs[0], 4, 2, C.addressof(r)) == -1


def capture_manual_framing(lib, pkg, orc_mod, sigma=40.0):
    """a noisy S1 capture decoded with manual framing and S1 soft values: K4S equals the host twin (and, given orc_mod,
    the restatement) on every polled candidate, and no repaired datagram differs from a sent one"""
    synth = synth_mod()
    ems = s1c.s1_emitters(synth)[:3]
    cu8, plan = synth.synth_capture(4 << 20, emitters=ems, seed=0x7173, noise_sigma=sigma)
    cu8 = np.ascontiguousarray(cu8.numpy())
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1, soft_bits_s1=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        soft = [ctx.frame_soft(arr[i]) for i in range(k)]
        n_soft = 0
        for s_max in S_MAXES:
            dev = ctx.repair_frames(arr, k, 3, device=True, s1_max=s_max, soft=soft)
            host = ctx.repair_frames(arr, k, 3, device=False, s1_max=s_max, soft=soft)
            assert [as_tuple(dev[i]) for i in range(k)] == [as_tuple(host[i]) for i in range(k)]
            for i in range(k):
                if host[i].outcome == rc.REPAIRED:
                    assert bytes(host[i].line.datagram[:host[i].line.len]) in sent
                if orc_mod is not None and s_max == 6 and arr[i].chain == 1 and soft[i] is not None:
                    w = np.ctypeslib.as_array(arr[i].bits, (arr[i].nbits,))
                    c = dict(chain=1, bits=(w & 1).astype(np.uint8), rssi=((w >> 1) & 0xFF).astype(np.uint8), soft=soft[i])
                    assert restated_tuple(s1c.restated(orc_mod, c, arr[i], 3, 6)) == as_tuple(host[i]), i
                    n_soft += 1
    return n_soft


def test_capture_manual_framing(hostsim_lib, pkg, orc_mod):
    assert capture_manual_framing(hostsim_lib, pkg, orc_mod) > 20


# ---- the streaming path -------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cap():
    return s1c.s1_capture()


SETTINGS = (0, 1, 3, 6)


@pytest.fixture(scope="module")
def want(hostsim_lib, pkg, cap):
    return s1c.restated_stream(pkg, hostsim_lib, cap[0], "-v", 2, SETTINGS)


@pytest.fixture(scope="module")
def runs(hostsim_lib, pkg, cap):
    """the capture in 1 MiB batches at e_max 2, with quality and bursts on, per s_max"""
    return {s: s1c.stream(pkg, hostsim_lib, cap[0], "-v", 2, quality=True, burst_level=(14, 14), repair_s1_soft=s)
            for s in SETTINGS}


def s1_soft_records(recs):
    return [t for t in recs if t[-1]]


@pytest.mark.parametrize("s_max", SETTINGS)
def test_records_equal_the_restatement(runs, want, s_max):
    assert runs[s_max][0] == want[s_max]
    if s_max:
        assert sum(1 for t in s1_soft_records(runs[s_max][0]) if t[4] == rc.REPAIRED) >= 5
    else:
        assert not s1_soft_records(runs[s_max][0])


@pytest.mark.parametrize("s_max,batching", [(6, "one"), (3, "uneven"), (2, "uneven")])
def test_records_equal_the_restatement_other_batchings(hostsim_lib, pkg, cap, s_max, batching):
    got = s1c.stream(pkg, hostsim_lib, cap[0], "-v", 2, batching, batch_mib=8 if batching == "one" else 1,
                     repair_s1_soft=s_max)[0]
    assert got == s1c.restated_stream(pkg, hostsim_lib, cap[0], "-v", 2, [s_max])[s_max]


def test_weak_s1_telegrams_come_back_as_sent(runs, cap):
    _, plan, ems = cap
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    weak = {ems[p.emitter].payload(p.k): p for p in plan if ems[p.emitter].weak_flips and ems[p.emitter].mode == "S1"}
    alone = {d for d, p in weak.items()
             if not any(q is not p and q.start_iq < p.start_iq + p.n_iq and p.start_iq < q.start_iq + q.n_iq for q in plan)}
    assert len(alone) >= 5
    for s in SETTINGS:
        got = {t[-3] for t in runs[s][0] if t[4] == rc.REPAIRED}
        assert got <= sent, "a repaired datagram that was never sent"
        if s >= 3:
            assert alone <= got, (s, len(alone - got))


def test_off_means_off_and_nothing_else_moves(runs):
    """any s_max: the non-S1-soft records, lines, records, bursts and statistics but kernel_launches (+3 per gather:
    k3_soft, k3_soft_s1_kernel and K4S's S1 instance) and d2h_bytes stay"""
    recs0, lines0, info0, qual0, bursts0, st0 = runs[0]
    for s in SETTINGS[1:]:
        recs, lines, info, qual, bursts, st = runs[s]
        soft_keys = {(t[0], t[2], t[3]) for t in recs if t[-1]}
        assert [t for t in recs if not t[-1]] == [t for t in recs0 if (t[0], t[2], t[3]) not in soft_keys]
        assert all(t[4] in (rc.TOO_MANY, rc.UNREPAIRABLE) for t in recs0 if (t[0], t[2], t[3]) in soft_keys)
        assert lines == lines0
        assert info.tobytes() == info0.tobytes() and qual.tobytes() == qual0.tobytes()
        assert bursts.tobytes() == bursts0.tobytes()
        for name, _t in st._fields_:
            if name in ("kernel_launches", "d2h_bytes") or name.endswith("_ms"):
                continue
            a, b = getattr(st, name), getattr(st0, name)
            if not isinstance(a, (int, float)):
                a, b = bytes(a), bytes(b)
            assert a == b, name
        assert st.kernel_launches - st0.kernel_launches == 3 * (st.batches + 1)
        assert st.d2h_bytes >= st0.d2h_bytes


def test_off_is_the_parent_path(hostsim_lib, pkg, cap):
    """s_max 0 set explicitly: records, launches and copies equal a context that never heard of the setting"""
    a = s1c.stream(pkg, hostsim_lib, cap[0], "-v", 2)
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, max_batch_mib=1) as ctx:
        ctx.set_repair_s1_soft(3)
        ctx.set_repair_s1_soft(0)
        recs = []
        for lo, hi in rs.pushes(len(cap[0]), "1mib"):
            ctx.push(cap[0].ctypes.data + lo, hi - lo)
            recs += ctx.take_repairs()
        ctx.poll_flush()
        recs = [s1c.record_tuple(r) for r in recs + ctx.take_repairs()]
        st = ctx.stats()
    assert recs == a[0]
    assert (st.kernel_launches, st.d2h_bytes) == (a[5].kernel_launches, a[5].d2h_bytes)


def test_time_chunks_merge_to_the_sequential_records(hostsim_lib, pkg, runs, cap):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = cap[0]
    parts = []
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_s1_soft=6, max_batch_mib=1) as ctx:
        def push(lo, hi):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
        for rank in range(3):
            out, _ds, _de, _start = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, repairs=True)
            parts.append(out[-1])
    assert [s1c.record_tuple(r) for r in shard.merge_repairs(parts)] == runs[6][0]


def test_setter_and_boundary_state(hostsim_lib, pkg, cap):
    lib = hostsim_lib
    cu8 = cap[0]
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 7) == -1
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 6) == 0
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 1) != 0 and b"after samples were pushed" in lib.wmb_last_error()
        ctx.reset()
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 2) == 0
        ctx.seek(0)
        assert lib.wmb_set_repair_s1_soft(ctx._ctx, 0) == 0
    digests = {}
    for ks in ((0, 0, 0), (0, 0, 1), (0, 0, 6), (0, 1, 0), (0, 1, 1), (4, 4, 4)):
        with pkg.WmbusB200("-v", lib=lib, repair=2, repair_soft=ks[0], repair_t1_soft=ks[1], repair_s1_soft=ks[2],
                           max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, 3 * rs.MIB)
            digests[ks] = ctx.boundary_state()
    assert len({hashlib.sha256(v).digest() for v in digests.values()}) == len(digests)
    for ks in ((0, 0, 1), (0, 0, 6), (0, 1, 1), (4, 4, 4)):      # s_max appended: the bytes before it are unchanged
        base = digests[ks[:2] + (0,)] if ks[:2] + (0,) in digests else None
        if base is not None:
            assert digests[ks][:len(base)] == base and len(digests[ks]) == len(base) + 5


def test_cli_repaired_file(hostsim_lib, pkg, cap, tmp_path):
    cu8 = cap[0]
    path = tmp_path / "repaired.txt"
    plain = cli(["-v"], cu8, {})
    assert plain.returncode == 0, plain.stderr
    r = cli(["-v"], cu8, {"WMBUS_B200_REPAIRED": str(path), "WMBUS_B200_REPAIR_ERASURES": "2",
                          "WMBUS_B200_REPAIR_S1_SOFT_BITS": "4"})
    assert r.returncode == 0, r.stderr
    assert r.stdout == plain.stdout or [blank_ts(l, True) for l in r.stdout.decode().splitlines()] == \
        [blank_ts(l, True) for l in plain.stdout.decode().splitlines()]
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_s1_soft=4, max_batch_mib=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        recs = ctx.take_repairs()
        want = [ctx.repaired_line(x, b"rla;" if x.algo == 0 else b"t2a;") for x in recs if x.repair.outcome == rc.REPAIRED]
        n_soft = sum(1 for x in recs if x.soft_s1 and x.repair.outcome == rc.REPAIRED)
    got = [blank_ts(l, True) for l in path.read_text().splitlines()]
    assert got == want and n_soft >= 5


@pytest.mark.parametrize("env", [{"WMBUS_B200_REPAIR_S1_SOFT_BITS": "2"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_S1_SOFT_BITS": "0"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_S1_SOFT_BITS": "7"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_S1_SOFT_BITS": "x"}])
def test_cli_bad_setting_fails_at_start_up(hostsim_lib, tmp_path, env):
    env = {k: v.replace("{tmp}", str(tmp_path / "r.txt")) for k, v in env.items()}
    r = cli(["-v"], np.zeros(8192, np.uint8), env)
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_REPAIR_S1_SOFT_BITS" in r.stderr, r.stderr
