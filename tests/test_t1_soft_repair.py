"""The T1 soft repair (wmb_frame_repair_t1_soft; wmbus_b200_framer.h) on the CPU build: ML decoding of clean T1 lines
gives their hard symbols; the distance of the block codes in nibble substitutions; the host twin, the device repair K4S
(wmb_frame_repair_t1_soft_device) and the restatement (tests/t1_soft_cases.py) agree frame by frame on a corpus of T1
telegrams with weak and strong chip errors; and on the streaming path the records equal the restatement from manual
framing, the lines and statistics do not move, time chunks merge, and setter, boundary state and CLI behave."""
import ctypes as C
import hashlib
import importlib

import numpy as np
import pytest

import orc
import receiver_oracle as ro
import repair_cases as rc
import repair_stream_cases as rs
import soft_repair_cases as sc
import t1_soft_cases as tc
from test_repair import as_tuple, make_frames, planted_cases, restated_tuple
from test_repair_stream import blank_ts, cli

S_MAXES = (1, 2, 3, 4, 5, 6)


def synth_mod():
    return importlib.import_module("rtl-wmbus_b200.synth")


def t1_clean_capture(n=4 << 20, sigma=8.0):
    synth = synth_mod()
    ems = [synth.Emitter("T1", 0x20338739, amp=60.0, offset_hz=-5e3, l_field=0x19, period_s=0.05, start_s=0.010, seed=31),
           synth.Emitter("T1", 0x20210116, amp=60.0, offset_hz=4e3, l_field=0x2E, period_s=0.07, start_s=0.030, seed=32)]
    cu8, _ = synth.synth_capture(n, emitters=ems, seed=0x7171, noise_sigma=sigma)
    return np.ascontiguousarray(cu8.numpy())


# ---- ML on clean telegrams ----------------------------------------------------------------------------------------------

def t1_d_scores(cu8):
    """{algo: [mean of (2 chip - 1) v over the chips [13, P) of every CRC-clean T1 line, for D = 0 .. 15]}"""
    o = orc.opts_from_flags("")
    st = orc.stages(cu8, o, 0)
    L = orc.lib()
    buf = C.create_string_buffer(4096)
    got = C.c_int(0)
    out = {}
    for algo in (0, 1):
        ev = ro.stream_events(st, 0, algo, 2, 0)
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
            if got.value and buf.value.startswith(b"T1;1;"):
                sel.append(np.arange(c + 13, c + used))
            busy = c + used
        idx = np.concatenate(sel)
        sign = 2 * bits[idx].astype(np.int64) - 1
        scores = []
        for d in range(16):
            v = sc.soft_values(st["fir"], ev, algo, d, d)[idx].astype(np.int64)
            ok = v != sc.NONE
            scores.append(float((sign[ok] * v[ok]).mean()))
        out[algo] = scores
    return out


def test_t1_chip_centre_delays(orc_mod):
    """the argmax of the mean signed value over clean T1 lines, reported for DESIGN.md section 8; the delays stay those
    calibrated on C1 (changing them would change the C1 soft values).  The T1 rule needs the values' sign and order,
    which the next test checks symbol by symbol."""
    s = t1_d_scores(t1_clean_capture())
    best = {algo: max(range(16), key=lambda x: s[algo][x]) for algo in (0, 1)}
    print("T1 chip-centre delay argmax (rla, t2a):", best[0], best[1],
          "margins at D_RL / D_T2:", round(s[0][sc.D_RL]), round(s[1][sc.D_T2]))
    assert s[0][sc.D_RL] > 0 and s[1][sc.D_T2] > 0


def test_ml_gives_the_hard_symbols_of_clean_lines(hostsim_lib, pkg):
    """every symbol of every CRC-ok T1 line of a clean capture (sigma 8): ML of its soft values is its hard symbol"""
    cu8 = t1_clean_capture()
    lib = hostsim_lib
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    n = 0
    with pkg.WmbusB200("", lib=lib, manual_frames=1, soft_bits=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        for i in range(k):
            f = arr[i]
            d = pkg.WmbDecoded()
            lib.wmb_frame_decode(C.addressof(f), C.addressof(d))
            if f.chain != 0 or d.status != 1 or d.mode != b"T1" or not d.crc_ok:
                continue
            w = np.ctypeslib.as_array(f.bits, (f.nbits,)) & 1
            soft = ctx.frame_soft(f)
            P = int(d.consumed)
            y, _ = tc.centred(w, soft, P)
            for s in range(2, (P - 1) // 6):
                first = 1 + 6 * s
                ml, _, _ = tc.symbol_scores(y[first:first + 6])
                assert rc.ENC_3OF6[ml] == tc.word(w, first, 6), (i, s)
                n += 1
    assert n > 5000


# ---- the block codes in nibble substitutions ----------------------------------------------------------------------------

def test_symbol_distance_of_the_blocks():
    """the least number of nibble substitutions (distinct symbols) that cancel in the block CRC: 3 in the first block's
    22 searchable symbols and in a later block's 36, so a block can be AMBIGUOUS from K = 3 on"""
    for nbytes, first in ((12, 1), (18, 0)):
        assert tc.min_substitutions(nbytes, first, 2) is None
        word = tc.min_substitutions(nbytes, first, 4)
        assert word is not None and len(word) == 3 and len({s for s, _ in word}) == 3
        subs = tc.substitution_syndromes(nbytes, first)
        acc = 0
        for k in word:
            acc ^= subs[k]
        assert acc == 0


# ---- the rule -----------------------------------------------------------------------------------------------------------

def full_corpus(s_max):
    """T1 telegrams (tests/t1_soft_cases.py corpus and crafted AMBIGUOUS blocks), C1 telegrams with soft values and S1
    telegrams with flipped chips"""
    from test_soft_repair import corpus as c1_corpus
    synth = synth_mod()
    s1 = [c for c in planted_cases(synth, 2) if c["chain"] == 1]
    t1 = tc.corpus(synth, s_max)
    no_soft = [dict(c, soft=None) for c in t1[::4]]            # the erasure rule's outcome, TOO_MANY included, stands
    from test_repair import telegram_chips
    chips, p = telegram_chips(synth, "S1", 0x19, 0)               # a Manchester violation, the list ending before P
    chips[1 + 16 * 3] ^= 1
    P = 1 + 16 * rc.tlg_len_a(0x19)
    cut = dict(chain=1, bits=chips[:P - 5], rssi=np.full(P - 5, 100, np.uint8), sent=p)
    return t1 + tc.ambiguous_cases(synth) + no_soft + c1_corpus(synth, 3)[:20] + s1 + [cut]


@pytest.mark.parametrize("e_max", [1, 3])
@pytest.mark.parametrize("s_max", S_MAXES)
def test_rule_host_device_restatement(hostsim_lib, pkg, orc_mod, s_max, e_max):
    cases = full_corpus(s_max)
    (frames, keep, arrs), host, dev = tc.run_rule(hostsim_lib, pkg, cases, e_max, s_max)
    seen = set()
    for i, c in enumerate(cases):
        h = as_tuple(host[i])
        assert as_tuple(dev[i]) == h, i
        assert restated_tuple(tc.restated(orc_mod, c, frames[i], e_max, s_max)) == h, i
        if c["chain"] == 0 and "wire" in c:
            seen.add(host[i].outcome)
        if "weight" in c:                                     # crafted: AMBIGUOUS exactly from the distance on
            assert (host[i].outcome == rc.AMBIGUOUS) == (s_max >= c["weight"]), (i, s_max)
    assert {rc.REPAIRED, rc.UNREPAIRABLE, rc.NONE} <= seen
    if s_max >= 3:
        assert rc.AMBIGUOUS in seen


def test_every_outcome_occurs(hostsim_lib, pkg):
    """over the corpus at s_max 1 and 6 with e_max 1 and 3, the T1 rule and the erasure rule give every outcome (TOO_MANY:
    T1 frames without soft values; TRUNCATED: S1 aborts whose list ends before P)"""
    seen = set()
    for s_max in (1, 6):
        for e_max in (1, 3):
            cases = full_corpus(s_max)
            _, host, _ = tc.run_rule(hostsim_lib, pkg, cases, e_max, s_max)
            seen |= {host[i].outcome for i in range(len(cases))}
    assert seen == set(range(6)), seen


@pytest.mark.parametrize("s_max", [1, 2, 3, 6])
def test_wrong_symbols_among_the_searched_come_back(hostsim_lib, pkg, s_max):
    """every corpus telegram whose wrong symbols lie among its K searched ones (ML or runner-up the sent value), block by
    block, comes back as sent -- unless the erasure rule repaired it first or found it AMBIGUOUS, which stands"""
    synth = synth_mod()
    cases = [c for seed in (5, 6) for c in tc.corpus(synth, s_max, seed=seed)]
    _, host, _ = tc.run_rule(hostsim_lib, pkg, cases, 1, s_max)
    frames, keep = make_frames(pkg, cases)
    n = 0
    for i, c in enumerate(cases):
        if not tc.within_k(c, s_max):
            continue
        r0 = pkg.WmbRepaired()
        assert hostsim_lib.wmb_frame_repair(C.addressof(frames[i]), 1, C.addressof(r0)) == 0
        if r0.outcome == rc.AMBIGUOUS:
            continue
        n += 1
        assert host[i].outcome == rc.REPAIRED, (i, host[i].outcome)
        assert bytes(host[i].line.datagram[:host[i].line.len]) == c["sent"], i
    assert n >= 5, n


def test_erasure_outcomes_stand_and_other_frames_are_wmb_frame_repair(hostsim_lib, pkg):
    """frames the erasure rule repairs or finds AMBIGUOUS / TRUNCATED / NONE, C1 and S1 frames, s_max 0 and soft = NULL all
    give exactly wmb_frame_repair"""
    synth = synth_mod()
    cases = full_corpus(4) + planted_cases(synth, 2)
    frames, keep = make_frames(pkg, cases)
    arrs, ptrs = tc.soft_ptrs(cases)
    n_stand = 0
    for e_max, s_max, use_soft in ((1, 0, True), (3, 4, True), (2, 6, False), (1, 6, True)):
        for i in range(len(cases)):
            a, b = pkg.WmbRepaired(), pkg.WmbRepaired()
            assert hostsim_lib.wmb_frame_repair(C.addressof(frames[i]), e_max, C.addressof(a)) == 0
            assert hostsim_lib.wmb_frame_repair_t1_soft(C.addressof(frames[i]), ptrs[i] if use_soft else None, e_max,
                                                        s_max, C.addressof(b)) == 0
            if cases[i]["chain"] == 0 and use_soft and s_max and a.outcome in (rc.TOO_MANY, rc.UNREPAIRABLE) \
                    and arrs[i] is not None:
                continue                                      # possibly the soft rule
            n_stand += a.outcome in (rc.REPAIRED, rc.AMBIGUOUS)
            assert as_tuple(a) == as_tuple(b), (i, e_max, s_max)
    assert n_stand >= 20
    r = pkg.WmbRepaired()
    assert hostsim_lib.wmb_frame_repair_t1_soft(C.addressof(frames[0]), ptrs[0], 2, 7, C.addressof(r)) == -1
    assert hostsim_lib.wmb_frame_repair_t1_soft(C.addressof(frames[0]), ptrs[0], 4, 2, C.addressof(r)) == -1


def capture_manual_framing(lib, pkg, orc_mod, sigma=40.0):
    """a noisy T1 capture decoded with manual framing and soft values: K4S equals the host twin (and, given orc_mod, the
    restatement) on every polled candidate, and no repaired datagram differs from a sent one"""
    synth = synth_mod()
    ems = tc.t1_emitters(synth)[:3]
    cu8, plan = synth.synth_capture(4 << 20, emitters=ems, seed=0x7172, noise_sigma=sigma)
    cu8 = np.ascontiguousarray(cu8.numpy())
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1, soft_bits=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        soft = [ctx.frame_soft(arr[i]) for i in range(k)]
        dev = ctx.repair_frames(arr, k, 3, device=True, s_max=6, soft=soft)
        host = ctx.repair_frames(arr, k, 3, device=False, s_max=6, soft=soft)
        assert [as_tuple(dev[i]) for i in range(k)] == [as_tuple(host[i]) for i in range(k)]
        n_soft = 0
        for i in range(k):
            if host[i].outcome == rc.REPAIRED:
                assert bytes(host[i].line.datagram[:host[i].line.len]) in sent
            if orc_mod is not None and arr[i].chain == 0 and soft[i] is not None:
                w = np.ctypeslib.as_array(arr[i].bits, (arr[i].nbits,))
                c = dict(chain=0, bits=(w & 1).astype(np.uint8), rssi=((w >> 1) & 0xFF).astype(np.uint8), soft=soft[i])
                assert restated_tuple(tc.restated(orc_mod, c, arr[i], 3, 6)) == as_tuple(host[i]), i
                n_soft += 1
    return n_soft


def test_capture_manual_framing(hostsim_lib, pkg, orc_mod):
    assert capture_manual_framing(hostsim_lib, pkg, orc_mod) > 20


# ---- the streaming path -------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cap():
    return tc.t1_capture()


SETTINGS = [(0, 0), (0, 1), (0, 3), (0, 6), (4, 0), (4, 6)]


@pytest.fixture(scope="module")
def want(hostsim_lib, pkg, cap):
    return tc.restated_stream(pkg, hostsim_lib, cap[0], "-v", 2, SETTINGS)


@pytest.fixture(scope="module")
def runs(hostsim_lib, pkg, cap):
    """the capture in 1 MiB batches at e_max 2, with quality and bursts on, per (k_max, s_max)"""
    return {ks: tc.stream(pkg, hostsim_lib, cap[0], "-v", 2, quality=True, burst_level=(14, 14), repair_soft=ks[0],
                          repair_t1_soft=ks[1]) for ks in SETTINGS}


def t1_soft_records(recs):
    return [t for t in recs if t[-1]]


@pytest.mark.parametrize("ks", SETTINGS)
def test_records_equal_the_restatement(runs, want, ks):
    assert runs[ks][0] == want[ks]
    if ks[1]:
        assert sum(1 for t in t1_soft_records(runs[ks][0]) if t[4] == rc.REPAIRED) >= 10
    else:
        assert not t1_soft_records(runs[ks][0])


@pytest.mark.parametrize("ks,batching", [((0, 6), "one"), ((4, 3), "uneven"), ((0, 2), "uneven")])
def test_records_equal_the_restatement_other_batchings(hostsim_lib, pkg, cap, ks, batching):
    got = tc.stream(pkg, hostsim_lib, cap[0], "-v", 2, batching, batch_mib=8 if batching == "one" else 1,
                    repair_soft=ks[0], repair_t1_soft=ks[1])[0]
    assert got == tc.restated_stream(pkg, hostsim_lib, cap[0], "-v", 2, [ks])[ks]


def test_weak_t1_telegrams_come_back_as_sent(runs, cap):
    _, plan, ems = cap
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    weak = {ems[p.emitter].payload(p.k): p for p in plan if ems[p.emitter].weak_flips and ems[p.emitter].mode == "T1"}
    alone = {d for d, p in weak.items()
             if not any(q is not p and q.start_iq < p.start_iq + p.n_iq and p.start_iq < q.start_iq + q.n_iq for q in plan)}
    assert len(alone) >= 10
    for ks in SETTINGS:
        got = {t[-2] for t in runs[ks][0] if t[4] == rc.REPAIRED}
        assert got <= sent, "a repaired datagram that was never sent"
        if ks[1] >= 3:
            assert alone <= got, (ks, len(alone - got))


def test_off_means_off_and_nothing_else_moves(runs):
    """s_max 0: the records, launches and copies of the parent's settings.  Any s_max: the non-T1-soft records, lines,
    records, bursts and statistics but kernel_launches (+2 per gather when no soft rule was on) and d2h_bytes stay"""
    for k in (0, 4):
        recs0, lines0, info0, qual0, bursts0, st0 = runs[(k, 0)]
        for ks in SETTINGS:
            if ks[0] != k or not ks[1]:
                continue
            recs, lines, info, qual, bursts, st = runs[ks]
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
            assert st.kernel_launches - st0.kernel_launches == (0 if k else 2 * (st.batches + 1))
            assert st.d2h_bytes >= st0.d2h_bytes


def test_off_is_the_parent_path(hostsim_lib, pkg, cap):
    """s_max 0 set explicitly: launches and copies equal a context that never heard of the setting"""
    a = tc.stream(pkg, hostsim_lib, cap[0], "-v", 2)
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, max_batch_mib=1) as ctx:
        ctx.set_repair_t1_soft(3)
        ctx.set_repair_t1_soft(0)
        recs = []
        for lo, hi in rs.pushes(len(cap[0]), "1mib"):
            ctx.push(cap[0].ctypes.data + lo, hi - lo)
            recs += ctx.take_repairs()
        ctx.poll_flush()
        recs = [tc.record_tuple(r) for r in recs + ctx.take_repairs()]
        st = ctx.stats()
    assert recs == a[0]
    assert (st.kernel_launches, st.d2h_bytes) == (a[5].kernel_launches, a[5].d2h_bytes)


def test_time_chunks_merge_to_the_sequential_records(hostsim_lib, pkg, runs, cap):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = cap[0]
    parts = []
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_t1_soft=6, max_batch_mib=1) as ctx:
        def push(lo, hi):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
        for rank in range(3):
            out, _ds, _de, _start = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, repairs=True)
            parts.append(out[-1])
    assert [tc.record_tuple(r) for r in shard.merge_repairs(parts)] == runs[(0, 6)][0]


def test_setter_and_boundary_state(hostsim_lib, pkg, cap):
    lib = hostsim_lib
    cu8 = cap[0]
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 7) == -1
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 6) == 0
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 1) != 0 and b"after samples were pushed" in lib.wmb_last_error()
        ctx.reset()
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 2) == 0
        ctx.seek(0)
        assert lib.wmb_set_repair_t1_soft(ctx._ctx, 0) == 0
    digests = {}
    for ks in ((0, 0), (0, 1), (0, 6), (1, 0), (6, 0), (4, 0), (4, 4)):
        with pkg.WmbusB200("-v", lib=lib, repair=2, repair_soft=ks[0], repair_t1_soft=ks[1], max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, 3 * rs.MIB)
            digests[ks] = ctx.boundary_state()
    assert len({hashlib.sha256(v).digest() for v in digests.values()}) == len(digests)
    for ks in ((0, 1), (0, 6), (4, 4)):                       # s_max appended: the bytes before it are unchanged
        base = digests[(ks[0], 0)]
        assert digests[ks][:len(base)] == base and len(digests[ks]) == len(base) + 5


def test_cli_repaired_file(hostsim_lib, pkg, cap, tmp_path):
    cu8 = cap[0]
    path = tmp_path / "repaired.txt"
    plain = cli(["-v"], cu8, {})
    assert plain.returncode == 0, plain.stderr
    r = cli(["-v"], cu8, {"WMBUS_B200_REPAIRED": str(path), "WMBUS_B200_REPAIR_ERASURES": "2",
                          "WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "4"})
    assert r.returncode == 0, r.stderr
    assert r.stdout == plain.stdout or [blank_ts(l, True) for l in r.stdout.decode().splitlines()] == \
        [blank_ts(l, True) for l in plain.stdout.decode().splitlines()]
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_t1_soft=4, max_batch_mib=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        recs = ctx.take_repairs()
        want = [ctx.repaired_line(x, b"rla;" if x.algo == 0 else b"t2a;") for x in recs if x.repair.outcome == rc.REPAIRED]
        n_soft = sum(1 for x in recs if x.soft_t1 and x.repair.outcome == rc.REPAIRED)
    got = [blank_ts(l, True) for l in path.read_text().splitlines()]
    assert got == want and n_soft >= 10


@pytest.mark.parametrize("env", [{"WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "2"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "0"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "7"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "x"}])
def test_cli_bad_setting_fails_at_start_up(hostsim_lib, tmp_path, env):
    env = {k: v.replace("{tmp}", str(tmp_path / "r.txt")) for k, v in env.items()}
    r = cli(["-v"], np.zeros(8192, np.uint8), env)
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS" in r.stderr, r.stderr
