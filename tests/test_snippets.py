"""`not gpu`: burst snippets (wmb_set_snippets / wmb_take_snippets) on the CPU-simulation build of the library: every
record and its bytes against the restatement (tests/snippet_cases.py) over captures, flags, batch sizes, pushes, thread
orders and seeks; no granule missing (the keep lemma); mode 2's decisions; the replay contract; off means off; time
chunks; the overflow knob; setter rules; the CLI's files."""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import burst_cases as bc
import orc
import receiver_cases as rc
import snippet_cases as sc
from conftest import ROOT

CAPTURES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls]


@pytest.mark.parametrize("name,flags", CAPTURES, ids=[f"{n}|{f}" for n, f in CAPTURES])
def test_parity_committed(hostsim_lib, pkg, name, flags):
    cu8 = rc.cached_capture(name)
    for mode in (1, 2):
        sc.check_parity(pkg, hostsim_lib, cu8, flags, mode, max_batch_mib=1)


@pytest.mark.parametrize("flags", ["-v -s", "-v -p S", "-v -p T", "-v -o", "-v -a"])
def test_parity_flags(hostsim_lib, pkg, flags):
    recs, *_ = sc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_1m6.cu8"), flags, 1, max_batch_mib=1)
    if "-s" not in flags:
        assert len(recs) >= 5


def test_parity_batches_and_pushes(hostsim_lib, pkg):
    """one batch, 1 MiB and 256 MiB batches, ragged host pushes; the records and bytes do not depend on the cut"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    runs = [sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1, max_batch_mib=mib)[:2] for mib in (1, 256)]
    runs.append(sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1, pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777],
                                max_batch_mib=1)[:2])
    runs.append(sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1, pushes=[4096] * 40 + [100000, 3], max_batch_mib=1)[:2])
    for r, d in runs[1:]:
        assert sc.as_tuples(r) == sc.as_tuples(runs[0][0]) and d == runs[0][1]
    cu8 = rc.cached_capture("excerpt_issue48_2m4.cu8")
    sc.check_parity(pkg, hostsim_lib, cu8, "-v -d 3 -s", 1, (8, 8), pushes=[4096 * 3] * 20)


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the snippets do not depend on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, snippet_cases as sc, burst_cases as bc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "sc.check_parity(pkg, lib, rc.cached_capture('synth_mixed_1m6.cu8'), '-v', 1, (8, 8), max_batch_mib=1);"
            "cu8, _ = bc.cw_capture(4 << 20); sc.check_parity(pkg, lib, cu8, '-v', 1, max_batch_mib=1)"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.parametrize("seek", [2048 * 2 * 37, (1 << 41) + 2048 * 2 * 5])
def test_seek(hostsim_lib, pkg, seek):
    """a capture pushed after wmb_seek: snippets carry capture positions; far past 2^41 IQ samples too"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    recs, *_ = sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1, seek=seek, max_batch_mib=1)
    assert len(recs) >= 5 and recs["start_iq"].min() >= seek


def test_clipped_at_both_ends(hostsim_lib, pkg):
    """a capture cut inside a telegram: the first snippet starts at the first granule pushed; a capture whose end is a
    partial granule (-d 3, a multiple of 4096 bytes but not of 12288, and a ragged tail the reference drops)"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    first = [w for w in bc.oracle_bursts(cu8, "-v", bc.DEFAULT_LEVEL) if w[1] - w[0] > 2100 and w[0] > 20000][0]
    cut_g = first[0] // 2048 + 1
    assert first[0] < cut_g * 2048 < first[1]
    part = np.ascontiguousarray(cu8[cut_g * 8192:])
    recs, *_ = sc.check_parity(pkg, hostsim_lib, part, "-v", 1, seek=cut_g * 4096, max_batch_mib=1)
    assert recs["start_iq"][0] == cut_g * 4096
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8")
    n = len(cu8) // 12288 * 12288 - 12288 + 8192 + 1000
    recs, data, *_ = sc.check_parity(pkg, hostsim_lib, np.ascontiguousarray(cu8[:n]), "-v -d 3 -s", 1, max_batch_mib=1)
    assert len(recs)


def test_cw_carrier_cut(hostsim_lib, pkg):
    """an in-band carrier over 60 % of a 4 MiB capture, cut into pieces on the 2^16 grid: every granule kept"""
    cu8, _ = bc.cw_capture(4 << 20)
    for mib in (1, 256):
        recs, *_ = sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1, max_batch_mib=mib)
        assert (recs["flags"] & bc.CUT).sum() >= 3 and (recs["lost"] == 0).all()


def test_mode2_far_off_meter(hostsim_lib, pkg):
    """mode 2: the in-tune T1 meter's bursts are not saved, the meter 60 kHz off (which nothing decodes) is"""
    em, far = bc.planted_emitters()
    cu8, plan = bc.planted_capture(em)
    recs, data, lines, info, bursts = sc.check_parity(pkg, hostsim_lib, cu8, "-v", 2)
    fi = em.index(far)

    def hits(ei):
        return [r for r in recs if any(p.emitter == ei and p.start_iq < int(r["end_sample"]) * 2
                                       and p.start_iq + p.n_iq > int(r["start_sample"]) * 2 for p in plan)]
    assert len(hits(fi)) >= 5
    ok = [int(r["sync_sample"]) for r in info if r["crc_ok"] and r["chain"] == 0]
    assert ok and not any(r["start_sample"] <= m < r["end_sample"] for r in recs if r["chain"] == 0 for m in ok)
    assert (recs["decoded"] == 0).all()


def test_mode2_with_repair(hostsim_lib, pkg):
    """`decoded` joins the repair records too when repair is on"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    for mode in (1, 2):
        sc.check_parity(pkg, hostsim_lib, cu8, "-v", mode, repair=2, repair_t1_soft=2, max_batch_mib=1)


def test_waits_for_telegram_in_flight(hostsim_lib, pkg):
    """a run-length telegram cut by dead air waits for the next edge: its burst is handed out by the burst report, but
    its snippet only once pending_before clears"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1) as ctx:
        lines, info = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    r = [x for l, x in zip(lines, info) if x["crc_ok"] and x["chain"] == 0 and l.startswith("rla;")][0]
    mid = (int(r["sync_sample"]) + int(r["end_sample"])) // 2
    cut = mid * 4 // 4096 * 4096
    dead = np.full(1 << 20, 127, np.uint8)
    cap = np.ascontiguousarray(np.concatenate([cu8[:cut], dead, cu8[cut:]]))
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL, snippets=1) as ctx:
        ctx.push(cap.ctypes.data, cut + len(dead))
        b = ctx.take_bursts()
        piece = [x for x in b if x["chain"] == 0 and x["start_sample"] <= r["sync_sample"] < x["end_sample"]]
        assert piece and ctx.pending_before(int(piece[0]["end_sample"])) > 0
        early, _ = ctx.take_snippets()
        assert not any(x["start_sample"] == piece[0]["start_sample"] and x["chain"] == 0 for x in early)
        ctx.push(cap.ctypes.data + cut + len(dead), len(cap) - cut - len(dead))
        ctx.poll_flush()
        late, _ = ctx.take_snippets()
    x = [x for x in late if x["start_sample"] == piece[0]["start_sample"] and x["chain"] == 0]
    assert len(x) == 1


def test_replay(hostsim_lib, pkg):
    """every CRC-ok line's piece, replayed into a fresh context after wmb_seek(start_iq) -- and without a seek -- gives
    the line with its text and sync_sample, over the replay corpus"""
    total = 0
    for name, flags in sc.CORPUS:
        cu8 = sc.s_capture() if name == "s_capture" else rc.cached_capture(name)
        n = sc.check_replay(pkg, hostsim_lib, cu8, flags, max_batch_mib=1)
        if "-s" in flags:
            assert sc.check_replay(pkg, hostsim_lib, cu8, flags, seek=False, max_batch_mib=1) == n
        total += n
    assert total >= 60


def test_off_means_off(hostsim_lib, pkg):
    """mode 0 is a context that never heard of snippets; with snippets on, lines, line records, bursts and statistics are
    the same but kernel launches and D2H bytes"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = []
    for mode in (None, 0, 1, 2):
        kw = {} if mode is None else dict(snippets=mode)
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL, **kw) as ctx:
            lines, info = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            b = ctx.take_bursts()
            s, _ = ctx.take_snippets()
            st = ctx.stats()
        out.append((lines, info, b, s, st))
    base = out[0]
    for mode, (lines, info, b, s, st) in zip((None, 0, 1, 2), out):
        assert lines == base[0] and np.array_equal(info, base[1]) and np.array_equal(b, base[2])
        for f, _ in st._fields_:
            if f in ("kernel_launches", "d2h_bytes") or f.endswith("_ms"):
                continue
            assert getattr(st, f) == getattr(base[4], f) if not hasattr(getattr(st, f), "__len__") else \
                list(map(list, getattr(st, f))) == list(map(list, getattr(base[4], f))), f
        if mode:
            assert len(s) and st.kernel_launches == base[4].kernel_launches + 5 * st.batches
            assert st.d2h_bytes > base[4].d2h_bytes
        else:
            assert not len(s) and st.kernel_launches == base[4].kernel_launches and st.d2h_bytes == base[4].d2h_bytes


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks in mode 1 merge to the sequential snippets; merge_snippets(undecoded=True) gives mode 2's"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    seq = {m: sc.product(pkg, hostsim_lib, cu8, "-v", m, max_batch_mib=1) for m in (1, 2)}
    parts, infos = [], []
    for rank in range(3):
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL, snippets=1) as ctx:
            out, *_ = shard.decode_time_chunk(ctx, lambda a, b: ctx.push(cu8.ctypes.data + a, b - a), len(cu8), 2, rank,
                                              3, info=True, bursts=True, snippets=True)
        infos.append(out[1])
        parts.append(out[3])
    info = np.concatenate(infos)
    for m, undec in ((1, False), (2, True)):
        r, d = shard.merge_snippets(parts, info, undecoded=undec)
        assert sc.as_tuples(r) == sc.as_tuples(seq[m][0]) and d == seq[m][1]


def test_overflow_knob(hostsim_lib, pkg):
    """opts.reserved[1] bit 2: one granule per slot; snippets that lost a granule come out with lost = 1 and no bytes,
    and their batches count as overflow batches"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    recs, data, lines, info, bursts, reps, st = sc.product(pkg, hostsim_lib, cu8, "-v", 1, max_batch_mib=1,
                                                           reserved=(C.c_uint32 * 2)(0, 4))
    want = sc.restate(cu8, 2, bursts, sc.matches_ok(info), 1)
    assert len(recs) == len(want) and recs["lost"].all() and (recs["nbytes"] == 0).all() and not any(data)
    assert [t[:3] + t[4:7] for t in sc.as_tuples(recs)] == [w[0][:3] + w[0][4:7] for w in want]
    assert st.overflow_batches >= 1
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        assert ctx.stats().overflow_batches == 0


def test_setter_rules(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        assert L.wmb_set_snippets(ctx._ctx, 3) == -1 and L.wmb_set_snippets(ctx._ctx, -1) == -1
        ctx.set_snippets(1)
        assert L.wmb_push(ctx._ctx, cu8.ctypes.data, 1 << 20) == -6          # no chain has bursts on
        ctx.set_bursts(1, 14)
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert L.wmb_set_snippets(ctx._ctx, 2) == -6                         # after a push
        assert L.wmb_set_snippets(ctx._ctx, 7) == -1                         # the mode is checked first
        ctx.reset()                                                          # the mode survives reset
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        a, _ = ctx.take_snippets()
        ctx.seek(0)
        ctx.set_snippets(2)                                                  # allowed again after a seek
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        b, _ = ctx.take_snippets()
    assert len(a) and (a["chain"] == 1).all() and len(b) < len(a)


def test_partial_take(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want, wdata, *_ = sc.product(pkg, L, cu8, "-v", 1)
    with pkg.WmbusB200("-v", lib=L, burst_level=bc.DEFAULT_LEVEL, snippets=1) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        r = np.zeros(8, pkg.snippet_dtype())
        buf = np.zeros(1 << 20, np.uint8)
        n = C.c_size_t(0)
        assert L.wmb_take_snippets(ctx._ctx, r.ctypes.data, 3, buf.ctypes.data, len(buf), C.byref(n)) == 0 and n.value == 3
        got = [buf[:int(r["nbytes"][:3].sum())].tobytes()]
        small = int(want["nbytes"][3]) + int(want["nbytes"][4]) - 1                   # the fifth does not fit
        assert L.wmb_take_snippets(ctx._ctx, r[3:].ctypes.data, 5, buf.ctypes.data,
                                   small, C.byref(n)) == 0 and n.value == 1
        got.append(buf[:int(r["nbytes"][3])].tobytes())
        rest, rdata = ctx.take_snippets()
    assert sc.as_tuples(r[:4]) + sc.as_tuples(rest) == sc.as_tuples(want)
    assert b"".join(got) + b"".join(rdata) == b"".join(wdata)


def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def check_cli(run, pkg, lib, tmp_path, flags, cu8, mode_env):
    """the files and the index equal take_snippets(); each file piped back prints its burst's lines"""
    mode = {None: 2, "undecoded": 2, "all": 1}[mode_env]
    out = tmp_path / f"snip-{mode_env}-{flags.replace(' ', '')}"
    out.mkdir()
    env = {"WMBUS_B200_SNIPPETS": str(out)}
    if mode_env:
        env["WMBUS_B200_SNIPPET_MODE"] = mode_env
    r1 = run(env, cu8.tobytes(), flags)
    r0 = run({}, cu8.tobytes(), flags)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda txt: [orc.blank_ts(l) for l in txt.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout)
    recs, data, lines, info, *_ = sc.product(pkg, lib, cu8, flags, mode, max_batch_mib=64)
    chain = lambda r: "T1C1" if r["chain"] == 0 else "S1"
    names = [f"{int(r['start_iq']):014d}_{chain(r)}.cu8" for r in recs]
    want = [f"{nm};{chain(r)};{r['start_sample']};{r['end_sample']};{r['start_iq']};{r['nbytes']};{r['decoded']}"
            for nm, r in zip(names, recs)]
    assert (out / "snippets.txt").read_text().splitlines() == want and len(want) >= 3
    last = {nm: d for nm, d in zip(names, data)}                 # pieces with the same START_IQ share a file
    for nm, d in last.items():
        assert (out / nm).read_bytes() == d
    if mode == 1:
        for nm, r in zip(names, recs):
            m = [orc.blank_ts(l) for l, x in zip(lines, info) if x["crc_ok"] and x["chain"] == r["chain"]
                 and r["start_sample"] <= x["sync_sample"] < r["end_sample"]]
            if m:
                got = blank(run({}, (out / nm).read_bytes(), flags).stdout)
                assert all(l in got for l in m), (nm, m, got)


@pytest.mark.parametrize("flags,mode", [("-v", None), ("-v", "all"), ("-d 3 -s", "all")])
def test_cli_snippets(hostsim_lib, pkg, tmp_path, flags, mode):
    if "-d 3" in flags:
        cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8")
    else:
        em, _ = bc.planted_emitters()
        cu8, _ = bc.planted_capture(em, n_bytes=4 << 20)
    check_cli(_cli, pkg, hostsim_lib, tmp_path, flags, cu8, mode)


@pytest.mark.parametrize("env", [{"WMBUS_B200_SNIPPETS": "/nonexistent-dir/x"},
                                 {"WMBUS_B200_SNIPPETS": "@TMP", "WMBUS_B200_SNIPPET_MODE": "some"},
                                 {"WMBUS_B200_SNIPPET_MODE": "all"}])
def test_cli_bad_settings(hostsim_lib, tmp_path, env):
    """start-up failures: nothing read, nothing printed, EXIT_FAILURE"""
    env = {k: (str(tmp_path) if v == "@TMP" else v) for k, v in env.items()}
    r = _cli(env, rc.cached_capture("synth_mixed_1m6.cu8").tobytes())
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_SNIPPET" in r.stderr
