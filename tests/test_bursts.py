"""`not gpu`: the burst report (wmb_set_bursts / wmb_take_bursts) on the CPU-simulation build of the library (the
kernels' phase functions): every record against the numpy restatement on the oracle's stages (tests/burst_cases.py),
the cut grid, time chunks, coverage of the decoded lines, a planted emitter too far off to decode, off means off,
setter errors and the CLI's record file."""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import burst_cases as bc
import line_info_cases as lc
import orc
import receiver_cases as rc
from conftest import ROOT

CAPTURES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls]


@pytest.mark.parametrize("name,flags", CAPTURES, ids=[f"{n}|{f}" for n, f in CAPTURES])
def test_parity_committed(hostsim_lib, pkg, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        bc.check_parity(pkg, hostsim_lib, cu8, flags, max_batch_mib=mib)


@pytest.mark.parametrize("flags", ["-v -a", "-v -p T", "-v -p S", "-v -t 0 -r 0"])
def test_parity_flags(hostsim_lib, pkg, flags):
    want, recs = bc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_1m6.cu8"), flags, max_batch_mib=1)
    assert len(want) > 5
    if "-a" in flags:
        assert not recs["valid"].any() and np.isnan(recs["offset_hz"]).all()
    else:
        gains = lc.fir_gains()
        for r in recs:
            assert r["valid"] and abs(r["offset_hz"] - lc.offset_hz(r, gains[r["chain"]])) <= 1e-9 * max(1.0, abs(r["offset_hz"]))


def test_remove_dc_changes_nothing(hostsim_lib, pkg):
    """-o acts behind the tap the report reads: the same bursts"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    _, a, _ = bc.product_bursts(pkg, hostsim_lib, cu8, "-v", bc.DEFAULT_LEVEL, max_batch_mib=1)
    _, b, _ = bc.product_bursts(pkg, hostsim_lib, cu8, "-v -o", bc.DEFAULT_LEVEL, max_batch_mib=1)
    assert len(a) > 5 and np.array_equal(a, b)


def test_parity_prefilter_and_levels(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    bc.check_parity(pkg, hostsim_lib, cu8, "-v", max_batch_mib=1, prefilter=1)
    for level in ((1, 0), (0, 3), (60, 90), (255, 255)):
        bc.check_parity(pkg, hostsim_lib, cu8, "-v", level, max_batch_mib=1)


def test_parity_odd_pushes(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    bc.check_parity(pkg, hostsim_lib, cu8, "-v", pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777])
    bc.check_parity(pkg, hostsim_lib, cu8, "-v", (8, 8), pushes=[4096] * 40 + [100000, 3])
    cu8 = rc.cached_capture("excerpt_issue48_2m4.cu8")
    bc.check_parity(pkg, hostsim_lib, cu8, "-v -d 3 -s", pushes=[4096 * 3] * 20)


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the records do not depend on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, burst_cases as bc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "bc.check_parity(pkg, lib, rc.cached_capture('synth_mixed_1m6.cu8'), '-v', (8, 8), max_batch_mib=1);"
            "bc.check_parity(pkg, lib, rc.cached_capture('excerpt_samples2_a.cu8'), '-v', (5, 5), max_batch_mib=1);"
            "cu8, _ = bc.cw_capture(4 << 20); bc.check_parity(pkg, lib, cu8, '-v', max_batch_mib=1)"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


def test_cw_cut_grid(hostsim_lib, pkg):
    """an in-band carrier over 60 % of a 4 MiB capture (~6 spans of 2^17): cut on the 2^16 grid from 2^17 after its
    start, continued / cut flags; at 1 and 256 MiB batches"""
    cu8, _ = bc.cw_capture(4 << 20)
    for mib in (1, 256):
        want, recs = bc.check_parity(pkg, hostsim_lib, cu8, "-v", max_batch_mib=mib)
    for ch in (0, 1):
        r = recs[recs["chain"] == ch]
        long = r[r["end_sample"] - r["start_sample"] > 20000]
        assert len(long) >= 5, (ch, len(long))
        first, rest = long[0], long[1:]
        assert first["flags"] == bc.CUT and first["end_sample"] % bc.P == 0
        assert first["end_sample"] - first["start_sample"] >= bc.Q
        assert (rest["start_sample"] % bc.P == 0).all() and (rest["flags"] & bc.CONTINUED).all()
        assert (rest["flags"][:-1] == bc.CONTINUED | bc.CUT).all() and not rest["flags"][-1] & bc.CUT
        assert (rest["end_sample"][:-1] - rest["start_sample"][:-1] == bc.P).all()
        # the carrier's offset: a 20 kHz tone
        assert abs(np.median(long["offset_hz"]) - 20e3) < 500


def test_telegram_across_grid_not_cut(hostsim_lib, pkg):
    """a telegram that straddles a multiple of 2^16 is one piece"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    _, recs, _ = bc.product_bursts(pkg, hostsim_lib, cu8, "-v", bc.DEFAULT_LEVEL, max_batch_mib=1)
    straddle = [r for r in recs if r["start_sample"] // bc.P != (r["end_sample"] - 1) // bc.P]
    assert straddle
    assert all(r["flags"] == 0 for r in recs)


@pytest.mark.parametrize("seek", [False, True])
def test_clipped_at_stream_start(hostsim_lib, pkg, seek):
    """a capture cut inside a telegram: the samples before the first one pushed (or before the seek) are below"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    first = [w for w in bc.oracle_bursts(cu8, "-v", bc.DEFAULT_LEVEL) if w[1] - w[0] > 2100 and w[0] > 20000][0]
    cut_m = -(-(first[0] + 1) // 1024) * 1024
    assert first[0] < cut_m < first[1]
    part = np.ascontiguousarray(cu8[cut_m * 4:])
    base = cut_m if seek else 0
    want = bc.oracle_bursts(part, "-v", bc.DEFAULT_LEVEL, m0=base)
    assert want[0][0] - base < 64                   # the telegram in progress starts right at the first sample pushed
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL) as ctx:
        if seek:
            ctx.push(cu8.ctypes.data, 1 << 20)      # something before the seek, which it forgets
            ctx.take_bursts()
            ctx.seek(cut_m * 2)
        ctx.process(part.ctypes.data, len(part), flush=True)
        got = bc.as_tuples(ctx.take_bursts())
    assert got == want


def test_sample_index_wrap(hostsim_lib, pkg):
    """a stream positioned just below 2^40 decimated samples decodes across the wrap; the cut grid stays the grid"""
    cu8, _ = bc.cw_capture(4 << 20)
    m_total = len(cu8) // 4
    for back in (2048 * 20, (m_total // 2) // 2048 * 2048):
        first_m = (1 << 40) - back
        want = bc.oracle_bursts(cu8, "-v", bc.DEFAULT_LEVEL, m0=first_m)
        for step in (len(cu8), 1 << 19):
            with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL) as ctx:
                ctx.seek(first_m * 2)
                got = []
                for off in range(0, len(cu8), step):
                    ctx.push(cu8.ctypes.data + off, min(step, len(cu8) - off))
                    got.append(ctx.take_bursts())
                ctx.poll_flush()
                got.append(ctx.take_bursts())
            assert bc.as_tuples(np.concatenate(got)) == want
            assert max(w[1] for w in want) > (1 << 40)


def time_chunks(pkg, lib, cu8, flags, level, world=3):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    parts = []
    for rank in range(world):
        with pkg.WmbusB200(flags, lib=lib, max_batch_mib=1, burst_level=level) as ctx:
            push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
            (lines, b), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, world, 1 << 18, bursts=True)
        parts.append(b)
    return shard.merge_bursts(parts), parts


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks: the merged bursts equal the sequential run's -- also with a carrier across a chunk border"""
    for cu8, level in ((rc.cached_capture("synth_mixed_1m6.cu8"), (8, 8)), (bc.cw_capture(8 << 20)[0], bc.DEFAULT_LEVEL)):
        _, seq, _ = bc.product_bursts(pkg, hostsim_lib, cu8, "-v", level, max_batch_mib=1)
        merged, parts = time_chunks(pkg, hostsim_lib, cu8, "-v", level)
        assert all(len(p) for p in parts)
        assert np.array_equal(merged, seq)


def test_coverage_of_decoded_lines(hostsim_lib, pkg):
    """at the default level every CRC-ok line's access-code match lies inside a burst of its chain"""
    for name, fls in list(rc.COMMITTED.items()):
        cu8 = rc.cached_capture(name)
        flags = fls[0]
        with pkg.WmbusB200(flags, lib=hostsim_lib, burst_level=bc.DEFAULT_LEVEL) as ctx:
            lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            b = ctx.take_bursts()
        ok = recs[recs["crc_ok"] == 1]
        for r in ok:
            mine = b[b["chain"] == r["chain"]]
            assert ((mine["start_sample"] <= r["sync_sample"]) & (r["sync_sample"] < mine["end_sample"])).any(), (name, r)


def test_far_off_emitter(hostsim_lib, pkg):
    """a T1 meter 60 kHz above the tuned carrier decodes nowhere (the oracle prints none of its telegrams), but its
    bursts are reported with its offset; retuned by that offset, its telegrams decode with CRC ok"""
    em, far = bc.planted_emitters(60e3)
    cu8, plan = bc.planted_capture(em)
    want = [orc.blank_ts(l) for l in orc.run_lines(cu8, orc.opts_from_flags("-v"))]
    assert want and not any(f"{far.ident:08X}" in l for l in want)
    errs, skipped, far_mean = bc.check_planted(pkg, hostsim_lib, cu8, em, plan, far)
    assert skipped <= 20                             # measured: 13 of 58 overlap another emitter's telegram
    cu8b, _ = bc.planted_capture(em, center_shift_hz=-far_mean)
    with pkg.WmbusB200("-v", lib=hostsim_lib) as ctx:
        lines = ctx.process(cu8b.ctypes.data, len(cu8b), flush=True)
    mine = [l for l in lines if f"{far.ident:08X}" in l]
    ok = [l for l in mine if l.split(";")[2] == "1"]
    assert len(ok) >= 5 and 2 * len(ok) >= len(mine), (len(ok), len(mine))   # the rest collide with other telegrams


def test_off_means_off(hostsim_lib, pkg):
    """no level: the same lines, line records, kernel launches and D2H bytes as a context that never heard of bursts;
    wmb_take_bursts hands out nothing"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = []
    for level in (None, (0, 0)):
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=level) as ctx:
            lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            st = ctx.stats()
            b = ctx.take_bursts()
        out.append((lines, recs, st.kernel_launches, st.d2h_bytes, len(b)))
    (l0, r0, k0, d0, n0), (l1, r1, k1, d1, n1) = out
    assert l0 == l1 and np.array_equal(r0, r1) and k0 == k1 and d0 == d1 and n0 == n1 == 0
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=bc.DEFAULT_LEVEL) as ctx:
        lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
        st = ctx.stats()
    assert lines == l0 and np.array_equal(recs, r0) and st.kernel_launches > k0


def test_setter_rules(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        assert L.wmb_set_bursts(ctx._ctx, 2, 10) == -1
        assert L.wmb_set_bursts(ctx._ctx, -1, 10) == -1
        assert L.wmb_set_bursts(ctx._ctx, 0, 256) == -1
        assert L.wmb_set_bursts(ctx._ctx, 1, 255) == 0
        ctx.set_bursts(0, bc.DEFAULT_LEVEL[0])
        ctx.set_bursts(1, bc.DEFAULT_LEVEL[1])
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert L.wmb_set_bursts(ctx._ctx, 0, 20) == -6          # after a push
        n = C.c_size_t(7)
        assert L.wmb_take_bursts(ctx._ctx, None, 0, C.byref(n)) == 0 and n.value == 0
        ctx.reset()                                              # the level survives reset
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        a = ctx.take_bursts()
        ctx.seek(0)
        ctx.set_bursts(0, 0)                                     # allowed again after a seek
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        b = ctx.take_bursts()
    want = bc.oracle_bursts(cu8, "-v", bc.DEFAULT_LEVEL)
    assert bc.as_tuples(a) == want
    assert bc.as_tuples(b) == [w for w in want if w[6] == 1]


def test_partial_take(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L, burst_level=bc.DEFAULT_LEVEL) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        r = np.zeros(8, pkg.burst_dtype())
        n = C.c_size_t(0)
        assert L.wmb_take_bursts(ctx._ctx, r.ctypes.data, 3, C.byref(n)) == 0 and n.value == 3
        rest = ctx.take_bursts()
    want = bc.oracle_bursts(cu8, "-v", bc.DEFAULT_LEVEL)
    assert bc.as_tuples(r[:3]) + bc.as_tuples(rest) == want


def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def expected_file(recs):
    out = []
    for r in recs:
        off = f"{r['offset_hz']:.0f}" if r["valid"] else "nan"
        mean = r["rssi_sum"] / (r["end_sample"] - r["start_sample"])
        out.append(f"{'T1C1' if r['chain'] == 0 else 'S1'};{r['start_sample']};{r['end_sample']};{r['peak']};{mean:.1f};"
                   f"{r['carrier_hz']:.0f};{off};{r['flags']}")
    return out


def check_cli(run, pkg, lib, tmp_path, flags, cu8, level_env=None, level=bc.DEFAULT_LEVEL):
    path = tmp_path / "bursts.txt"
    env = {"WMBUS_B200_BURSTS": str(path)}
    if level_env:
        env["WMBUS_B200_BURST_LEVEL"] = level_env
    r1 = run(env, cu8.tobytes(), flags)
    r0 = run({}, cu8.tobytes(), flags)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout) and len(blank(r0.stdout)) > 5
    with pkg.WmbusB200(flags, lib=lib, burst_level=level) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        recs = ctx.take_bursts()
    got = path.read_text().splitlines()
    assert got == expected_file(recs) and len(got) > 5


@pytest.mark.parametrize("flags", ["-v", "-d 3 -s"])
def test_cli_bursts(hostsim_lib, pkg, tmp_path, flags):
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "synth_mixed_1m6.cu8")
    check_cli(_cli, pkg, hostsim_lib, tmp_path, flags, cu8)
    check_cli(_cli, pkg, hostsim_lib, tmp_path, flags, cu8, "9,0", (9, 0))


@pytest.mark.parametrize("env", [{"WMBUS_B200_BURSTS": "/nonexistent-dir/x/bursts.txt"},
                                 {"WMBUS_B200_BURSTS": "@TMP", "WMBUS_B200_BURST_LEVEL": "256"},
                                 {"WMBUS_B200_BURSTS": "@TMP", "WMBUS_B200_BURST_LEVEL": "x"},
                                 {"WMBUS_B200_BURSTS": "@TMP", "WMBUS_B200_BURST_LEVEL": "10,"}])
def test_cli_bad_settings(hostsim_lib, tmp_path, env):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    e = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    e.update({k: (str(tmp_path / "b.txt") if v == "@TMP" else v) for k, v in env.items()})
    # stdin stays open and empty: a program that read it would wait here
    p = subprocess.Popen([exe, "-v"], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e)
    try:
        rc_ = p.wait(timeout=120)
        out, err = p.stdout.read(), p.stderr.read()
    finally:
        if p.poll() is None:
            p.kill()
        p.stdin.close()
    assert rc_ == 1 and out == b"" and b"WMBUS_B200_BURST" in err
