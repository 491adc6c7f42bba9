"""`not gpu`: per-line carrier offsets (wmb_take_lines_info) on the CPU-simulation build of the library (the kernels'
phase functions): every line's (sync_sample, n, sum) against the oracle restatement (tests/line_info_cases.py), planted
offsets, clipping, the 2^40 sample wrap, time chunks, manual framing, partial takes and the CLI's record file."""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import line_info_cases as lc
import orc
import receiver_cases as rc
from conftest import ROOT

CAPTURES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls]


@pytest.mark.parametrize("name,flags", CAPTURES, ids=[f"{n}|{f}" for n, f in CAPTURES])
def test_parity_committed(hostsim_lib, pkg, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        lc.check_parity(pkg, hostsim_lib, cu8, flags, max_batch_mib=mib)


@pytest.mark.parametrize("flags", ["-v", "-v -o", "-v -p T", "-v -a", "-v -t 0 -a"])
def test_parity_flags(hostsim_lib, pkg, flags):
    want, recs = lc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_1m6.cu8"), flags, max_batch_mib=1)
    assert len(want) > 5
    if "-a" in flags:
        assert not recs["valid"].any() and np.isnan(recs["offset_hz"]).all()
    else:
        assert recs["valid"].all()
        gains = lc.fir_gains()
        for r in recs:
            assert abs(r["offset_hz"] - lc.offset_hz(r, gains[r["chain"]])) <= 1e-9 * max(1.0, abs(r["offset_hz"]))


def test_parity_shift_and_prefilter(hostsim_lib, pkg):
    lc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_2m4_shift.cu8"), "-v -d 3 -s", max_batch_mib=1)
    lc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_1m6.cu8"), "-v", max_batch_mib=1, prefilter=1)


def test_parity_access_code_errors_and_pushes(hostsim_lib, pkg):
    cu8 = rc.cached_capture("sync_errors_1m6")
    lc.check_parity(pkg, hostsim_lib, cu8, "-v", (2, 2), (3, 6), max_batch_mib=1)
    lc.check_parity(pkg, hostsim_lib, cu8, "-v", (2, 2), (3, 6), pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777])


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the sums do not depend on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, line_info_cases as lc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "lc.check_parity(pkg, lib, rc.cached_capture('sync_errors_1m6'), '-v', (2, 2), (3, 6), max_batch_mib=1);"
            "lc.check_parity(pkg, lib, rc.cached_capture('synth_mixed_2m4_shift.cu8'), '-v -d 3 -s', max_batch_mib=1)"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.parametrize("case", lc.PLANTED, ids=[f"{c[0]}|{c[1]}" for c in lc.PLANTED])
def test_planted_offsets(hostsim_lib, pkg, case):
    config, flags, n, fs, seed, shift = case
    lc.check_planted(pkg, hostsim_lib, config, flags, n, fs, seed, shift)


def _s1_cut(cu8):
    """a cut on a whole 4096-byte item (1024 decimated samples at d = 2) that leaves an S1 access-code match 800-1350
    samples after it: far enough for the match to be found, close enough for its 1367-sample window to be clipped"""
    for w in lc.oracle_info(cu8, "-v"):
        cut = (w[1] - 800) // 1024 * 1024
        if w[4] == 1 and w[1] - cut < 1350:
            return cut
    raise AssertionError("no S1 match to cut in front of")


@pytest.mark.parametrize("seek", [False, True])
def test_window_clipped_at_stream_start(hostsim_lib, pkg, seek):
    """a capture cut so that an S1 match lies ~1000 samples after its first sample: the window is clipped there (and at
    a wmb_seek position), n is the restated one"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    cut_m = _s1_cut(cu8)
    part = np.ascontiguousarray(cu8[cut_m * 4:])
    want = lc.oracle_info(part, "-v")
    clipped = [w for w in want if w[2] < lc.WINDOW[w[4]][0] - lc.WINDOW[w[4]][1]]
    assert clipped and clipped[0][2] > 0
    base = cut_m if seek else 0
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1) as ctx:
        if seek:
            ctx.push(cu8.ctypes.data, 1 << 20)            # something before the seek, which it forgets
            ctx.seek(cut_m * 2)
        lines, recs = ctx.process(part.ctypes.data, len(part), flush=True, info=True)
    assert [orc.blank_ts(l) for l in lines] == [w[0] for w in want]
    got = [(int(r["sync_sample"]) - base, int(r["n"]), int(r["sum"])) for r in recs]
    assert got == [w[1:4] for w in want]


def test_sample_index_wrap(hostsim_lib, pkg):
    """a stream positioned just below 2^40 decimated samples: the device's 40-bit window positions wrap"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = lc.oracle_info(cu8, "-v")
    m_total = len(cu8) // 4
    for back in (2048 * 20, (m_total // 2) // 2048 * 2048):
        first_m = (1 << 40) - back
        for step in (len(cu8), 1 << 17):
            with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1) as ctx:
                ctx.seek(first_m * 2)
                lines, recs = [], []
                for off in range(0, len(cu8), step):
                    ctx.push(cu8.ctypes.data + off, min(step, len(cu8) - off))
                ctx.poll_flush()
                lines, recs = ctx.take_lines(info=True)
            assert [orc.blank_ts(l) for l in lines] == [w[0] for w in want]
            assert [(int(r["sync_sample"]) - first_m, int(r["n"]), int(r["sum"])) for r in recs] == [w[1:4] for w in want]
            assert int(recs["sync_sample"].max()) > (1 << 40)


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks in process: the merged records equal the sequential run's"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("sync_errors_1m6")
    flags, lock, errors = "-v", (2, 2), (3, 6)
    with pkg.WmbusB200(flags, lib=hostsim_lib, max_batch_mib=1, clock_lock=lock, access_code_errors=errors) as ctx:
        seq_lines, seq = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    parts, infos = [], []
    for rank in range(3):
        with pkg.WmbusB200(flags, lib=hostsim_lib, max_batch_mib=1, clock_lock=lock, access_code_errors=errors) as ctx:
            push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
            (lines, recs), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, 1 << 18, info=True)
        parts.append(lines)
        infos.append(recs)
    lines, recs = shard.merge_lines(parts, infos)
    assert lines == [orc.blank_ts(l) for l in seq_lines]
    assert all(len(p) for p in parts)
    for f in ("sync_sample", "end_sample", "chain", "algo", "crc_ok", "valid", "n", "sum", "carrier_hz"):
        assert np.array_equal(recs[f], seq[f]), f
    assert np.array_equal(recs["offset_hz"], seq["offset_hz"])


def test_manual_frames_have_no_offset(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        ctx.decode_frames(arr, k)
        lines, recs = ctx.take_lines(info=True)
    assert len(lines) > 10 and len(recs) == len(lines)
    assert not recs["valid"].any() and np.isnan(recs["offset_hz"]).all() and not recs["n"].any()


def test_info_cap_leaves_the_rest_queued(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        ref_lines, ref = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
        ctx.reset()
        nl = C.c_size_t(0)
        L.wmb_process(ctx._ctx, cu8.ctypes.data, len(cu8), 1, ctx._out, 0, C.byref(nl), 1)
        assert nl.value == 0
        buf = C.create_string_buffer(1 << 20)
        info = np.zeros(8, pkg.line_info_dtype())
        n = L.wmb_take_lines_info(ctx._ctx, buf, len(buf), C.byref(nl), 1, info.ctypes.data, 3)
        assert nl.value == 3 and C.string_at(buf, n).decode().count("\n") == 3
        assert np.array_equal(info[:3], ref[:3]) and not info["sync_sample"][3:].any()
        rest_lines, rest = ctx.take_lines(info=True)
    assert ref_lines[3:] == rest_lines and np.array_equal(rest, ref[3:])


def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def cli_records(exe_env_fn, tmp_path, flags, cu8):
    """run the CLI with and without WMBUS_B200_LINE_INFO; returns (stdout with, stdout without, record lines)"""
    path = tmp_path / "info.txt"
    r1 = exe_env_fn({"WMBUS_B200_LINE_INFO": str(path)}, cu8.tobytes(), flags)
    r0 = exe_env_fn({}, cu8.tobytes(), flags)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    return r1.stdout, r0.stdout, path.read_text().splitlines()


def expected_records(pkg, lib, cu8, flags):
    with pkg.WmbusB200(flags, lib=lib) as ctx:
        lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    out = []
    for l, r in zip(lines, recs):
        f = l.split(";")
        if f[0] in ("rla", "t2a"):
            f = f[1:]
        off = f"{r['offset_hz']:.0f}" if r["valid"] else "nan"
        out.append(f"{'rla' if r['algo'] == 0 else 't2a'};{f[0]};{r['crc_ok']};{f[6]};{r['sync_sample']};"
                   f"{r['carrier_hz']:.0f};{off}")
    return lines, out


@pytest.mark.parametrize("flags", ["-v", "", "-d 3 -s"])
def test_cli_line_info(hostsim_lib, pkg, tmp_path, flags):
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "synth_mixed_1m6.cu8")
    out1, out0, recs = cli_records(_cli, tmp_path, flags, cu8)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(out1) == blank(out0)                          # stdout does not change (but for the wall-clock time)
    lines, want = expected_records(pkg, hostsim_lib, cu8, flags)
    assert len(out1.decode().splitlines()) == len(recs) == len(lines) > 10
    assert recs == want


def test_cli_line_info_unwritable(hostsim_lib, tmp_path):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env["WMBUS_B200_LINE_INFO"] = str(tmp_path / "no" / "such" / "dir" / "info.txt")
    # stdin stays open and empty: a program that read it would wait here
    p = subprocess.Popen([exe, "-v"], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    try:
        rc_ = p.wait(timeout=120)
        out, err = p.stdout.read(), p.stderr.read()
    finally:
        if p.poll() is None:
            p.kill()
        p.stdin.close()
    assert rc_ == 1 and out == b"" and b"WMBUS_B200_LINE_INFO" in err
