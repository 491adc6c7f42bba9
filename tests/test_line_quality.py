"""`not gpu`: signal quality (wmb_set_line_quality, wmb_take_lines_quality, wmb_take_bursts_quality) on the CPU-simulation
build of the library (the kernels' phase functions): every line's and every burst's class sums and consumed bits against
the oracle restatement (tests/quality_cases.py), exactly and in order, across captures, flags, batch sizes, pushes, thread
orders, clipping, the 2^40 wrap, batch boundaries and time chunks; off means off; the setter, manual framing and the CLI's
record files; and the planted deviation, chip-rate and noise checks whose bounds DESIGN.md §8 states."""
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
import quality_cases as qc
import receiver_cases as rc
from conftest import ROOT

CAPTURES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls]
LEVEL = bc.DEFAULT_LEVEL


@pytest.mark.parametrize("name,flags", CAPTURES, ids=[f"{n}|{f}" for n, f in CAPTURES])
def test_parity_committed(hostsim_lib, pkg, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        qc.check_parity(pkg, hostsim_lib, cu8, flags, max_batch_mib=mib, level=LEVEL)


@pytest.mark.parametrize("flags", ["-v", "-v -o", "-v -a", "-v -t 0 -a"])
def test_parity_flags(hostsim_lib, pkg, flags):
    want, quals, bq = qc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_1m6.cu8"), flags, max_batch_mib=1,
                                      level=LEVEL)
    assert len(want) > 5 and len(bq) > 5
    if "-a" in flags:
        assert not quals["valid"].any() and not bq["valid"].any()
        assert np.isnan(quals["deviation_hz"]).all() and np.isnan(bq["eye_snr_db"]).all()
        assert np.isfinite(quals["chip_rate_hz"]).all()                 # the chip rate needs no discriminator sums
    else:
        assert quals["valid"].all()


def test_parity_shift_d3(hostsim_lib, pkg):
    qc.check_parity(pkg, hostsim_lib, rc.cached_capture("synth_mixed_2m4_shift.cu8"), "-v -d 3 -s", max_batch_mib=1,
                    level=LEVEL)


def test_parity_access_code_errors_and_pushes(hostsim_lib, pkg):
    cu8 = rc.cached_capture("sync_errors_1m6")
    qc.check_parity(pkg, hostsim_lib, cu8, "-v", (2, 2), (3, 6), max_batch_mib=1, level=LEVEL)
    qc.check_parity(pkg, hostsim_lib, cu8, "-v", (2, 2), (3, 6), pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777],
                    level=LEVEL)


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the sums do not depend on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, quality_cases as qc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "qc.check_parity(pkg, lib, rc.cached_capture('sync_errors_1m6'), '-v', (2, 2), (3, 6), max_batch_mib=1, level=(14, 14));"
            "qc.check_parity(pkg, lib, rc.cached_capture('synth_mixed_2m4_shift.cu8'), '-v -d 3 -s', max_batch_mib=1, level=(14, 14))"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


def _boundary_pushes(want):
    """push sizes (bytes, d = 2) that put batch boundaries (i) between an S1 line's match and its last bit, so its
    candidate is carried into the next batch, and (ii) inside another S1 line's window, so its sums reach back into
    the previous batch's history prefix.  Boundaries fall on whole 2048-sample granules."""
    s1 = [w for w in want if w[4] == 1]
    carried = s1[0][1] // 2048 * 2048 + 2048                  # after the match, long before the telegram's end
    assert carried < s1[0][2]
    lo, hi = lc.WINDOW[1]
    for w in s1[1:]:
        g = (w[1] - hi) // 2048 * 2048
        if g > w[1] - lo and g > carried:
            return [carried * 4, (g - carried) * 4], (s1[0], w)
    raise AssertionError("no S1 window across a granule")


def test_batch_boundaries(hostsim_lib, pkg):
    """a carried candidate takes its sums from the batch of its match; a window across a batch boundary reads the
    history prefix"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = qc.oracle_quality(cu8, "-v")
    pushes, (carried, across) = _boundary_pushes(want)
    _, quals, _, _, _ = qc.product(pkg, hostsim_lib, cu8, "-v", pushes=pushes, max_batch_mib=1)
    for w in (carried, across):
        r = quals[[i for i, x in enumerate(want) if x is w][0]]
        assert int(r["sync_sample"]) == w[1] and qc.sums_of(r) == w[6:] and r["valid"]
    qc.check_parity(pkg, hostsim_lib, cu8, "-v", pushes=pushes, max_batch_mib=1, level=LEVEL)


def _s1_cut(cu8):
    for w in lc.oracle_info(cu8, "-v"):
        cut = (w[1] - 800) // 1024 * 1024
        if w[4] == 1 and w[1] - cut < 1350:
            return cut
    raise AssertionError("no S1 match to cut in front of")


@pytest.mark.parametrize("seek", [False, True])
def test_window_clipped_at_stream_start(hostsim_lib, pkg, seek):
    """an S1 match ~1000 samples after the first sample: the window is clipped there (and at a wmb_seek position)"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    cut_m = _s1_cut(cu8)
    part = np.ascontiguousarray(cu8[cut_m * 4:])
    want = qc.oracle_quality(part, "-v")
    base = cut_m if seek else 0
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, quality=True) as ctx:
        if seek:
            ctx.push(cu8.ctypes.data, 1 << 20)
            ctx.seek(cut_m * 2)
        ctx.push(part.ctypes.data, len(part))
        ctx.poll_flush()
        lines, quals = ctx.take_lines(quality=True)
    assert [orc.blank_ts(l) for l in lines] == [w[0] for w in want]
    assert [(int(r["sync_sample"]) - base,) + qc.sums_of(r) for r in quals] == [(w[1],) + w[6:] for w in want]


def test_sample_index_wrap(hostsim_lib, pkg):
    """a stream positioned just below 2^40 decimated samples"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = qc.oracle_quality(cu8, "-v")
    first_m = (1 << 40) - (len(cu8) // 4 // 2) // 2048 * 2048
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, quality=True) as ctx:
        ctx.seek(first_m * 2)
        for off in range(0, len(cu8), 1 << 17):
            ctx.push(cu8.ctypes.data + off, min(1 << 17, len(cu8) - off))
        ctx.poll_flush()
        lines, quals = ctx.take_lines(quality=True)
    assert [orc.blank_ts(l) for l in lines] == [w[0] for w in want]
    assert [(int(r["sync_sample"]) - first_m, int(r["bits"])) + qc.sums_of(r) for r in quals] == \
        [(w[1], w[3]) + w[6:] for w in want]
    assert int(quals["sync_sample"].max()) > (1 << 40)


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks: the merged line and burst quality records equal the sequential run's"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("sync_errors_1m6")
    kw = dict(lib=hostsim_lib, max_batch_mib=1, clock_lock=(2, 2), access_code_errors=(3, 6), burst_level=LEVEL, quality=True)
    with pkg.WmbusB200("-v", **kw) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        seq_lines, seq_q = ctx.take_lines(quality=True)
        seq_b, seq_bq = ctx.take_bursts(quality=True)
    parts, quals, bursts, bquals = [], [], [], []
    for rank in range(3):
        with pkg.WmbusB200("-v", **kw) as ctx:
            push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
            (lines, q, b, bq), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, 1 << 18, bursts=True,
                                                                 quality=True)
        parts.append(lines); quals.append(q); bursts.append(b); bquals.append(bq)
    lines, q = shard.merge_lines(parts, quals=quals)
    assert lines == [orc.blank_ts(l) for l in seq_lines] and all(len(p) for p in parts)
    assert q.tobytes() == seq_q.tobytes()
    b, bq = shard.merge_bursts(bursts, bquals)
    assert b.tobytes() == seq_b.tobytes() and bq.tobytes() == seq_bq.tobytes()


def test_manual_frames(hostsim_lib, pkg):
    """frames handed to wmb_decode_frames: no sums (valid 0), the chip rate as the device framer's lines have it"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    _, dev_q, _, _, _ = qc.product(pkg, hostsim_lib, cu8, "-v")
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1, quality=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        ctx.decode_frames(arr, k)
        lines, quals = ctx.take_lines(quality=True)
    assert len(lines) > 10 and len(quals) == len(dev_q)
    assert not quals["valid"].any() and not quals["n_hi"].any() and np.isnan(quals["eye_snr_db"]).all()
    assert np.array_equal(quals["bits"], dev_q["bits"]) and np.array_equal(quals["chip_rate_hz"], dev_q["chip_rate_hz"])


def test_off_means_off(hostsim_lib, pkg):
    """on or off, the lines, line records, bursts and kernel launches are the same; off copies no quality bytes and
    reports zero sums; on adds 40 bytes per candidate and per burst record copied"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = {}
    for on in (False, True):
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=LEVEL, quality=on) as ctx:
            ctx.push(cu8.ctypes.data, len(cu8))
            ctx.poll_flush()
            lines, info, quals = ctx.take_lines(info=True, quality=True)
            out[on] = (lines, info, ctx.take_bursts(), quals, ctx.stats())
    (l0, i0, b0, q0, s0), (l1, i1, b1, q1, s1) = out[False], out[True]
    assert l0 == l1 and i0.tobytes() == i1.tobytes() and b0.tobytes() == b1.tobytes()
    assert s0.kernel_launches == s1.kernel_launches
    assert s1.d2h_bytes > s0.d2h_bytes and (s1.d2h_bytes - s0.d2h_bytes) % 40 == 0
    assert not q0["valid"].any() and not q0["n_hi"].any() and not q0["s2_lo"].any()
    assert np.array_equal(q0["chip_rate_hz"], q1["chip_rate_hz"]) and q1["valid"].all()


def test_setter(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        assert L.wmb_set_line_quality(ctx._ctx, 2) == -1                  # WMB_E_INVAL
        assert L.wmb_set_line_quality(None, 1) == -1
        assert L.wmb_set_line_quality(ctx._ctx, 1) == 0
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert L.wmb_set_line_quality(ctx._ctx, 0) != 0 and b"after samples were pushed" in L.wmb_last_error()
        ctx.reset()                                                       # the setting survives reset ...
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        _, q = ctx.take_lines(quality=True)
        assert len(q) > 10 and q["valid"].all()
        ctx.seek(0)                                                       # ... and seek; off again after it
        ctx.set_line_quality(False)
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        _, q = ctx.take_lines(quality=True)
        assert len(q) > 10 and not q["valid"].any()


def test_partial_take(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L, quality=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        nl = C.c_size_t(0)
        buf = C.create_string_buffer(1 << 20)
        q = np.zeros(8, pkg.line_quality_dtype())
        n = L.wmb_take_lines_quality(ctx._ctx, buf, len(buf), C.byref(nl), 1, None, q.ctypes.data, 3)
        assert nl.value == 3 and C.string_at(buf, n).decode().count("\n") == 3 and q["valid"][:3].all()
        _, rest = ctx.take_lines(quality=True)
    want = qc.oracle_quality(cu8, "-v")
    assert [qc.sums_of(r) for r in q[:3]] + [qc.sums_of(r) for r in rest] == [w[6:] for w in want]


# ---- the CLI's record files -------------------------------------------------------------------------------------------

def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def _fmt(valid, prec, v):
    return f"{v:.{prec}f}" if valid and v == v else "nan"


@pytest.mark.parametrize("flags", ["-v", "", "-d 3 -s"])
def test_cli_files(hostsim_lib, pkg, tmp_path, flags):
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "synth_mixed_1m6.cu8")
    lq, bf, bq = tmp_path / "lq.txt", tmp_path / "b.txt", tmp_path / "bq.txt"
    r1 = _cli({"WMBUS_B200_LINE_QUALITY": str(lq), "WMBUS_B200_BURSTS": str(bf), "WMBUS_B200_BURST_QUALITY": str(bq)},
              cu8.tobytes(), flags)
    r2 = _cli({"WMBUS_B200_BURSTS": str(tmp_path / "b0.txt")}, cu8.tobytes(), flags)
    assert r1.returncode == 0 and r2.returncode == 0, (r1.stderr, r2.stderr)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(r1.stdout) == blank(r2.stdout)                        # stdout does not change
    assert bf.read_text() == (tmp_path / "b0.txt").read_text()         # nor does the burst file
    with pkg.WmbusB200(flags, lib=hostsim_lib, burst_level=LEVEL, quality=True) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        lines, quals = ctx.take_lines(quality=True)
        bursts, bquals = ctx.take_bursts(quality=True)
    want = []
    for l, r in zip(lines, quals):
        f = l.split(";")
        f = f[1:] if f[0] in ("rla", "t2a") else f
        want.append(f"{'rla' if r['algo'] == 0 else 't2a'};{f[0]};{r['crc_ok']};{f[6]};{r['sync_sample']};"
                    f"{_fmt(r['valid'], 0, r['deviation_hz'])};{_fmt(r['valid'], 2, r['eye_snr_db'])};"
                    f"{_fmt(1, 1, r['chip_rate_hz'])}")
    got = lq.read_text().splitlines()
    assert len(got) == len(r1.stdout.decode().splitlines()) > 10 and got == want
    bwant = [f"{'T1C1' if q['chain'] == 0 else 'S1'};{q['start_sample']};{_fmt(q['valid'], 0, q['deviation_hz'])};"
             f"{_fmt(q['valid'], 2, q['eye_snr_db'])}" for q in bquals]
    bgot = bq.read_text().splitlines()
    assert len(bgot) == len(bf.read_text().splitlines()) == len(bursts) > 5 and bgot == bwant


@pytest.mark.parametrize("env", [{"WMBUS_B200_LINE_QUALITY": "{bad}"},
                                 {"WMBUS_B200_BURSTS": "{ok}", "WMBUS_B200_BURST_QUALITY": "{bad}"},
                                 {"WMBUS_B200_BURST_QUALITY": "{ok}"}], ids=["line", "burst", "burst-without-bursts"])
def test_cli_bad_path(hostsim_lib, tmp_path, env):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    e = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    e.update({k: v.format(bad=tmp_path / "no" / "such" / "x.txt", ok=tmp_path / "ok.txt") for k, v in env.items()})
    # stdin stays open and empty: a program that read it would wait here
    p = subprocess.Popen([exe, "-v"], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e)
    try:
        rc_ = p.wait(timeout=120)
        out, err = p.stdout.read(), p.stderr.read()
    finally:
        if p.poll() is None:
            p.kill()
        p.stdin.close()
    assert rc_ == 1 and out == b"" and b"QUALITY" in err


# ---- planted signals ---------------------------------------------------------------------------------------------------
# Bounds measured on the CPU build, stated in DESIGN.md §8.

def _emitters(devs, rates, mode="T1"):
    E = lc.synth_mod().Emitter
    out = []
    for i, (d, r) in enumerate(zip(devs, rates)):
        e = E(mode, 0x11110001 + i, amp=90.0, offset_hz=0.0, dev_hz=d, l_field=0x19, period_s=0.09,
              start_s=0.004 + 0.03 * i, seed=40 + i)
        e.chip_rate *= r
        out.append(e)
    return out


def test_planted_deviation(hostsim_lib, pkg):
    """40 / 50 / 60 kHz emitters read back in that order, each at 0.77 .. 0.82 of the planted deviation (the post-demod
    FIR's ISI keeps the tones from reaching their full deviation inside a chip; measured 0.787 .. 0.804)"""
    devs = (40e3, 50e3, 60e3)
    got = qc.planted_quality(pkg, hostsim_lib, _emitters(devs, (1, 1, 1)))
    assert sorted(got) == [0, 1, 2]
    for i, d in enumerate(devs):
        v = np.array(got[i][0])
        assert len(v) >= 20 and (v / d).min() >= qc.DEV_RATIO[0] and (v / d).max() <= qc.DEV_RATIO[1], (d, v.min(), v.max())
    assert max(got[0][0]) < min(got[1][0]) and max(got[1][0]) < min(got[2][0])


@pytest.mark.parametrize("mode", ["T1", "S1"])
def test_planted_chip_rate(hostsim_lib, pkg, mode):
    """chip clocks scaled by -2 % / +2 % read back within CHIP_PPM of the planted rate"""
    rates = (0.98, 1.02)
    em = _emitters((50e3, 50e3), rates, mode)
    got = qc.planted_quality(pkg, hostsim_lib, em)
    assert sorted(got) == [0, 1]
    for i, e in enumerate(em):
        v = np.array(got[i][2])
        ppm = (v / e.chip_rate - 1.0) * 1e6
        assert len(v) >= 10 and np.abs(ppm).max() <= qc.CHIP_PPM, (mode, e.chip_rate, ppm.min(), ppm.max())


def test_planted_snr_falls_with_noise(hostsim_lib, pkg):
    """the same telegrams at noise sigma 4 / 8 / 16 / 32 LSB: each emitter's mean eye SNR falls at every step, and none
    exceeds the noiseless ceiling the FIR's ISI sets"""
    em = _emitters((50e3,) * 3, (1, 1, 1))
    ceiling = qc.planted_quality(pkg, hostsim_lib, em, noise_sigma=0.0)
    top = max(x for v in ceiling.values() for x in v[1])
    assert abs(top - qc.SNR_CEILING_DB) < 0.1, top
    means = []
    for s in (4, 8, 16, 32):
        got = qc.planted_quality(pkg, hostsim_lib, em, noise_sigma=s)
        assert sorted(got) == [0, 1, 2] and all(len(got[i][1]) == len(ceiling[i][1]) for i in got)   # the same telegrams
        means.append([float(np.mean(got[i][1])) for i in range(3)])
        assert max(x for v in got.values() for x in v[1]) <= top + 0.1
    for a, b in zip(means, means[1:]):
        assert all(x > y for x, y in zip(a, b)), means
