"""`not gpu`: the band survey (wmb_set_spectrum / wmb_take_spectrum) on the CPU-simulation build of the library (the
kernels' phase functions): every record against the numpy restatement (tests/spectrum_cases.py), bit for bit, over
captures, sizes, pushes, batch sizes, thread orders, seeks, a line window and time chunks; the carrier finder on planted
and committed captures; off means off, setter errors and the CLI's spectrum file."""
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import orc
import receiver_cases as rc
import spectrum_cases as sc
from conftest import GOLDEN, ROOT

CAPTURES = [("excerpt_samples2_a.cu8", "-v"), ("excerpt_issue47_c1.cu8", "-v"), ("excerpt_issue48_2m4.cu8", "-v -d 3 -s"),
            ("synth_mixed_1m6.cu8", "-v"), ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s")]


def d_of(flags):
    return 3 if "-d 3" in flags else 2


def test_tables_equal_library(hostsim_lib):
    for n in sc.BINS:
        hann, tw = np.zeros(n, np.float32), np.zeros(n, np.float32)
        assert hostsim_lib.wmb_debug_spectrum_tables(n, hann.ctypes.data, tw.ctypes.data) == 0
        h, wr, wi = sc.tables(n)
        assert np.array_equal(hann.view(np.uint32), h.view(np.uint32))
        assert np.array_equal(tw[0::2].view(np.uint32), wr.view(np.uint32))
        assert np.array_equal(tw[1::2].view(np.uint32), wi.view(np.uint32))


@pytest.mark.parametrize("name,flags", CAPTURES, ids=[f"{n}|{f}" for n, f in CAPTURES])
def test_parity_committed(hostsim_lib, pkg, name, flags):
    cu8 = rc.cached_capture(name)
    for mib, B in ((1, 16), (256, 64)):                 # (B = 16 at 256 MiB batches needs a table above 2^23 bins)
        sc.check_parity(pkg, hostsim_lib, cu8, flags, 1024, B, d=d_of(flags), max_batch_mib=mib)


@pytest.mark.parametrize("bins", sc.BINS)
def test_parity_sizes(hostsim_lib, pkg, bins):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    for B in (1, 3, 16, 1 << 20):
        rows, _, _ = sc.check_parity(pkg, hostsim_lib, cu8, "-v", bins, B, max_batch_mib=1)
        assert len(rows) == (1 if B == 1 << 20 else -(-(len(cu8) // (2 * bins)) // B))


def test_flags_do_not_matter(hostsim_lib, pkg):
    """the survey reads the raw input: -s, the prefilter and the chains change nothing, and it runs with no chain"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = sc.restated(cu8, 512, 7)
    for flags, kw in (("-v -s", {}), ("-v", {"prefilter": 1}), ("-p T -p S", {}), ("-a -o", {})):
        sc.assert_same(sc.product(pkg, hostsim_lib, cu8, flags, 512, 7, max_batch_mib=1, **kw), want)


def test_parity_odd_pushes(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = sc.restated(cu8, 1024, 3)
    for pushes in ([12345, 1 << 19, 4096 * 3 + 17, 777777], [4096] * 40 + [100000, 3]):
        got = sc.product(pkg, hostsim_lib, cu8, "-v", 1024, 3, pushes=pushes, take_every=True, max_batch_mib=1)
        sc.assert_same(got, want)
    cu8 = rc.cached_capture("excerpt_issue48_2m4.cu8")
    got = sc.product(pkg, hostsim_lib, cu8, "-v -d 3 -s", 2048, 5, pushes=[4096 * 3] * 20, take_every=True, max_batch_mib=1)
    sc.assert_same(got, sc.restated(cu8, 2048, 5, d=3))


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the records do not depend on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, spectrum_cases as sc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "cu8 = rc.cached_capture('synth_mixed_1m6.cu8');"
            "[sc.check_parity(pkg, lib, cu8, '-v', n, b, max_batch_mib=1) for n, b in ((256, 3), (1024, 16), (2048, 1 << 20))];"
            "sc.check_parity(pkg, lib, rc.cached_capture('excerpt_issue48_2m4.cu8'), '-v -d 3 -s', 512, 16, d=3, max_batch_mib=1)"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


def test_seek_off_grid_and_far(hostsim_lib, pkg):
    """a seek to a position that is not on the record grid (the first record is partial), and one past 2^41 IQ samples"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    for q0 in (4096 * 5, (1 << 41) + 4096 * 7):
        for N, B in ((1024, 16), (256, 3)):
            rows, _, _ = sc.check_parity(pkg, hostsim_lib, cu8, "-v", N, B, q0=q0, max_batch_mib=1)
            assert rows["record"][0] == q0 // N // B and rows["blocks"][0] == B - (q0 // N) % B


def test_line_window(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    for window in ((100000, 250000), (12345, 1 << 63)):
        sc.check_parity(pkg, hostsim_lib, cu8, "-v", 1024, 16, window=window, max_batch_mib=1)


def time_chunks(pkg, lib, cu8, flags, N, B, d=2, world=3):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    parts = []
    for rank in range(world):
        with pkg.WmbusB200(flags, lib=lib, max_batch_mib=1, spectrum=(N, B)) as ctx:
            push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
            (lines, sp), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), d, rank, world, 1 << 18, spectrum=True)
        parts.append(sp)
    return shard.merge_spectrum(parts), parts


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks: the merged records equal the sequential run's (records straddle the borders)"""
    for name, flags, N, B in (("synth_mixed_1m6.cu8", "-v", 1024, 100), ("excerpt_issue48_2m4.cu8", "-v -d 3 -s", 256, 7)):
        cu8 = rc.cached_capture(name)
        merged, parts = time_chunks(pkg, hostsim_lib, cu8, flags, N, B, d=d_of(flags))
        assert all(len(p[0]) for p in parts)
        assert len(merged[0]) < sum(len(p[0]) for p in parts)            # some record has a row in two chunks
        sc.assert_same(merged, sc.restated(cu8, N, B, d=d_of(flags)))


def test_off_means_off(hostsim_lib, pkg):
    """no survey: the same lines, line records, bursts, kernel launches and D2H bytes as a context that never heard of
    it; with it on, the same lines, records and bursts"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = []
    for spec in (None, (0, 0), (1024, 16)):
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, burst_level=(14, 14)) as ctx:
            if spec == (0, 0):
                ctx.set_spectrum(2048, 4)
                ctx.set_spectrum(0, 0)
            elif spec:
                ctx.set_spectrum(*spec)
            lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            st = ctx.stats()
            out.append((lines, recs, ctx.take_bursts(), st.kernel_launches, st.d2h_bytes, len(ctx.take_spectrum()[0])))
    (l0, r0, b0, k0, d0, n0), (l1, r1, b1, k1, d1, n1), (l2, r2, b2, k2, d2, n2) = out
    assert l0 == l1 == l2 and np.array_equal(r0, r1) and np.array_equal(r0, r2)
    assert np.array_equal(b0, b1) and np.array_equal(b0, b2) and len(b0)
    assert k0 == k1 and d0 == d1 and n0 == n1 == 0
    assert k2 > k0 and d2 > d0 and n2 > 0


def test_setter_rules(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        for bins, blocks in ((128, 16), (1000, 16), (4096, 16), (1024, 0), (1024, (1 << 20) + 1), (256, 1)):
            assert L.wmb_set_spectrum(ctx._ctx, bins, blocks) == -1, (bins, blocks)       # (256, 1): table too large
        assert L.wmb_set_spectrum(ctx._ctx, 0, 0) == 0
        ctx.set_spectrum(1024, 64)
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert L.wmb_set_spectrum(ctx._ctx, 512, 64) == -6          # after a push
        n = C.c_size_t(7)
        assert L.wmb_take_spectrum(ctx._ctx, None, None, None, 0, C.byref(n)) == 0 and n.value == 0
        ctx.reset()                                                  # the setting survives reset
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        a = ctx.take_spectrum()
        ctx.seek(0)
        ctx.set_spectrum(256, 64)                                     # allowed again after a seek
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        b = ctx.take_spectrum()
    sc.assert_same(a, sc.restated(cu8, 1024, 64))
    sc.assert_same(b, sc.restated(cu8, 256, 64))


def test_partial_take(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L, max_batch_mib=1, spectrum=(512, 8)) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        rows = np.zeros(3, pkg.spectrum_dtype())
        s, p = np.zeros((3, 512), np.uint64), np.zeros((3, 512), np.float32)
        n = C.c_size_t(0)
        assert L.wmb_take_spectrum(ctx._ctx, rows.ctypes.data, s.ctypes.data, p.ctypes.data, 3, C.byref(n)) == 0
        assert n.value == 3
        rest = ctx.take_spectrum()
    got = (np.concatenate([rows, rest[0]]), np.concatenate([s, rest[1]]), np.concatenate([p, rest[2]]))
    sc.assert_same(got, sc.restated(cu8, 512, 8))
    assert rows["bins"][0] == 512 and rows["hz_low"][0] == -800e3 and rows["hz_step"][0] == 1.6e6 / 512


# ---- the carrier finder ----------------------------------------------------------------------------------------

_planted = {}


def planted():
    if not _planted:
        em = sc.planted_emitters()
        cu8, plan = sc.planted_capture(em)
        _planted["v"] = (em, cu8, plan)
    return _planted["v"]


def survey(pkg, lib, cu8, flags, N=1024, B=16384):
    with pkg.WmbusB200(flags, lib=lib, spectrum=(N, B)) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        return ctx.take_spectrum()


def test_finder_planted(hostsim_lib, pkg):
    """T1, C1 and two S1 emitters spread over a 2.4 MS/s band, a CW tone and noise: each planted offset's 25 kHz grid
    point within 25 kHz, the tone as a tone; decode_carriers over the carriers prints each emitter's telegrams as the
    oracle does at those carriers"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    em, cu8, plan = planted()
    rows, s, p = survey(pkg, hostsim_lib, cu8, "-v -d 3")
    carriers, tones = shard.find_carriers(rows, s, p, 2.4e6)
    found = sorted({off for off, _ in carriers})
    for e in em:
        assert any(abs(off * 1e3 - round(e.offset_hz / 25e3) * 25e3) <= 25e3 for off in found), (e.offset_hz, found)
    assert len(found) == len(em), found
    assert len(tones) == 1 and abs(tones[0] - sc.TONE_HZ) < 5e3, tones
    got = shard.decode_carriers(lambda fl, **o: pkg.WmbusB200(fl, lib=hostsim_lib, **o),
                                lambda ctx: ctx.process(cu8.ctypes.data, len(cu8), flush=True), carriers, "-v -d 3")
    for e in em:
        kind = "S" if e.mode == "S1" else "T"
        off = min(found, key=lambda f: abs(f * 1e3 - e.offset_hz))
        o = orc.opts_from_flags("-v -d 3")
        o.simultaneous = 2
        o.carrier_25khz[0 if kind == "T" else 1] = off // 25
        o.carrier_25khz[1 if kind == "T" else 0] = 0
        if kind == "T":
            o.s1_enabled = 0
        else:
            o.t1c1_enabled = 0
        want = [orc.blank_ts(l) for l in orc.run_lines(cu8, o)]
        mine = [l for l in want if f"{e.ident:08X}" in l and l.split(";")[2] == "1"]
        assert len(mine) >= 5, (e.mode, off, len(mine))
        assert got[(off, kind)] == want


def test_finder_noise_alone(hostsim_lib, pkg):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("noise_1m6")
    assert shard.find_carriers(*survey(pkg, hostsim_lib, cu8, "-v"), 1.6e6) == ([], [])
    cu8, _ = sc.planted_capture([], tone_amp=0.0)
    assert shard.find_carriers(*survey(pkg, hostsim_lib, cu8, "-v -d 3"), 2.4e6) == ([], [])


@pytest.mark.parametrize("name,flags", [("excerpt_samples2_a.cu8", "-v"), ("excerpt_issue47_c1.cu8", "-v"),
                                        ("synth_mixed_1m6.cu8", "-v"), ("excerpt_issue48_2m4.cu8", "-v -d 3 -s"),
                                        ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s")])
def test_finder_committed(hostsim_lib, pkg, name, flags):
    """every CRC-ok datagram the reference printed for the capture in its default and -s runs (tests/golden/
    golden_lines.json) is among the CRC-ok lines that decode_carriers prints over the carriers the finder returns"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture(name)
    base = flags.replace(" -s", "")
    d = d_of(flags)
    carriers, _ = shard.find_carriers(*survey(pkg, hostsim_lib, cu8, base), 0.8e6 * d)
    assert carriers
    got = shard.decode_carriers(lambda fl, **o: pkg.WmbusB200(fl, lib=hostsim_lib, **o),
                                lambda ctx: ctx.process(cu8.ctypes.data, len(cu8), flush=True), carriers, base)
    have = {l.split(";")[-1] for ls in got.values() for l in ls if l.split(";")[2] == "1"}
    runs = json.load(open(os.path.join(GOLDEN, "golden_lines.json")))[name]
    want = set()
    for key in (("-d 3", "-d 3 -s") if d == 3 else ("", "-v -s")):
        for l in runs[key]:
            f = l.split(";")
            k = 1 if f[0] in ("rla", "t2a") else 0
            if f[k + 1] == "1":
                want.add(f[-1])
    assert want <= have, sorted(want - have)[:3]           # (excerpt_issue48_2m4 has no CRC-ok datagram)


# ---- the CLI's spectrum file ---------------------------------------------------------------------------------

def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def expected_file(rows, s, p):
    out = []
    with np.errstate(divide="ignore"):
        for r, ss, pp in zip(rows, s, p):
            head = f"{r['record']};{r['start_iq']};{r['blocks']};{r['hz_low']:.2f};{r['hz_step']:.2f}"
            mean = 10 * np.log10(ss.astype(np.float64) / float(r["blocks"]))
            peak = 10 * np.log10(pp.astype(np.float64))
            out.append("mean;" + head + "".join(f";{v:.2f}" for v in mean))
            out.append("peak;" + head + "".join(f";{v:.2f}" for v in peak))
    return out


@pytest.mark.parametrize("flags,name,env,N,B", [("-v", "synth_mixed_1m6.cu8", {}, 1024, 16384),
                                                 ("-d 3 -s", "synth_mixed_2m4_shift.cu8",
                                                  {"WMBUS_B200_SPECTRUM_BINS": "256", "WMBUS_B200_SPECTRUM_BLOCKS": "100"},
                                                  256, 100)])
def test_cli_spectrum(hostsim_lib, pkg, tmp_path, flags, name, env, N, B):
    cu8 = rc.cached_capture(name)
    path = tmp_path / "spectrum.txt"
    r1 = _cli(dict(env, WMBUS_B200_SPECTRUM=str(path)), cu8.tobytes(), flags)
    r0 = _cli({}, cu8.tobytes(), flags)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout) and len(blank(r0.stdout)) > 5
    got = path.read_text().splitlines()
    assert got == expected_file(*sc.product(pkg, hostsim_lib, cu8, flags, N, B)) and len(got) >= 2
    # the CLI users' finder reads the file
    t = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "find_carriers.py"), str(path)],
                       capture_output=True, text=True, timeout=120)
    assert t.returncode == 0 and "carrier" in t.stdout, t.stderr


@pytest.mark.parametrize("env", [{"WMBUS_B200_SPECTRUM": "/nonexistent-dir/x/spectrum.txt"},
                                 {"WMBUS_B200_SPECTRUM": "@TMP", "WMBUS_B200_SPECTRUM_BINS": "1000"},
                                 {"WMBUS_B200_SPECTRUM": "@TMP", "WMBUS_B200_SPECTRUM_BINS": "x"},
                                 {"WMBUS_B200_SPECTRUM": "@TMP", "WMBUS_B200_SPECTRUM_BLOCKS": "0"},
                                 {"WMBUS_B200_SPECTRUM": "@TMP", "WMBUS_B200_SPECTRUM_BLOCKS": "2000000"}])
def test_cli_bad_settings(hostsim_lib, tmp_path, env):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    e = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    e.update({k: (str(tmp_path / "s.txt") if v == "@TMP" else v) for k, v in env.items()})
    # stdin stays open and empty: a program that read it would wait here
    p = subprocess.Popen([exe, "-v"], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e)
    try:
        rc_ = p.wait(timeout=120)
        out, err = p.stdout.read(), p.stderr.read()
    finally:
        if p.poll() is None:
            p.kill()
        p.stdin.close()
    assert rc_ == 1 and out == b"" and b"WMBUS_B200_SPECTRUM" in err


def test_merge_with_an_empty_chunk(hostsim_lib, pkg):
    """a chunk that holds no record ([0, N] arrays) merges with the others"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, spectrum=(512, 16)) as ctx:
        empty = ctx.take_spectrum()
    assert empty[1].shape == (0, 512) and empty[2].shape == (0, 512)
    full = sc.product(pkg, hostsim_lib, cu8, "-v", 512, 16, max_batch_mib=1)
    sc.assert_same(shard.merge_spectrum([empty, full, empty]), sc.restated(cu8, 512, 16))
    with pytest.raises(ValueError):
        shard.find_carriers(*full, 2.4e6)                 # a 1.6 MS/s survey is not a 2.4 MS/s one
