"""Receiver settings (wmb_set_receiver): the clock-lock threshold of the time2 algorithm and the access-code bit errors
accepted, the reference's two tuning constants (rtl_wmbus.c:865-866, :99, :103).  `not gpu`: the CPU oracle against
what reference builds with those constants changed printed (tests/golden/reference_runs_receiver.json), and the
CPU-simulation build of the library (the kernels' phase functions) against both, stage by stage and line by line.  The
oracle with other settings is tests/receiver_oracle.py, built on oracle/wmbus_oracle.c."""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import orc
import pipeline_checks as pc
import receiver_cases as rc
import receiver_oracle as ro
from conftest import ROOT

# every variant but the default on every capture is the oracle's job; the library gets these
LIB_VARIANTS = [((1, 1), (0, 0)), ((3, 3), (0, 0)), ((4, 4), (0, 0)), ((2, 2), (1, 1)), ((2, 2), (2, 2)),
                ((2, 2), (3, 6)), ((1, 3), (2, 4))]


@pytest.mark.parametrize("lock,errors", rc.VARIANTS, ids=[rc.variant_name(*v) for v in rc.VARIANTS])
def test_oracle_matches_reference_variants(orc_mod, lock, errors):
    for name, flags in rc.cases():
        got = ro.run_lines(rc.cached_capture(name), flags, lock, errors)
        assert got == rc.want_lines(lock, errors, name, flags), (name, flags)


@pytest.mark.parametrize("flags", ["-v", "-v -o", "", "-v -r 0", "-v -t 0 -a", "-v -d 3 -s -o"])
def test_oracle_defaults_are_the_oracle(orc_mod, flags):
    """with the reference's constants the restatement is the CPU oracle itself, stage by stage and line by line"""
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "synth_mixed_1m6.cu8")
    o = orc.opts_from_flags(flags)
    assert ro.run_lines(cu8, flags) == pc.oracle_lines(cu8, flags)
    data = np.ascontiguousarray(cu8[:len(cu8) // 12288 * 12288])
    for chain in (0, 1):
        st = orc.stages(data, o, chain)
        assert np.array_equal(ro.strobes(st["clk"], 2), st["strobe"])
        for algo in (0, 1):
            want, got = orc.events(st, chain, algo), ro.stream_events(st, chain, algo, 2, 0)
            for f in ("m", "bit", "sync", "reset", "rssi"):
                assert np.array_equal(got[f].astype(np.uint64), want[f].astype(np.uint64)), (chain, algo, f)


def test_fixture_is_not_vacuous():
    """the sync-error capture: the defaults print only the clean telegrams; tolerance prints the others, and the lines
    of the default build are the unmodified reference's"""
    base = rc.want_lines((2, 2), (0, 0), "sync_errors_1m6", "-v")
    assert len(base) > 10
    assert len(rc.want_lines((2, 2), (1, 1), "sync_errors_1m6", "-v")) > len(base)
    assert len(rc.want_lines((2, 2), (3, 6), "sync_errors_1m6", "-v")) > len(rc.want_lines((2, 2), (1, 1), "sync_errors_1m6", "-v"))
    assert len(rc.want_lines((1, 1), (0, 0), "excerpt_issue48_2m4.cu8", "-v -d 3 -s")) != len(
        rc.want_lines((2, 2), (0, 0), "excerpt_issue48_2m4.cu8", "-v -d 3 -s"))
    golden = pc.oracle_lines(rc.cached_capture("synth_mixed_1m6.cu8"), "-v")
    assert rc.want_lines((2, 2), (0, 0), "synth_mixed_1m6.cu8", "-v") == golden


@pytest.mark.parametrize("lock,errors", LIB_VARIANTS, ids=[rc.variant_name(*v) for v in LIB_VARIANTS])
def test_lines_match_reference_variants(hostsim_lib, pkg, lock, errors):
    for name, flags in rc.cases():
        rc.check_lines(pkg, hostsim_lib, name, flags, lock, errors)


@pytest.mark.parametrize("flags", ["-v", "-v -o", "-v -d 3 -s"])
@pytest.mark.parametrize("lock,errors", [((1, 1), (1, 2)), ((3, 4), (2, 5)), ((4, 1), (3, 6)), ((16, 16), (0, 0))])
def test_stages_match_oracle(hostsim_lib, pkg, flags, lock, errors):
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "sync_errors_1m6")
    rc.check_stages(pkg, hostsim_lib, cu8, flags, lock, errors)


@pytest.mark.parametrize("flags", ["-v", "-v -o"])
def test_stages_monolithic_run_length_lanes(hostsim_lib, pkg, flags):
    """the T1/C1 run-length stream through the monolithic lanes (k2m_edge) instead of the two-phase path (k2p2w_c)"""
    rc.check_stages(pkg, hostsim_lib, rc.cached_capture("sync_errors_1m6"), flags, (1, 3), (3, 6),
                    reserved=(C.c_uint32 * 2)(1, 0))


@pytest.mark.parametrize("lock,errors", [((1, 3), (2, 4)), ((3, 3), (0, 0)), ((2, 2), (3, 6))])
def test_batch_borders_and_push_patterns(hostsim_lib, pkg, lock, errors):
    """stencil histories and shift registers carried across lanes, batches and ragged pushes"""
    for flags in ("-v", "-v -o"):
        for tuning in ({"max_batch_mib": 1}, {"max_batch_mib": 1, "chunk_samples": 1024, "warmup_samples": 4096},
                       {"pushes": [12345, 1 << 19, 4096 * 3 + 17, 777777]}):
            tuning = dict(tuning)
            pushes = tuning.pop("pushes", None)
            rc.check_lines(pkg, hostsim_lib, "sync_errors_1m6", flags, lock, errors, pushes=pushes, **tuning)


def test_manual_frames(hostsim_lib, pkg):
    """wmb_poll + wmb_decode_frames with candidates a few bits apart: the first match in idle wins, later ones inside
    the telegram are ignored (t1_c1_packet_decoder.h:272-278), as in the reference"""
    lock, errors = (2, 2), (3, 6)
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want = rc.want_lines(lock, errors, "synth_mixed_1m6.cu8", "-v")
    lines = []
    with pkg.WmbusB200("-v", lib=hostsim_lib, manual_frames=1, max_batch_mib=1, clock_lock=lock, access_code_errors=errors) as ctx:
        step = 1 << 19
        for off in range(0, len(cu8), step):
            ctx.push(cu8.ctypes.data + off, min(step, len(cu8) - off))
            arr, k = ctx.poll(flush=False)
            ctx.decode_frames(arr, k)
            lines += ctx.take_lines()
        arr, k = ctx.poll(flush=True)
        ctx.decode_frames(arr, k)
        lines += ctx.take_lines()
        st = ctx.stats()
    assert lines == want
    # matches closer together than a telegram exist (the preamble matches within 3 errors several bits before the sync
    # word) and most of them are ignored
    assert sum(st.candidates[0]) > 4 * sum(st.lines[0])


def test_first_match_in_idle_wins(hostsim_lib, pkg):
    """with E > 0 one stream's matches lie a few bits apart: the candidates the device gathers are consecutive bit
    ordinals, and the lines are still exactly the reference's (which honours only the first)"""
    lock, errors = (2, 2), (3, 6)
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    st = rc.check_lines(pkg, hostsim_lib, "synth_mixed_1m6.cu8", "-v", lock, errors, max_batch_mib=1)
    s = orc.stages(np.ascontiguousarray(cu8), orc.opts_from_flags("-v"), 0)
    ev = ro.stream_events(s, 0, 1, 2, 3)
    idx = np.nonzero(ev["sync"])[0]
    assert len(idx) == st.candidates[0][1]
    assert np.min(np.diff(idx)) <= 2                     # matches on neighbouring bits of one stream
    assert len(rc.want_lines(lock, errors, "synth_mixed_1m6.cu8", "-v")) < len(rc.want_lines((2, 2), (0, 0), "synth_mixed_1m6.cu8", "-v"))


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: nothing depends on their order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, receiver_cases as rc; from conftest import HOSTSIM_SO;"
            "pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "rc.check_lines(pkg, lib, 'sync_errors_1m6', '-v', (1, 3), (2, 4), max_batch_mib=1);"
            "rc.check_lines(pkg, lib, 'sync_errors_1m6', '-v -o', (1, 3), (2, 4), chunk_samples=1024, warmup_samples=4096)"
            % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, WMB_HOSTSIM_ORDER=order)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.parametrize("flags,lock,errors", [("-v", (1, 1), (2, 2)), ("-v -o", (3, 4), (3, 6))])
def test_time_chunks(hostsim_lib, pkg, flags, lock, errors):
    cu8 = rc.cached_capture("sync_errors_1m6")
    rc.check_time_chunks(pkg, hostsim_lib, cu8, flags, lock, errors, world=3, halo_m=1 << 18, max_batch_mib=1)


def test_boundary_state_holds_the_settings(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    n = 1 << 20
    digests = set()
    for lock, errors in [((2, 2), (0, 0)), ((2, 2), (1, 0)), ((2, 3), (0, 0))]:
        with pkg.WmbusB200("-v", lib=hostsim_lib, clock_lock=lock, access_code_errors=errors) as ctx:
            ctx.push(cu8.ctypes.data, n)
            digests.add(hashlib.sha256(ctx.boundary_state()).digest())
    assert len(digests) == 3


def test_explicit_defaults_are_the_defaults(hostsim_lib, pkg):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    outs = []
    for kw in ({}, {"clock_lock": (2, 2), "access_code_errors": (0, 0)}):
        with pkg.WmbusB200("-v", lib=hostsim_lib, **kw) as ctx:
            raw = ctx.process(cu8.ctypes.data, len(cu8), flush=True, raw=True)
            st = ctx.stats()
            ctx.reset()
            ctx.push(cu8.ctypes.data, 1 << 20)
            bs = ctx.boundary_state()
        fields = {f: getattr(st, f) for f, _ in st._fields_ if not f.endswith("_ms")}
        fields = {k: (list(map(list, v)) if not isinstance(v, int) else v) for k, v in fields.items()}
        outs.append((raw, fields, bs))
    assert outs[0] == outs[1]


def test_setter_errors_and_state(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        c = ctx._ctx
        for chain, lock, err in [(0, 0, 0), (0, 17, 0), (1, 0, 0), (0, 2, 4), (1, 2, 7), (2, 2, 0), (-1, 2, 0)]:
            assert L.wmb_set_receiver(c, chain, lock, err) == -1, (chain, lock, err)
            assert L.wmb_last_error()
        assert L.wmb_set_receiver(None, 0, 2, 0) == -1
        for chain, lock, err in [(0, 1, 0), (0, 16, 3), (1, 16, 6), (1, 2, 0), (0, 2, 0)]:
            assert L.wmb_set_receiver(c, chain, lock, err) == 0
        ctx.push(cu8.ctypes.data, 100)                      # less than one granule: held back, but pushed
        assert L.wmb_set_receiver(c, 0, 1, 0) == -6
        ctx.push(cu8.ctypes.data + 100, 1 << 20)
        assert L.wmb_set_receiver(c, 0, 1, 0) == -6
        ctx.reset()
        assert L.wmb_set_receiver(c, 0, 1, 1) == 0
        ctx.push(cu8.ctypes.data, 1 << 20)
        ctx.seek(4096 * 8)
        assert L.wmb_set_receiver(c, 1, 3, 2) == 0
    # the settings survive reset
    with pkg.WmbusB200("-v", lib=L, clock_lock=(1, 1), access_code_errors=(2, 2)) as ctx:
        first = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        ctx.reset()
        again = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
    assert first == again
    assert first == ro.run_lines(cu8, "-v", (1, 1), (2, 2))
    with pytest.raises(RuntimeError):
        pkg.WmbusB200("-v", lib=L, clock_lock=(0, 2))


def _cli(env_extra, name="synth_mixed_1m6.cu8", flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=rc.cached_capture(name).tobytes(), capture_output=True, env=env,
                          timeout=600)


def test_cli_environment(hostsim_lib):
    for env, lock, errors in [({"WMBUS_B200_CLOCK_LOCK": "1"}, (1, 1), (0, 0)),
                              ({"WMBUS_B200_CLOCK_LOCK": "1,3", "WMBUS_B200_ACCESS_CODE_ERRORS": "2,4"}, (1, 3), (2, 4)),
                              ({"WMBUS_B200_ACCESS_CODE_ERRORS": "3,6"}, (2, 2), (3, 6))]:
        r = _cli(env, "sync_errors_1m6")
        assert r.returncode == 0, r.stderr
        got = [orc.blank_ts(l) for l in r.stdout.decode().split("\n") if l]
        assert got == rc.want_lines(lock, errors, "sync_errors_1m6", "-v"), env
    for bad in [{"WMBUS_B200_CLOCK_LOCK": "0"}, {"WMBUS_B200_CLOCK_LOCK": "17"}, {"WMBUS_B200_CLOCK_LOCK": "2x"},
                {"WMBUS_B200_CLOCK_LOCK": ""}, {"WMBUS_B200_CLOCK_LOCK": "2,"}, {"WMBUS_B200_CLOCK_LOCK": "-1"},
                {"WMBUS_B200_ACCESS_CODE_ERRORS": "4"}, {"WMBUS_B200_ACCESS_CODE_ERRORS": "3,7"},
                {"WMBUS_B200_ACCESS_CODE_ERRORS": "1,2,3"}]:
        r = _cli(bad)
        assert r.returncode == 1 and r.stdout == b"" and b"rtl_wmbus_b200:" in r.stderr, (bad, r.returncode, r.stderr)


def test_noise_at_maximum_tolerance(hostsim_lib, pkg):
    """chance matches on noise at the largest accepted error counts stay inside the per-batch candidate tables"""
    st = rc.check_lines(pkg, hostsim_lib, "noise_1m6", "-v", (2, 2), (3, 6))
    m = st.decimated_samples
    assert sum(st.candidates[0]) + sum(st.candidates[1]) < m / 256
    assert st.overflow_batches == 0


def test_frame_word_overflow_keeps_the_stream(hostsim_lib, pkg):
    """T1/C1 at 3 access-code errors on 192 MiB of noise in one batch: ~90 k chance matches want more frame words than
    the batch's table holds.  The batch loses them (overflow_batches) and carries them all as incomplete; the carried
    list holds 65 536 per stream, and the count the next gather and wmb_pending_before read must not exceed that."""
    synth = __import__("importlib").import_module("rtl-wmbus_b200.synth")
    n = 192 << 20
    buf, _ = synth.synth_capture(n, fs=1.6e6, emitters=[], seed=0xB2000064)
    cu8 = np.ascontiguousarray(buf.numpy())
    with pkg.WmbusB200("-v -p S", lib=hostsim_lib, max_batch_mib=256, access_code_errors=(3, 0)) as ctx:
        ctx.push(cu8.ctypes.data, n)
        assert ctx.pending_before(1 << 62) >= 0
        ctx.poll_flush()
        lines = ctx.take_lines()
        st = ctx.stats()
    assert st.overflow_batches >= 1
    assert sum(st.candidates[0]) > 65536
    assert lines == []
