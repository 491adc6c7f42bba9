"""`not gpu`: every bit-sync stage and bit event, batch by batch, against the oracle on the CPU build (tests/hostsim),
whose tiny time2 tiles, scan tiles and "warps" cross every boundary with small captures (tests/batch_stage_checks.py).
Every comparison runs at the reference's receiver settings and at clock lock 1 with access-code errors (3, 6), where
about 1 % of random bits carry the access-code flag, so that a wrong carried shift register shows at nearly every
boundary."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import batch_stage_checks as bsc
import receiver_cases as rc
from conftest import ROOT, load_fixture

MIB = 1 << 20


def uneven_pushes(n_bytes, d, max_bytes=3 * MIB // 4, ragged=0):
    """whole-granule push sizes of varying length, each at most max_bytes (a host push above 3/4 of the batch size is
    cut in two batches); ragged: a last push of that many bytes (less than a granule), decoded by the flush"""
    gran = 4096 * d
    top = max_bytes // gran
    sizes, at, k = [], 0, 0
    body = n_bytes - ragged
    while at < body:
        n = min(body - at, gran * (5, top - 3, 1, top // 2 + 7, top, 19)[k % 6])
        sizes.append(n)
        at += n
        k += 1
    return sizes + ([ragged] if ragged else [])


CASES = [("excerpt_samples2_a.cu8", "-v", 0), ("excerpt_samples2_a.cu8", "-v -o", 0),
         ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s", 4096), ("synth_mixed_1m6.cu8", "-v -p S", 0),
         ("sync_errors_1m6", "-v", 0), ("sync_errors_1m6", "-v -o", 0)]


@pytest.mark.parametrize("name,flags,ragged", CASES, ids=[f"{n}|{f}" for n, f, _ in CASES])
def test_batch_by_batch(pkg, hostsim_lib, name, flags, ragged):
    """1 MiB batches: serialized in uneven pushes (with a ragged final batch at -d 3), and pipelined"""
    cu8 = rc.cached_capture(name)
    d = max(1, int(flags.split("-d ")[1].split()[0]) if "-d " in flags else 2)
    n = len(cu8) // (4096 * d) * 4096 * d
    if ragged:
        n -= 4096 * d - ragged
    data = np.ascontiguousarray(cu8[:n])
    ref = bsc.Reference(data, flags)
    pushes = uneven_pushes(n, d, ragged=ragged)
    assert len(pushes) >= 3
    for s in bsc.SETTINGS:
        r = bsc.run_serialized(pkg, hostsim_lib, ref, data, pushes, s, max_batch_mib=1)
        if ragged:
            assert r["batches"][-1][1] % 32 != 0, "the last batch is meant to end in a partial word"
        assert bsc.run_pipelined(pkg, hostsim_lib, ref, data, s, max_batch_mib=1)[0] >= 2
    assert sum(ref.sync_counts(bsc.DENSE).values()) > 10 * sum(ref.sync_counts(bsc.DEFAULT).values())


def _long_capture():
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    cap, _ = synth.synth_capture(12 * MIB, fs=1.6e6, emitters=synth.default_emitters("mixed"), seed=0xB2000091)
    return np.ascontiguousarray(cap.numpy())


def test_event_rings_wrap_inside_a_batch(pkg, hostsim_lib):
    """opts.reserved[1] & 2 sizes the run-length rings like time2's; over 12 MiB in 1 MiB batches both T1/C1 rings wrap,
    and at least once strictly inside a batch, where k2t_flush's per-slot mask and the run-length ring writes split"""
    cu8 = _long_capture()
    ref = bsc.Reference(cu8, "-v")
    ring = bsc.ring_events(1, 2)
    assert ring == 1 << 18
    pushes = uneven_pushes(len(cu8), 2)
    for s in bsc.SETTINGS:
        r = bsc.run_serialized(pkg, hostsim_lib, ref, cu8, pushes, s, reserved1=2, max_batch_mib=1)
        for algo in (0, 1):
            inside = bsc.wraps_inside(r["totals"][(0, algo)], ring)
            assert inside, ("no ring wrap inside a batch", algo, r["totals"][(0, algo)][-1], ring)
            print(f"[rings] {bsc.setting_name(s)} chain 0 algo {algo}: {r['totals'][(0, algo)][-1]} events, "
                  f"ring {ring}, wraps inside batches {inside}")
        bsc.run_pipelined(pkg, hostsim_lib, ref, cu8, s, reserved1=2, max_batch_mib=1)


def _shift_into_codes(cu8, ref, d):
    """the capture delayed by p decimated samples (its own first samples repeated in front, as many cut at the end),
    p chosen so that the most real access codes straddle a granule boundary"""
    wins = bsc.code_windows(ref)
    best, best_p = -1, 0
    for p in range(0, bsc.GRANULE_M, 4):
        k = sum(1 for first, last, _, _ in wins if (first + p) // bsc.GRANULE_M != (last + p) // bsc.GRANULE_M)
        if k > best:
            best, best_p = k, p
    nb = best_p * 2 * d
    return np.ascontiguousarray(np.concatenate([cu8[:nb], cu8[:len(cu8) - nb]]))


@pytest.mark.parametrize("name", ["sync_errors_1m6", "synth_mixed_1m6.cu8"])
def test_batch_boundaries_inside_access_codes(pkg, hostsim_lib, name):
    """batch boundaries between the first and the last bit of real access codes (T1/C1: 16 strobes / run-length
    events, S1: 24): the shift register carried across the boundary decides a real line, not only a flag"""
    ref0 = bsc.Reference(rc.cached_capture(name), "-v", settings=[bsc.DEFAULT], lines=False)
    cu8 = _shift_into_codes(rc.cached_capture(name), ref0, 2)
    ref = bsc.Reference(cu8, "-v")
    inside = bsc.boundaries_in_codes(bsc.code_windows(ref))
    assert len(inside) >= 2, inside
    pushes = bsc.pushes_through(inside, ref.M, 2, 3 << 16)
    for s in bsc.SETTINGS:
        r = bsc.run_serialized(pkg, hostsim_lib, ref, cu8, pushes, s, max_batch_mib=1)
        starts = {m0 for m0, _ in r["batches"]}
        assert set(inside) <= starts
        assert r["lines_compared"] and len(ref.lines[s]) >= 3
    print(f"[codes] {name}: batch boundaries inside access codes at {sorted(inside.items())}")


def test_pipelined_batches_beyond_the_copy_prefix(pkg, hostsim_lib):
    """8 MiB batches with more candidates than the first prefix copy fetches, several in flight: every candidate is
    read, whichever prefix was current when its batch was gathered"""
    cu8 = bsc.dense_8mib_capture()
    ref = bsc.Reference(cu8, "-v")
    for s in bsc.SETTINGS:
        n, ovf, compared = bsc.run_pipelined(pkg, hostsim_lib, ref, cu8, s, max_batch_mib=8, min_batches=6)
        assert compared, (bsc.setting_name(s), n, ovf)
    assert sum(ref.sync_counts(bsc.DENSE).values()) / n > bsc.FIRST_LINE_PREFIX


@pytest.mark.parametrize("order", [1, 2])
def test_simulated_thread_order(hostsim_lib, order):
    """the checks above with the CPU build's threads run backwards (1) and scrambled (2), in a process of their own
    (WMB_HOSTSIM_ORDER is read once; see test_hostsim_pipeline.py)"""
    env = dict(os.environ, WMB_HOSTSIM_ORDER=str(order))
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "not gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_batch_stages.py"), "-k", "not thread_order"],
                       env=env, cwd=ROOT, capture_output=True, timeout=1200)
    assert r.returncode == 0, r.stdout.decode()[-3000:]
    assert b"passed" in r.stdout
