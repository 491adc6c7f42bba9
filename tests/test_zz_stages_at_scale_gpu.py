"""`-m gpu`: every bit-sync stage and bit event against the oracle at the benchmark's batch size and across batches on
the device (tests/batch_stage_checks.py).

The other tap tests see one small batch.  Here: a 1 GiB batch (2^28 decimated samples per chain at d = 2: 8192 time2
tiles over two scan tiles, 131072 run-length phase-1 lanes) as the benchmark runs it, the benchmark's other legs' paths,
and 1 GiB as 128 MiB batches -- serialized with batch boundaries inside real access codes and the event rings wrapping,
and pipelined.  Every event comparison runs at the reference's settings and at L = 1, E = (3, 6).  The output reports
the tiles and scan tiles crossed, the ring wraps, the boundaries inside access codes, the densest warp round and the
access-code flag counts."""
import importlib
import resource
import time

import numpy as np
import pytest

import batch_stage_checks as bsc

pytestmark = pytest.mark.gpu

GIB = 1 << 30
MIB = 1 << 20
SCAN_BOUNDARY = 1 << 27          # decimated sample of the first time2 scan-tile boundary of a 1 GiB batch at d = 2


def _report(tag, **kw):
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6
    print(f"[{tag}] " + ", ".join(f"{k} {v}" for k, v in kw.items()) + f" (peak RSS {rss:.1f} GB)")


def _t1x2_capture():
    """config 2's 1 GiB capture plus one T1 telegram whose access code straddles decimated sample 2^27"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, plan = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB2000020)
    e = synth.Emitter("T1", 0x71200023, amp=80.0, offset_hz=3e3, l_field=0x19, seed=77)
    b = synth.fsk_burst(e.chips(0), e.chip_rate, 1.6e6, e.dev_hz, e.offset_hz, e.amp)
    at = 2 * SCAN_BOUNDARY - 50 * 16                 # chip 50 (of the code's chips 42..57) on the boundary; 16 IQ per chip
    assert not any(p.start_iq < at + len(b) and at < p.start_iq + p.n_iq for p in plan), "the planted burst collides"
    x = host.numpy().reshape(-1, 2)
    x[at:at + len(b)] = np.clip(np.round(x[at:at + len(b)].astype(np.float32) + b), 0, 255).astype(np.uint8)
    return host


@pytest.fixture(scope="module")
def t1x2():
    import torch
    t0 = time.perf_counter()
    host = _t1x2_capture()
    t1 = time.perf_counter()
    ref = bsc.Reference(host.numpy(), "-v -p S")
    t2 = time.perf_counter()
    dev = host.cuda()
    torch.cuda.synchronize()
    _report("t1x2 1 GiB", synth_s=f"{t1 - t0:.0f}", oracle_s=f"{t2 - t1:.0f}", M=ref.M)
    # the planted access code: a real sync within 16 strobes after the scan-tile boundary, on time2
    ev = ref.events[(0, 1, bsc.DEFAULT)]
    i = int(np.searchsorted(ev["m"], SCAN_BOUNDARY))
    assert ev["sync"][i:i + 16].any(), "the planted telegram's access code is meant to straddle the scan-tile boundary"
    yield host, dev, ref
    del dev


def test_benchmark_shape_one_1gib_batch(pkg, gpu_lib, t1x2):
    """-v -p S, device-resident, one process_device(..., flush=True) of the whole 1 GiB, as the benchmark's leg"""
    host, dev, ref = t1x2
    geo = bsc.geometry(gpu_lib)
    tiles = (ref.M + 32 * geo["tile_words"] - 1) // (32 * geo["tile_words"])
    for s in bsc.SETTINGS:
        t = time.perf_counter()
        n, ovf, lines = bsc.run_pipelined(pkg, gpu_lib, ref, GIB, s, device_ptr=dev.data_ptr(), min_batches=1,
                                          max_batch_mib=GIB // MIB)
        assert n == 1
        _report(f"1 GiB batch {bsc.setting_name(s)}", tiles=tiles, scan_tiles=-(-tiles // geo["scan_tile"]),
                sync_flags=ref.sync_counts(s), overflow_batches=ovf, lines_compared=lines,
                seconds=f"{time.perf_counter() - t:.0f}")
        assert s != bsc.DEFAULT or len(ref.lines[s]) > 100


def test_1gib_as_serialized_128mib_device_pushes(pkg, gpu_lib, t1x2):
    """1 GiB as 128 MiB device pushes, one batch each, boundaries moved inside real access codes; the time2 ring of a
    128 MiB batch (2^24 events) wraps inside batches"""
    host, dev, ref = t1x2
    max_m = 128 * MIB // 4
    inside = bsc.boundaries_in_codes(bsc.code_windows(ref))
    chosen = []
    for k in range(1, 8):                 # per 128 MiB step the last boundary inside a code before it
        c = [b for b in inside if k * max_m - max_m // 2 < b <= k * max_m]
        if c:
            chosen.append(max(c))
    assert len(chosen) >= 3, (len(inside), chosen)
    pushes = bsc.pushes_through(chosen, ref.M, 2, max_m)
    ring = bsc.ring_events(128, 2)
    assert ring == 1 << 24
    for s in bsc.SETTINGS:
        t = time.perf_counter()
        r = bsc.run_serialized(pkg, gpu_lib, ref, GIB, pushes, s, device_ptr=dev.data_ptr(), max_batch_mib=128)
        wraps = bsc.wraps_inside(r["totals"][(0, 1)], ring)
        assert wraps, r["totals"][(0, 1)]
        _report(f"serialized 128 MiB {bsc.setting_name(s)}", batches=len(r["batches"]),
                boundaries_in_codes=[(b, inside[b]) for b in chosen], time2_ring_wraps_inside_batches=wraps,
                overflow_batches=r["overflow_batches"], lines_compared=r["lines_compared"],
                seconds=f"{time.perf_counter() - t:.0f}")


def test_1gib_pipelined_as_128mib_batches(pkg, gpu_lib, t1x2):
    """the same capture in one process_device call of 8 overlapping 128 MiB batches: the last batch's taps, the lines"""
    host, dev, ref = t1x2
    for s in bsc.SETTINGS:
        n, ovf, lines = bsc.run_pipelined(pkg, gpu_lib, ref, GIB, s, device_ptr=dev.data_ptr(), max_batch_mib=128)
        assert n == 8
        _report(f"pipelined 8 x 128 MiB {bsc.setting_name(s)}", overflow_batches=ovf, lines_compared=lines)


def test_pipelined_8mib_batches_beyond_the_copy_prefix(pkg, gpu_lib):
    """48 MiB in one process_device call of 8 MiB batches with more candidates than the first prefix copy fetches"""
    import torch
    cu8 = bsc.dense_8mib_capture()
    ref = bsc.Reference(cu8, "-v")
    dev = torch.from_numpy(cu8).cuda()
    torch.cuda.synchronize()
    for s in bsc.SETTINGS:
        n, ovf, lines = bsc.run_pipelined(pkg, gpu_lib, ref, len(cu8), s, device_ptr=dev.data_ptr(), min_batches=6,
                                          max_batch_mib=8)
        assert lines, (bsc.setting_name(s), n, ovf)
        _report(f"pipelined 8 MiB {bsc.setting_name(s)}", batches=n, sync_flags=ref.sync_counts(s), lines=len(ref.lines[s]))
    assert sum(ref.sync_counts(bsc.DENSE).values()) / n > bsc.FIRST_LINE_PREFIX
    del dev


def test_densest_warp_round(t1x2):
    host, dev, ref = t1x2
    per_word, word = bsc.densest_round(ref, 1)
    _report("strobe density t1x2 L=1", densest_round_per_word=f"{per_word:.2f}", densest_word=word)
    assert word <= 11


LEGS = [("mixed", "-v", 2, 1.6e6, 0xB2000021, GIB), ("mixed", "-v -d 3", 3, 2.4e6, 0xB2000040, GIB),
        ("t1x2", "-v -o -p S", 2, 1.6e6, 0xB2000064, 640 * MIB)]


@pytest.mark.parametrize("emitters,flags,d,fs,seed,n_bytes", LEGS, ids=[f for _, f, *_ in LEGS])
def test_benchmark_legs_one_batch(pkg, gpu_lib, emitters, flags, d, fs, seed, n_bytes):
    """the other legs' paths in one batch: both chains and both algorithms (-v), the general front end (-d 3), and the
    -o path (the clock lanes write the data bits) across the time2 scan tile (above 512 MiB)"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(n_bytes, fs=fs, emitters=synth.default_emitters(emitters), seed=seed)
    t = time.perf_counter()
    ref = bsc.Reference(host.numpy(), flags)
    oracle_s = time.perf_counter() - t
    dev = host.cuda()
    torch.cuda.synchronize()
    for s in bsc.SETTINGS:
        n, ovf, lines = bsc.run_pipelined(pkg, gpu_lib, ref, n_bytes, s, device_ptr=dev.data_ptr(), min_batches=1,
                                          max_batch_mib=n_bytes // MIB)
        assert n == 1
        _report(f"{flags} {n_bytes // MIB} MiB {bsc.setting_name(s)}", M=ref.M, sync_flags=ref.sync_counts(s),
                overflow_batches=ovf, lines_compared=lines, oracle_s=f"{oracle_s:.0f}")
    per_word, word = bsc.densest_round(ref, 1)
    _report(f"strobe density {flags} L=1", densest_round_per_word=f"{per_word:.2f}", densest_word=word)
    del dev


def test_mixer_phase_carry_64mib_in_4mib_batches(pkg, gpu_lib):
    """-v -d 3 -s: the mixer's phase is carried from batch to batch (the FM discriminator is blind to a constant phase
    error, so only the samples at a boundary show a wrong carry); dphi of every sample of every 4 MiB batch"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(64 * MIB, fs=2.4e6, emitters=synth.default_emitters("mixed"), seed=0xB2000065,
                                  center_shift_hz=325e3)
    data = np.ascontiguousarray(host.numpy())
    ref = bsc.Reference(data, "-v -d 3 -s")
    gran = 4096 * 3
    body = len(data) // gran * gran
    pushes = []
    while sum(pushes) < body:
        pushes.append(min(body - sum(pushes), (4 * MIB // gran - len(pushes) % 3) * gran))
    pushes.append(len(data) - body)                # a ragged final batch (one 4096-byte item), decoded by the flush
    assert 0 < pushes[-1] < gran and len(pushes) >= 16
    dev = torch.from_numpy(data).cuda()
    torch.cuda.synchronize()
    for s in bsc.SETTINGS:
        r = bsc.run_serialized(pkg, gpu_lib, ref, len(data), pushes, s, device_ptr=dev.data_ptr(), max_batch_mib=4)
        _report(f"-v -d 3 -s 64 MiB in 4 MiB batches {bsc.setting_name(s)}", batches=len(r["batches"]),
                overflow_batches=r["overflow_batches"], lines_compared=r["lines_compared"])
    del dev
