"""`-m gpu`: signal quality on the H100 -- the class sums k3_fill takes in a second pass over a new match's offset window
(split over the 8 threads that rank it, added with shuffles) and kb_reduce over a burst's, against the oracle restatement
(tests/quality_cases.py), exactly and in order; off means off; the planted checks; the CLI's record files; and a 1 GiB
synthetic capture against its own time-chunked merge."""
import importlib
import os
import subprocess

import numpy as np
import pytest

import burst_cases as bc
import orc
import quality_cases as qc
import receiver_cases as rc
from conftest import ROOT

pytestmark = pytest.mark.gpu

GIB = 1 << 30
LEVEL = bc.DEFAULT_LEVEL
CASES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls] + \
        [("synth_mixed_1m6.cu8", "-v -p T"), ("synth_mixed_1m6.cu8", "-v -a")]


@pytest.mark.parametrize("name,flags", CASES, ids=[f"{n}|{f}" for n, f in CASES])
def test_parity(pkg, gpu_lib, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        qc.check_parity(pkg, gpu_lib, cu8, flags, max_batch_mib=mib, level=LEVEL)


def test_parity_errors_and_pushes(pkg, gpu_lib):
    cu8 = rc.cached_capture("sync_errors_1m6")
    qc.check_parity(pkg, gpu_lib, cu8, "-v", (2, 2), (3, 6), max_batch_mib=1, level=LEVEL)
    qc.check_parity(pkg, gpu_lib, cu8, "-v", (2, 2), (3, 6), pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777], level=LEVEL)


def test_off_means_off(pkg, gpu_lib):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = {}
    for on in (False, True):
        with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=1, burst_level=LEVEL, quality=on) as ctx:
            ctx.push(cu8.ctypes.data, len(cu8))
            ctx.poll_flush()
            lines, info = ctx.take_lines(info=True)
            out[on] = (lines, info, ctx.take_bursts(), ctx.stats())
    (l0, i0, b0, s0), (l1, i1, b1, s1) = out[False], out[True]
    assert l0 == l1 and i0.tobytes() == i1.tobytes() and b0.tobytes() == b1.tobytes()
    assert s0.kernel_launches == s1.kernel_launches and s1.d2h_bytes > s0.d2h_bytes


def test_planted(pkg, gpu_lib):
    E = importlib.import_module("rtl-wmbus_b200.synth").Emitter
    em = []
    for i, (d, r) in enumerate(zip((40e3, 50e3, 60e3), (0.98, 1.0, 1.02))):
        e = E("T1", 0x11110001 + i, amp=90.0, dev_hz=d, l_field=0x19, period_s=0.09, start_s=0.004 + 0.03 * i, seed=40 + i)
        e.chip_rate *= r
        em.append(e)
    got = qc.planted_quality(pkg, gpu_lib, em)
    assert sorted(got) == [0, 1, 2]
    for i, e in enumerate(em):
        dev, rate = np.array(got[i][0]), np.array(got[i][2])
        assert qc.DEV_RATIO[0] <= (dev / e.dev_hz).min() and (dev / e.dev_hz).max() <= qc.DEV_RATIO[1]
        assert np.abs((rate / e.chip_rate - 1.0) * 1e6).max() <= qc.CHIP_PPM


def test_cli_files(pkg, gpu_lib, tmp_path):
    exe = os.path.join(ROOT, "rtl-wmbus_b200", "rtl_wmbus_b200")
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    lq, bf, bq = tmp_path / "lq.txt", tmp_path / "b.txt", tmp_path / "bq.txt"
    r1 = subprocess.run([exe, "-v"], input=cu8.tobytes(), capture_output=True, timeout=600,
                        env=dict(env, WMBUS_B200_LINE_QUALITY=str(lq), WMBUS_B200_BURSTS=str(bf),
                                 WMBUS_B200_BURST_QUALITY=str(bq)))
    r0 = subprocess.run([exe, "-v"], input=cu8.tobytes(), capture_output=True, env=env, timeout=600)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout)
    want = qc.oracle_quality(cu8, "-v")
    got = lq.read_text().splitlines()
    assert len(got) == len(want) > 10
    assert [int(g.split(";")[4]) for g in got] == [w[1] for w in want]
    assert len(bq.read_text().splitlines()) == len(bf.read_text().splitlines()) > 5


def test_1gib_against_time_chunks(pkg, gpu_lib):
    """1 GiB `-v -p S` in one device push against four time chunks of it: the merged line and burst quality records
    are the sequential run's, byte for byte"""
    import torch
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    cap, _ = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB20000A3, device="cuda")
    torch.cuda.synchronize()
    kw = dict(lib=gpu_lib, max_batch_mib=256, burst_level=LEVEL, quality=True)
    with pkg.WmbusB200("-v -p S", **kw) as ctx:
        ctx.push_device(cap.data_ptr(), GIB)
        ctx.poll_flush()
        seq_lines, seq_q = ctx.take_lines(quality=True)
        seq_b, seq_bq = ctx.take_bursts(quality=True)
        assert ctx.stats().overflow_batches == 0
    assert len(seq_lines) > 100 and seq_q["valid"].mean() > 0.9
    parts, quals, bursts, bquals = [], [], [], []
    for rank in range(4):
        with pkg.WmbusB200("-v -p S", **kw) as ctx:
            push = lambda lo, hi: ctx.push_device(cap.data_ptr() + lo, hi - lo)
            (lines, q, b, bqr), _, _, _ = shard.decode_time_chunk(ctx, push, GIB, 2, rank, 4, 1 << 18, bursts=True,
                                                                  quality=True)
        parts.append(lines); quals.append(q); bursts.append(b); bquals.append(bqr)
    del cap
    lines, q = shard.merge_lines(parts, quals=quals)
    assert lines == [orc.blank_ts(l) for l in seq_lines]
    assert q.tobytes() == seq_q.tobytes()
    b, bqm = shard.merge_bursts(bursts, bquals)
    assert b.tobytes() == seq_b.tobytes() and bqm.tobytes() == seq_bq.tobytes()
