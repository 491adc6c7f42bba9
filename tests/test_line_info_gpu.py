"""`-m gpu`: per-line carrier offsets (wmb_take_lines_info) on the H100 -- the sums k3_fill takes where a match is
first seen, split over the threads that rank it and added with shuffles, against the oracle restatement
(tests/line_info_cases.py), exactly; planted offsets; time chunks; the CLI's record file; and a 1 GiB capture."""
import importlib
import os
import subprocess

import numpy as np
import pytest

import line_info_cases as lc
import orc
import receiver_cases as rc
from conftest import ROOT

pytestmark = pytest.mark.gpu

GIB = 1 << 30
CASES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls] + \
        [("synth_mixed_1m6.cu8", "-v -p T"), ("synth_mixed_1m6.cu8", "-v -a")]


@pytest.mark.parametrize("name,flags", CASES, ids=[f"{n}|{f}" for n, f in CASES])
def test_parity(pkg, gpu_lib, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        lc.check_parity(pkg, gpu_lib, cu8, flags, max_batch_mib=mib)


def test_parity_errors_pushes_prefilter(pkg, gpu_lib):
    cu8 = rc.cached_capture("sync_errors_1m6")
    for mib in (1, 256):
        lc.check_parity(pkg, gpu_lib, cu8, "-v", (2, 2), (3, 6), max_batch_mib=mib)
    lc.check_parity(pkg, gpu_lib, cu8, "-v", (2, 2), (3, 6), pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777])
    lc.check_parity(pkg, gpu_lib, rc.cached_capture("synth_mixed_1m6.cu8"), "-v", max_batch_mib=1, prefilter=2)


@pytest.mark.parametrize("case", lc.PLANTED, ids=[f"{c[0]}|{c[1]}" for c in lc.PLANTED])
def test_planted_offsets(pkg, gpu_lib, case):
    config, flags, n, fs, seed, shift = case
    lc.check_planted(pkg, gpu_lib, config, flags, n, fs, seed, shift)


def test_time_chunks(pkg, gpu_lib):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = rc.cached_capture("sync_errors_1m6")
    with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=1, access_code_errors=(3, 6)) as ctx:
        seq_lines, seq = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    parts, infos = [], []
    for rank in range(3):
        with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=1, access_code_errors=(3, 6)) as ctx:
            push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
            (lines, recs), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, 1 << 18, info=True)
        parts.append(lines)
        infos.append(recs)
    lines, recs = shard.merge_lines(parts, infos)
    assert lines == [orc.blank_ts(l) for l in seq_lines]
    assert recs.tobytes() == seq.tobytes()


def test_cli_line_info(pkg, gpu_lib, tmp_path):
    exe = os.path.join(ROOT, "rtl-wmbus_b200", "rtl_wmbus_b200")
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    path = tmp_path / "info.txt"
    r1 = subprocess.run([exe, "-v"], input=cu8.tobytes(), capture_output=True, env=dict(env, WMBUS_B200_LINE_INFO=str(path)), timeout=600)
    r0 = subprocess.run([exe, "-v"], input=cu8.tobytes(), capture_output=True, env=env, timeout=600)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda out: [orc.blank_ts(l) for l in out.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout)
    with pkg.WmbusB200("-v", lib=gpu_lib) as ctx:
        lines, recs = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    want = []
    for l, r in zip(lines, recs):
        f = l.split(";")[1:]
        off = f"{r['offset_hz']:.0f}" if r["valid"] else "nan"
        want.append(f"{'rla' if r['algo'] == 0 else 't2a'};{f[0]};{r['crc_ok']};{f[6]};{r['sync_sample']};{r['carrier_hz']:.0f};{off}")
    got = path.read_text().splitlines()
    assert len(got) == len(blank(r1.stdout)) > 10 and got == want
    bad = subprocess.run([exe, "-v"], input=b"", capture_output=True, timeout=120,
                         env=dict(env, WMBUS_B200_LINE_INFO=str(tmp_path / "no" / "dir" / "x")))
    assert bad.returncode == 1 and bad.stdout == b""


def test_fullsize_t1x2_1gib(pkg, gpu_lib):
    """1 GiB `-v -p S` in one device push: every line's record equals the oracle restatement"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB2000063)
    cap = host.cuda()
    torch.cuda.synchronize()
    with pkg.WmbusB200("-v -p S", lib=gpu_lib, max_batch_mib=GIB >> 20) as ctx:
        lines, recs = ctx.process_device(cap.data_ptr(), GIB, flush=True, info=True)
        assert ctx.stats().overflow_batches == 0
    del cap
    want = lc.oracle_info(host.numpy(), "-v -p S")
    assert len(want) > 100
    assert [orc.blank_ts(l) for l in lines] == [w[0] for w in want]
    got = [(int(r["sync_sample"]), int(r["n"]), int(r["sum"]), int(r["chain"]), int(r["algo"])) for r in recs]
    assert got == [w[1:] for w in want]
