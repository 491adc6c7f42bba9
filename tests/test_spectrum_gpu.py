"""`-m gpu`: the band survey on the H100 -- the FFT and close kernels (csrc/wmb_spectrum.cuh) against the numpy
restatement (tests/spectrum_cases.py), bit for bit; a 256 MiB capture; a 1 GiB capture in one device push against its
time-chunked merge and the restatement on a sample of records; the carrier finder; off means off; the CLI."""
import importlib
import os
import subprocess

import numpy as np
import pytest

import receiver_cases as rc
import spectrum_cases as sc
import test_spectrum as ts
from conftest import ROOT

pytestmark = pytest.mark.gpu

GIB = 1 << 30


@pytest.mark.parametrize("name,flags", ts.CAPTURES, ids=[f"{n}|{f}" for n, f in ts.CAPTURES])
def test_parity(pkg, gpu_lib, name, flags):
    cu8 = rc.cached_capture(name)
    for mib, B in ((1, 16), (256, 64)):
        sc.check_parity(pkg, gpu_lib, cu8, flags, 1024, B, d=ts.d_of(flags), max_batch_mib=mib)


def test_parity_sizes_pushes_seek_window(pkg, gpu_lib):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    for N in sc.BINS:
        for B in (1, 3, 16, 1 << 20):
            sc.check_parity(pkg, gpu_lib, cu8, "-v", N, B, max_batch_mib=1)
    got = sc.product(pkg, gpu_lib, cu8, "-v", 1024, 3, pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777], take_every=True,
                     max_batch_mib=1)
    sc.assert_same(got, sc.restated(cu8, 1024, 3))
    for q0 in (4096 * 5, (1 << 41) + 4096 * 7):
        sc.check_parity(pkg, gpu_lib, cu8, "-v", 256, 3, q0=q0, max_batch_mib=1)
    sc.check_parity(pkg, gpu_lib, cu8, "-v", 1024, 16, window=(100000, 250000), max_batch_mib=1)
    sc.check_parity(pkg, gpu_lib, cu8, "-p T -p S", 512, 7, max_batch_mib=1)


def test_time_chunks(pkg, gpu_lib):
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    merged, parts = ts.time_chunks(pkg, gpu_lib, cu8, "-v", 1024, 100)
    assert all(len(p[0]) for p in parts)
    sc.assert_same(merged, sc.restated(cu8, 1024, 100))


def test_off_means_off(pkg, gpu_lib):
    ts.test_off_means_off(gpu_lib, pkg)


def test_finder_planted(pkg, gpu_lib):
    ts.test_finder_planted(gpu_lib, pkg)


def test_cli_spectrum(pkg, gpu_lib, tmp_path):
    exe = os.path.join(ROOT, "rtl-wmbus_b200", "rtl_wmbus_b200")
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    path = tmp_path / "spectrum.txt"
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    r = subprocess.run([exe, "-v"], input=cu8.tobytes(), capture_output=True, timeout=600,
                       env=dict(env, WMBUS_B200_SPECTRUM=str(path), WMBUS_B200_SPECTRUM_BLOCKS="64"))
    assert r.returncode == 0, r.stderr
    assert path.read_text().splitlines() == ts.expected_file(*sc.product(pkg, gpu_lib, cu8, "-v", 1024, 64))
    bad = subprocess.run([exe, "-v"], input=b"", capture_output=True, timeout=600,
                         env=dict(env, WMBUS_B200_SPECTRUM=str(path), WMBUS_B200_SPECTRUM_BINS="100"))
    assert bad.returncode == 1 and bad.stdout == b""


def test_capture_256mib(pkg, gpu_lib):
    """a 256 MiB capture in 256 MiB batches: every record against the restatement"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(256 << 20, fs=1.6e6, emitters=synth.default_emitters("mixed"), seed=0xB20000A2)
    cu8 = np.ascontiguousarray(host.numpy())
    got = sc.product(pkg, gpu_lib, cu8, "-v", 1024, 16384, max_batch_mib=256)
    want = sc.restated(cu8, 1024, 16384)
    assert len(want[0]) == 8
    sc.assert_same(got, want)


def test_fullsize_1gib(pkg, gpu_lib):
    """1 GiB `-p S` in one device push: the rows equal the time-chunked merge, and the restatement on a sample of
    records"""
    import torch
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB2000063)
    cap = host.cuda()
    torch.cuda.synchronize()
    N, B = 1024, 16384
    with pkg.WmbusB200("-p S", lib=gpu_lib, max_batch_mib=GIB >> 20, spectrum=(N, B)) as ctx:
        ctx.process_device(cap.data_ptr(), GIB, flush=True)
        seq = ctx.take_spectrum()
    assert len(seq[0]) == GIB // (2 * N * B)
    parts = []
    for rank in range(3):
        with pkg.WmbusB200("-p S", lib=gpu_lib, max_batch_mib=256, spectrum=(N, B)) as ctx:
            push = lambda lo, hi: ctx.push_device(cap.data_ptr() + lo, hi - lo)
            (_, sp), _, _, _ = shard.decode_time_chunk(ctx, push, GIB, 2, rank, 3, 1 << 18, spectrum=True)
        parts.append(sp)
    del cap
    merged = shard.merge_spectrum(parts)
    sc.assert_same(merged, (sc.as_rows(seq[0]), seq[1], seq[2]))
    cu8 = host.numpy()
    for i in (0, len(seq[0]) // 2, len(seq[0]) - 1):
        r = int(seq[0]["record"][i])
        lo = r * B * N * 2
        want = sc.restated(cu8[lo:lo + B * N * 2], N, B, q0=r * B * N)
        sc.assert_same((seq[0][i:i + 1], seq[1][i:i + 1], seq[2][i:i + 1]), want)


def test_survey_only_records_longer_than_a_batch(pkg, gpu_lib):
    """no chain enabled (the demod stream then finishes long before the survey kernels), records longer than a batch,
    several batches: the flush's close and the next push's solo batch come after the last batch's survey kernels"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(64 << 20, fs=1.6e6, emitters=synth.default_emitters("mixed"), seed=0xB20000A3)
    cu8 = np.ascontiguousarray(host.numpy())
    want = sc.restated(cu8, 1024, 16384)
    assert len(want[0]) == 2 and want[0][0][2] == 16384
    sc.assert_same(sc.product(pkg, gpu_lib, cu8, "-p T -p S", 1024, 16384, max_batch_mib=16), want)
    # one batch per push: each is alone on the device, so its kernels go on the sequential stream
    sc.assert_same(sc.product(pkg, gpu_lib, cu8, "-p T -p S", 1024, 16384, pushes=[16 << 20] * 4, take_every=True,
                              max_batch_mib=16), want)
