"""`-m gpu`: receiver settings (wmb_set_receiver) on the H100 -- the cooperative clock-recovery lanes (three threads per
lane: time2 on, no DC block, whole words) and the per-thread lanes (-o, and a ragged final batch), the bit streams and
time-chunk sharding, against the reference builds' lines (tests/golden/reference_runs_receiver.json) and the CPU oracle;
plus a 1 GiB capture at L = 1 and at E = 2 against the oracle."""
import importlib

import numpy as np
import pytest

import receiver_cases as rc
import receiver_oracle as ro

pytestmark = pytest.mark.gpu

GIB = 1 << 30
VARIANTS = [((1, 1), (0, 0)), ((3, 3), (0, 0)), ((4, 4), (0, 0)), ((2, 2), (2, 2)), ((2, 2), (3, 6)), ((1, 3), (2, 4))]


@pytest.mark.parametrize("lock,errors", VARIANTS, ids=[rc.variant_name(*v) for v in VARIANTS])
def test_lines_match_reference_variants(pkg, gpu_lib, lock, errors):
    for name, flags in rc.cases():
        rc.check_lines(pkg, gpu_lib, name, flags, lock, errors)
        rc.check_lines(pkg, gpu_lib, name, flags, lock, errors, max_batch_mib=1)


@pytest.mark.parametrize("flags", ["-v", "-v -o", "-v -d 3 -s"])
@pytest.mark.parametrize("lock,errors", [((1, 1), (1, 2)), ((3, 4), (2, 5)), ((16, 16), (3, 6))])
def test_stages_match_oracle(pkg, gpu_lib, flags, lock, errors):
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8" if "-d 3" in flags else "sync_errors_1m6")
    rc.check_stages(pkg, gpu_lib, cu8, flags, lock, errors)


def test_ragged_final_batch(pkg, gpu_lib):
    """-d 3 and a capture of 4096 * (3 k + 1) bytes: the last batch ends in a partial lane word and takes the per-thread
    lanes, the others the cooperative ones (without -o)"""
    cu8 = rc.cached_capture("synth_mixed_2m4_shift.cu8")
    cut = np.ascontiguousarray(cu8[:(len(cu8) // 12288 - 1) * 12288 + 4096])
    for flags, lock, errors in (("-v -d 3 -s", (1, 3), (2, 4)), ("-v -d 3 -s -o", (3, 3), (3, 6))):
        want = ro.run_lines(cut, flags, lock, errors)
        assert len(want) > 5
        for mib in (1, 256):
            with pkg.WmbusB200(flags, lib=gpu_lib, max_batch_mib=mib, clock_lock=lock, access_code_errors=errors) as ctx:
                got = ctx.process(cut.ctypes.data, len(cut), flush=True)
            assert got == want, (flags, mib, len(got), len(want))


@pytest.mark.parametrize("flags,lock,errors", [("-v", (1, 1), (2, 2)), ("-v -o", (3, 4), (3, 6))])
def test_time_chunks(pkg, gpu_lib, flags, lock, errors):
    rc.check_time_chunks(pkg, gpu_lib, rc.cached_capture("sync_errors_1m6"), flags, lock, errors, world=3,
                         halo_m=1 << 18, max_batch_mib=1)


def test_noise_at_maximum_tolerance(pkg, gpu_lib):
    st = rc.check_lines(pkg, gpu_lib, "noise_1m6", "-v", (2, 2), (3, 6))
    assert st.overflow_batches == 0


def test_fullsize_lock1_and_errors2_1gib(pkg, gpu_lib):
    """1 GiB (T1/C1 chain, both algorithms) decoded on the GPU at L = 1 and at E = 2: the same lines, in order, as
    the CPU oracle with the same settings"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB2000063)
    settings = [((1, 1), (0, 0)), ((2, 2), (2, 2))]
    cap = host.cuda()
    torch.cuda.synchronize()
    got = []
    for lock, errors in settings:
        with pkg.WmbusB200("-v -p S", lib=gpu_lib, max_batch_mib=GIB >> 20, clock_lock=lock, access_code_errors=errors) as ctx:
            got.append(ctx.process_device(cap.data_ptr(), GIB, flush=True))
            assert ctx.stats().overflow_batches == 0
    del cap
    want = ro.run_lines_many(host.numpy(), "-v -p S", settings)
    for s, g, w in zip(settings, got, want):
        assert len(w) > 100
        assert g == w, (s, len(g), len(w))
