"""`gpu`: telegram records on the H100 -- the committed captures under the flag sets and repair settings of the CPU
tests, at the benchmark's batch size (1 GiB), equal to the restatement and to the CPU-simulation build's records; host
pushes and a device push agree; a 1 GiB device-resident capture against its time-chunked merge, with the same launches
and D2H bytes as telegrams off."""
import importlib

import numpy as np
import pytest

import receiver_cases as rc
import telegram_cases as tc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(rc.COMMITTED))
def test_parity_against_cpu_build(gpu_lib, hostsim_lib, pkg, name):
    cu8 = rc.cached_capture(name)
    for rp in tc.REPAIRS.values():
        for flags in tc.capture_flags(name):
            g = tc.check_parity(pkg, gpu_lib, cu8, flags, repair=rp, max_batch_mib=1024)
            h = tc.check_parity(pkg, hostsim_lib, cu8, flags, repair=rp, max_batch_mib=1)
            assert tc.as_tuples(g[0]) == tc.as_tuples(h[0]) and g[1] == h[1], (name, flags, rp)


def test_host_pushes_and_device_push(gpu_lib, pkg):
    import torch
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    rp = tc.REPAIRS["soft"]
    a = tc.check_parity(pkg, gpu_lib, cu8, "-v", repair=rp, pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777],
                        max_batch_mib=1)
    b = tc.check_parity(pkg, gpu_lib, cu8, "-v", repair=rp, device=torch, max_batch_mib=1024)
    c = tc.check_parity(pkg, gpu_lib, cu8, "-v", repair=rp, pushes=[8192] * (len(cu8) // 8192), max_batch_mib=1)
    assert tc.as_tuples(a[0]) == tc.as_tuples(b[0]) == tc.as_tuples(c[0]) and a[1] == b[1] == c[1]


def test_1gib_device_resident_time_chunks(gpu_lib, pkg):
    """the benchmark's capture (1 GiB t1x2, -p S) with the mixed emitters added: the restatement, the same lines,
    launches and D2H bytes as telegrams off, and three time chunks merged by merge_telegrams"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    n = 1 << 30
    em = synth.default_emitters("t1x2") + synth.default_emitters("mixed")
    cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=em, seed=shard.capture_seed(2, 0), device="cuda")
    rp = tc.REPAIRS["soft"]
    seq = tc.check_parity(pkg, gpu_lib, cap.cpu().numpy(), "-v", repair=rp, device=torch, max_batch_mib=1024)
    assert len(seq[0]) > 1000
    with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=1024, **rp) as ctx:
        lines, info = ctx.process_device(cap.data_ptr(), n, flush=True, info=True)
        st = ctx.stats()
    assert lines == seq[2] and np.array_equal(info, seq[3])
    assert (st.kernel_launches, st.d2h_bytes, st.h2d_bytes) == (seq[5].kernel_launches, seq[5].d2h_bytes, seq[5].h2d_bytes)
    parts, infos, reps = [], [], []
    for rank in range(3):
        with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=256, **rp) as ctx:
            out, *_ = shard.decode_time_chunk(ctx, lambda a, b: ctx.push_device(cap.data_ptr() + a, b - a), n, 2, rank,
                                              3, info=True, repairs=True)
        parts.append(out[0])
        infos.append(out[1])
        reps.append(out[2])
    lines, info = shard.merge_lines(parts, infos)
    recs, data = shard.merge_telegrams(lines, info, shard.merge_repairs(reps), lib=gpu_lib)
    assert tc.as_tuples(recs) == tc.as_tuples(seq[0]) and data == seq[1]
