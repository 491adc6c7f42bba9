"""Erasure repair on the streaming path on the H100 (the 32-lane parts of K4R run only here): the device's records equal
the CPU build's and the restatement from manual framing at 1 MiB and 256 MiB batches, a 256 MiB capture through
process_device equals the restatement from manual framing on the GPU, and the dense-match setting at 64 MiB."""
import importlib

import numpy as np
import pytest

import repair_cases as rc
import repair_stream_cases as rs


@pytest.mark.gpu
@pytest.mark.parametrize("e_max", (1, 2, 3))
def test_device_records_equal_cpu_build_and_restatement_gpu(gpu_lib, hostsim_lib, pkg, e_max):
    cu8, _plan, _ems = rs.flipped_capture()
    want = rs.restated(pkg, hostsim_lib, cu8, "-v", (e_max,))[e_max]
    assert sum(1 for t in want if t[4] == rc.REPAIRED) >= 20
    assert rs.stream(pkg, hostsim_lib, cu8, "-v", e_max)[0] == want
    assert rs.stream(pkg, gpu_lib, cu8, "-v", e_max)[0] == want
    assert rs.stream(pkg, gpu_lib, cu8, "-v", e_max, "one", batch_mib=256)[0] == want
    assert rs.stream(pkg, gpu_lib, cu8, "-v", e_max, "uneven")[0] == want


def device_records(pkg, lib, cap, n, e_max, batch_mib=256, **kw):
    with pkg.WmbusB200("-v", lib=lib, repair=e_max, max_batch_mib=batch_mib, **kw) as ctx:
        ctx.process_device(cap.data_ptr(), n, flush=True, raw=True)
        return [rs.record_tuple(r) for r in ctx.take_repairs()]


@pytest.mark.gpu
def test_256mib_capture_process_device_gpu(gpu_lib, pkg):
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    from test_repair import flipped_emitters
    n = 256 << 20
    ems = flipped_emitters(synth)
    cu8, plan = synth.synth_capture(n, emitters=ems, seed=0xB2000009)
    cu8 = np.ascontiguousarray(cu8.numpy())
    cap = torch.from_numpy(cu8).cuda()
    want = rs.restated(pkg, gpu_lib, cu8, "-v", (2,))[2]
    got = device_records(pkg, gpu_lib, cap, n, 2)
    assert got == want
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    rep = [t[-1] for t in got if t[4] == rc.REPAIRED]
    assert len(rep) > 500 and set(rep) <= sent


@pytest.mark.gpu
def test_dense_matches_64mib_gpu(gpu_lib, pkg):
    """clock lock 1, T1/C1 access-code errors 3 (and S1 6): the dense candidate load, in 16 MiB batches (a batch of
    64 MiB overflows its frame-word table there, with or without repair)"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    from test_repair import flipped_emitters
    n = 64 << 20
    cu8, _plan = synth.synth_capture(n, emitters=flipped_emitters(synth), seed=0xB200000A)
    cu8 = np.ascontiguousarray(cu8.numpy())
    cap = torch.from_numpy(cu8).cuda()
    kw = dict(clock_lock=(1, 2), access_code_errors=(3, 6))
    want = rs.restated(pkg, gpu_lib, cu8, "-v", (3,), max_batch_mib=16, **kw)[3]
    assert device_records(pkg, gpu_lib, cap, n, 3, batch_mib=16, **kw) == want
    assert {rc.REPAIRED, rc.TOO_MANY, rc.UNREPAIRABLE} <= {t[4] for t in want}
