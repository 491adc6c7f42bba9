"""The S1 soft repair on the H100: K4S's S1 instance (32 lanes per candidate, only here) equals its host twin frame by frame
on the corpus of tests/test_s1_soft_repair.py at every s_max and on a noisy S1 capture; the streaming records equal the CPU
build's restatement from manual framing at 1 MiB and 256 MiB batches; and a 256 MiB capture through process_device equals
manual framing of the same bytes on the GPU."""
import importlib

import pytest

import repair_cases as rc
import s1_soft_cases as s1c
from test_repair import as_tuple
from test_s1_soft_repair import capture_manual_framing, full_corpus


@pytest.mark.gpu
@pytest.mark.parametrize("s_max", [1, 2, 3, 4, 5, 6])
def test_k4s_s1_matches_host_twin_gpu(gpu_lib, pkg, s_max):
    cases = full_corpus(s_max)
    for e_max in (1, 3):
        _, host, dev = s1c.run_rule(gpu_lib, pkg, cases, e_max, s_max)
        bad = [i for i in range(len(cases)) if as_tuple(dev[i]) != as_tuple(host[i])]
        assert not bad, (s_max, e_max, len(bad), bad[0])
        assert any(host[i].outcome == rc.REPAIRED for i in range(len(cases)))


@pytest.mark.gpu
def test_capture_manual_framing_gpu(gpu_lib, pkg):
    capture_manual_framing(gpu_lib, pkg, None)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_mib", [1, 256])
def test_stream_records_equal_the_cpu_restatement_gpu(gpu_lib, pkg, hostsim_lib, batch_mib):
    cu8 = s1c.s1_capture()[0]
    settings = [3, 6]
    want = s1c.restated_stream(pkg, hostsim_lib, cu8, "-v", 2, settings)
    for s in settings:
        got = s1c.stream(pkg, gpu_lib, cu8, "-v", 2, "1mib" if batch_mib == 1 else "one", batch_mib=batch_mib,
                         repair_s1_soft=s)[0]
        assert got == want[s], (s, len(got), len(want[s]))
        assert sum(1 for t in got if t[4] == rc.REPAIRED and t[-1]) >= 5


@pytest.mark.gpu
def test_process_device_256mib_gpu(gpu_lib, pkg):
    """256 MiB on the device in one process_device call at e_max 2, s_max 6: the records equal the restatement from
    manual framing of the same bytes, and every datagram the S1 soft rule repaired was sent"""
    import torch
    import repair_stream_cases as rs
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = s1c.s1_emitters(synth)
    cap, plan = synth.synth_capture(256 << 20, emitters=ems, seed=0xB200000E, device="cuda")
    cu8 = cap.cpu().numpy()
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    with pkg.WmbusB200("-v", lib=gpu_lib, repair=2, repair_s1_soft=6, max_batch_mib=256) as ctx:
        ctx.process_device(cap.data_ptr(), cap.numel(), flush=True)
        got = [s1c.record_tuple(r) for r in ctx.take_repairs()]
    torch.cuda.synchronize()
    want = s1c.restated_stream(pkg, gpu_lib, cu8, "-v", 2, [6], max_batch_mib=256)[6]
    assert got == want
    soft = [t for t in got if t[4] == rc.REPAIRED and t[-1]]
    assert len(soft) >= 200 and all(t[-3] in sent for t in soft)
    assert rs.key(got[0]) <= rs.key(got[-1])
