"""Soft values and the C1 soft repair on the H100: every polled T1/C1 frame's soft values equal the restatement on the
oracle's stages at 1 MiB and 256 MiB batches, and the device repair K4S (32 lanes per candidate, only here) equals its
host twin frame by frame on the corpus of tests/test_soft_repair.py and on a noisy C1 capture."""
import importlib

import pytest

import repair_cases as rc
import soft_repair_cases as sc
from test_repair import as_tuple
from test_soft_repair import c1_capture, corpus, golden, run_rule, test_capture_soft_repair_manual_framing


@pytest.mark.gpu
@pytest.mark.parametrize("name,batch_mib", [("synth_mixed_1m6.cu8", 1), ("synth_mixed_1m6.cu8", 256), ("c1", 1), ("c1", 256)])
def test_soft_values_equal_the_restatement_gpu(gpu_lib, pkg, name, batch_mib):
    cu8 = c1_capture() if name == "c1" else golden(name)
    got = sc.polled_soft(pkg, gpu_lib, cu8, "", "1mib" if batch_mib == 1 else "one", batch_mib)
    assert sc.check_polled_soft(got, sc.oracle_streams(cu8, "")) > 1000


@pytest.mark.gpu
@pytest.mark.parametrize("k_max", [1, 2, 3, 4, 5, 6])
def test_k4s_matches_host_twin_gpu(gpu_lib, pkg, k_max):
    cases = corpus(importlib.import_module("rtl-wmbus_b200.synth"), k_max)
    _, host, dev = run_rule(gpu_lib, pkg, cases, 2, k_max)
    bad = [i for i in range(len(cases)) if as_tuple(dev[i]) != as_tuple(host[i])]
    assert not bad, (k_max, len(bad), bad[0])
    assert any(host[i].outcome == rc.REPAIRED for i in range(len(cases)))


@pytest.mark.gpu
def test_capture_soft_repair_manual_framing_gpu(gpu_lib, pkg):
    test_capture_soft_repair_manual_framing(gpu_lib, pkg, None)


# ---- the streaming path --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("batch_mib", [1, 256])
def test_stream_records_equal_the_restatement_gpu(gpu_lib, pkg, batch_mib):
    import repair_stream_cases as rs
    cu8 = sc.weak_capture()[0]
    want = sc.restated_stream(pkg, gpu_lib, cu8, "-v", 2, (1, 4, 6))
    for k_max in (1, 4, 6):
        got = rs.stream(pkg, gpu_lib, cu8, "-v", 2, "1mib" if batch_mib == 1 else "one", batch_mib=batch_mib,
                        repair_soft=k_max)[0]
        assert got == want[k_max], (k_max, len(got), len(want[k_max]))
        assert sum(1 for t in got if t[4] == rc.REPAIRED and t[11] == b"C1") >= 20


@pytest.mark.gpu
def test_process_device_256mib_gpu(gpu_lib, pkg):
    """256 MiB on the device in one process_device call at e_max 2, k_max 6: the records equal the restatement from
    manual framing of the same bytes, and every repaired C1 datagram was sent"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    ems = sc.weak_emitters(synth)
    cap, plan = synth.synth_capture(256 << 20, emitters=ems, seed=0xB200000A, device="cuda")
    cu8 = cap.cpu().numpy()
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    with pkg.WmbusB200("-v", lib=gpu_lib, repair=2, repair_soft=6, max_batch_mib=256) as ctx:
        ctx.process_device(cap.data_ptr(), cap.numel(), flush=True)
        import repair_stream_cases as rs
        got = [rs.record_tuple(r) for r in ctx.take_repairs()]
    torch.cuda.synchronize()
    want = sc.restated_stream(pkg, gpu_lib, cu8, "-v", 2, (6,), max_batch_mib=256)[6]
    assert got == want
    c1 = [t for t in got if t[4] == rc.REPAIRED and t[11] == b"C1"]
    assert len(c1) >= 500 and all(t[-1] in sent for t in c1)
