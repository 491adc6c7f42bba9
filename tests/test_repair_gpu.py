"""Erasure repair on the H100: the device repair K4R (wmb_frame_repair_device) against its host twin frame by frame at
every e_max, on the candidates of tests/test_repair.py, planted telegrams back as sent, and a capture decoded with
manual framing whose candidates are repaired on the device."""
import importlib

import pytest

import repair_cases as rc
from test_repair import E_MAX, all_cases, as_tuple, check_capture_repair, device_repair, host_repair, make_frames


@pytest.mark.gpu
def test_device_repair_matches_host_twin_gpu(gpu_lib, pkg):
    cases = all_cases(importlib.import_module("rtl-wmbus_b200.synth"))
    assert len(cases) >= 10000
    frames, _keep = make_frames(pkg, cases)
    for e_max in E_MAX:
        host = [as_tuple(r) for r in host_repair(gpu_lib, frames, e_max)]
        dev = device_repair(gpu_lib, pkg, frames, e_max)
        bad = [i for i in range(len(cases)) if as_tuple(dev[i]) != host[i]]
        assert not bad, (e_max, len(bad), bad[0])
        n_rep = 0
        for i, c in enumerate(cases):
            r = dev[i]
            if r.outcome == rc.REPAIRED:
                assert bytes(r.line.datagram[:r.line.len]) == c.get("sent"), i
                n_rep += 1
            if c["planted"] is not None and c["planted"]["worst"] <= e_max:
                assert r.outcome == rc.REPAIRED, (e_max, i)
        assert n_rep > 100


@pytest.mark.gpu
def test_capture_with_flipped_chips_manual_framing_gpu(gpu_lib, pkg):
    check_capture_repair(gpu_lib, pkg)
