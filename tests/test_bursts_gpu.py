"""`-m gpu`: the burst report on the H100 -- the mask, event, run and reduce kernels (csrc/wmb_bursts.cuh) against the
numpy restatement on the oracle's stages (tests/burst_cases.py), exactly; time chunks; the far-off emitter; the CLI's
record file; and a 1 GiB capture in one device push."""
import importlib
import os
import subprocess

import numpy as np
import pytest

import burst_cases as bc
import orc
import receiver_cases as rc
from conftest import ROOT

pytestmark = pytest.mark.gpu

GIB = 1 << 30
CASES = [(name, fl) for name, fls in rc.COMMITTED.items() for fl in fls] + [("synth_mixed_1m6.cu8", "-v -a")]


@pytest.mark.parametrize("name,flags", CASES, ids=[f"{n}|{f}" for n, f in CASES])
def test_parity(pkg, gpu_lib, name, flags):
    cu8 = rc.cached_capture(name)
    for mib in (1, 256):
        bc.check_parity(pkg, gpu_lib, cu8, flags, max_batch_mib=mib)


def test_parity_levels_pushes_prefilter_cw(pkg, gpu_lib):
    cu8 = rc.cached_capture("excerpt_samples2_a.cu8")
    for level in ((5, 5), (1, 0), (255, 255)):
        bc.check_parity(pkg, gpu_lib, cu8, "-v", level, max_batch_mib=1)
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    bc.check_parity(pkg, gpu_lib, cu8, "-v", pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777])
    bc.check_parity(pkg, gpu_lib, cu8, "-v", max_batch_mib=1, prefilter=2)
    cw, _ = bc.cw_capture(8 << 20)
    for mib in (1, 256):
        _, recs = bc.check_parity(pkg, gpu_lib, cw, "-v", max_batch_mib=mib)
        assert ((recs["flags"] & bc.CONTINUED) != 0).sum() >= 8


def test_time_chunks(pkg, gpu_lib):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    for cu8, level in ((rc.cached_capture("synth_mixed_1m6.cu8"), (8, 8)), (bc.cw_capture(8 << 20)[0], bc.DEFAULT_LEVEL)):
        _, seq, _ = bc.product_bursts(pkg, gpu_lib, cu8, "-v", level, max_batch_mib=1)
        parts = []
        for rank in range(3):
            with pkg.WmbusB200("-v", lib=gpu_lib, max_batch_mib=1, burst_level=level) as ctx:
                push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
                (_, b), _, _, _ = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, 1 << 18, bursts=True)
            parts.append(b)
        assert shard.merge_bursts(parts).tobytes() == seq.tobytes()


def test_far_off_emitter(pkg, gpu_lib):
    em, far = bc.planted_emitters(60e3)
    cu8, plan = bc.planted_capture(em)
    _, _, far_mean = bc.check_planted(pkg, gpu_lib, cu8, em, plan, far)
    cu8b, _ = bc.planted_capture(em, center_shift_hz=-far_mean)
    with pkg.WmbusB200("-v", lib=gpu_lib) as ctx:
        lines = ctx.process(cu8b.ctypes.data, len(cu8b), flush=True)
    mine = [l for l in lines if f"{far.ident:08X}" in l]
    ok = [l for l in mine if l.split(";")[2] == "1"]
    assert len(ok) >= 5 and 2 * len(ok) >= len(mine), (len(ok), len(mine))   # the rest collide with other telegrams


def test_cli_bursts(pkg, gpu_lib, tmp_path):
    import test_bursts as tb
    exe = os.path.join(ROOT, "rtl-wmbus_b200", "rtl_wmbus_b200")

    def run(env_extra, stdin_bytes, flags):
        env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
        env.update(env_extra)
        return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)
    tb.check_cli(run, pkg, gpu_lib, tmp_path, "-v", rc.cached_capture("synth_mixed_1m6.cu8"))
    bad = run({"WMBUS_B200_BURSTS": str(tmp_path / "b.txt"), "WMBUS_B200_BURST_LEVEL": "300"}, b"", "-v")
    assert bad.returncode == 1 and bad.stdout == b""


def test_fullsize_t1x2_1gib(pkg, gpu_lib):
    """1 GiB `-v -p S` in one device push: every record equals the restatement on the oracle's stages"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    host, _ = synth.synth_capture(GIB, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=0xB2000063)
    cap = host.cuda()
    torch.cuda.synchronize()
    with pkg.WmbusB200("-v -p S", lib=gpu_lib, max_batch_mib=GIB >> 20, burst_level=bc.DEFAULT_LEVEL) as ctx:
        lines = ctx.process_device(cap.data_ptr(), GIB, flush=True)
        recs = ctx.take_bursts()
    del cap
    want = bc.oracle_bursts(host.numpy(), "-v -p S", bc.DEFAULT_LEVEL)
    assert len(want) > 100 and len(lines) > 100
    assert bc.as_tuples(recs) == want
