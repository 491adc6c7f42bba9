"""`gpu`: burst snippets on the H100 -- the same parity as the CPU-simulation build and the restatement at 1 MiB and
256 MiB batches, a 1 GiB device-resident capture against its time-chunked merge, the replay contract, the snippet
kernels' resources, and the default path's machine code unchanged by them."""
import importlib
import json
import os

import numpy as np
import pytest

import burst_cases as bc
import receiver_cases as rc
import snippet_cases as sc
from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mib", [1, 256])
def test_parity_against_cpu_build(gpu_lib, hostsim_lib, pkg, mib):
    for name, flags in [("synth_mixed_1m6.cu8", "-v"), ("excerpt_issue48_2m4.cu8", "-v -d 3 -s"),
                        ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s")]:
        cu8 = rc.cached_capture(name)
        for mode in (1, 2):
            g = sc.check_parity(pkg, gpu_lib, cu8, flags, mode, max_batch_mib=mib)
            h = sc.check_parity(pkg, hostsim_lib, cu8, flags, mode, max_batch_mib=mib)
            assert sc.as_tuples(g[0]) == sc.as_tuples(h[0]) and g[1] == h[1]
    cu8, _ = bc.cw_capture(4 << 20)
    g = sc.check_parity(pkg, gpu_lib, cu8, "-v", 1, max_batch_mib=mib)
    assert (g[0]["lost"] == 0).all()


def test_host_pushes_and_device_push(gpu_lib, pkg):
    """ragged host pushes (the H2D into an input buffer waits for the snippet copy of its last batch) and
    process_device give the same snippets"""
    import torch
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    a = sc.check_parity(pkg, gpu_lib, cu8, "-v", 1, pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777], max_batch_mib=1)
    b = sc.check_parity(pkg, gpu_lib, cu8, "-v", 1, device=torch, max_batch_mib=1)
    assert sc.as_tuples(a[0]) == sc.as_tuples(b[0]) and a[1] == b[1]


def test_1gib_device_resident_time_chunks(gpu_lib, pkg):
    """a 1 GiB capture through process_device: the restatement, and three time chunks merged (64 MiB batches: the pool
    holds a whole batch).  At 256 MiB batches this dense capture keeps more than the 64 MiB pool: the snippets that lost
    a granule come out with lost = 1 and no bytes, their batches count as overflow batches, and the others are exact"""
    import torch
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    n = 1 << 30
    em, far = bc.planted_emitters()
    cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=em, seed=0xB20000A3, device="cuda")
    host = cap.cpu().numpy()
    seq = {}
    for mode, mib in ((1, 64), (2, 64), (1, 256)):
        with pkg.WmbusB200("-v", lib=gpu_lib, burst_level=bc.DEFAULT_LEVEL, snippets=mode, max_batch_mib=mib) as ctx:
            lines, info = ctx.process_device(cap.data_ptr(), n, flush=True, info=True)
            recs, data = ctx.take_snippets()
            bursts = ctx.take_bursts()
            st = ctx.stats()
        want = sc.restate(host, 2, bursts, sc.matches_ok(info), mode)
        got = sc.as_tuples(recs)
        assert len(got) == len(want) > 100
        lost = recs["lost"] == 1
        assert (st.overflow_batches > 0) == bool(lost.any()) and (mib == 64) == (not lost.any())
        for g, x, w in zip(got, data, want):
            if g[7]:
                assert g[:3] + g[4:7] == w[0][:3] + w[0][4:7] and g[3] == 0 and x == b""
            else:
                assert g == w[0] and x == w[1]
        if mib == 64:
            seq[mode] = (recs, data)
    parts, infos = [], []
    for rank in range(3):
        with pkg.WmbusB200("-v", lib=gpu_lib, burst_level=bc.DEFAULT_LEVEL, snippets=1, max_batch_mib=64) as ctx:
            out, *_ = shard.decode_time_chunk(ctx, lambda a, b: ctx.push_device(cap.data_ptr() + a, b - a), n, 2, rank,
                                              3, info=True, bursts=True, snippets=True)
        infos.append(out[1])
        parts.append(out[3])
    info = np.concatenate(infos)
    for mode in (1, 2):
        r, d = shard.merge_snippets(parts, info, undecoded=mode == 2)
        assert sc.as_tuples(r) == sc.as_tuples(seq[mode][0]) and d == seq[mode][1]


def test_replay(gpu_lib, pkg):
    total = 0
    for name, flags in sc.CORPUS:
        cu8 = sc.s_capture() if name == "s_capture" else rc.cached_capture(name)
        n = sc.check_replay(pkg, gpu_lib, cu8, flags)
        if "-s" in flags:
            assert sc.check_replay(pkg, gpu_lib, cu8, flags, seek=False) == n
        total += n
    assert total >= 60


def test_snippet_kernels_do_not_spill(pkg):
    use = sc.resource_usage(pkg.library_path())
    ksn = {k: v for k, v in use.items() if "ksn_" in k}
    assert len(ksn) == 2, sorted(use)
    for k, v in ksn.items():
        assert v.get("STACK", 0) == 0 and v.get("LOCAL", 0) == 0, (k, v)


def test_default_path_sass_unchanged(pkg):
    """every kernel the parent commit had is bit-identical machine code (tests/golden/sass_default_path.json holds the
    digests of the library built before the snippet kernels were added)"""
    want = json.load(open(os.path.join(GOLDEN, "sass_default_path.json")))
    got = sc.sass_digests(pkg.library_path())
    assert {k: got.get(k) for k in want} == want
