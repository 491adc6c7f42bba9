"""`not gpu`: the C1 soft repair on the streaming path (wmb_set_repair_soft; wmbus_b200_framer.h) on the CPU build.  The
records of a context that frames for itself equal the restatement from manual framing with soft values
(soft_repair_cases.restated_stream) at k_max 1, 4 and 6; C1 telegrams with weak chips come back as sent; lines,
records, bursts and statistics do not move; time chunks merge to the sequential records; setter, boundary state, CLI."""
import hashlib
import importlib

import numpy as np
import pytest

import repair_cases as rc
import repair_stream_cases as rs
import soft_repair_cases as sc
from test_repair_stream import blank_ts, cli

K_MAXES = (1, 4, 6)


@pytest.fixture(scope="module")
def weak():
    return sc.weak_capture()


@pytest.fixture(scope="module")
def weak_want(hostsim_lib, pkg, weak):
    return sc.restated_stream(pkg, hostsim_lib, weak[0], "-v", 2, (0,) + K_MAXES)


@pytest.fixture(scope="module")
def runs(hostsim_lib, pkg, weak):
    """the capture in 1 MiB batches at e_max 2, with quality and bursts on, per k_max (0: the soft repair off)"""
    return {k: rs.stream(pkg, hostsim_lib, weak[0], "-v", 2, quality=True, burst_level=(14, 14), repair_soft=k)
            for k in (0,) + K_MAXES}


def c1_records(recs):
    return [t for t in recs if t[2] == 0 and t[7] and (t[4] != rc.REPAIRED or t[11] == b"C1")]


@pytest.mark.parametrize("k_max", K_MAXES)
def test_records_equal_the_restatement(runs, weak_want, k_max):
    assert runs[k_max][0] == weak_want[k_max]
    assert sum(1 for t in c1_records(runs[k_max][0]) if t[4] == rc.REPAIRED) >= 20


@pytest.mark.parametrize("k_max,batching", [(4, "one"), (6, "uneven")])
def test_records_equal_the_restatement_other_batchings(hostsim_lib, pkg, weak, weak_want, k_max, batching):
    got = rs.stream(pkg, hostsim_lib, weak[0], "-v", 2, batching, batch_mib=8 if batching == "one" else 1,
                    repair_soft=k_max)[0]
    assert got == weak_want[k_max]


def test_weak_telegrams_come_back_as_sent(runs, weak):
    _, plan, ems = weak
    sent = {ems[p.emitter].payload(p.k) for p in plan}
    weak_sent = {ems[p.emitter].payload(p.k): p for p in plan if ems[p.emitter].weak_flips}
    alone = {d for d, p in weak_sent.items()
             if not any(q is not p and q.start_iq < p.start_iq + p.n_iq and p.start_iq < q.start_iq + q.n_iq for q in plan)}
    assert len(alone) >= 10
    for k in K_MAXES:
        got = {t[-1] for t in c1_records(runs[k][0]) if t[4] == rc.REPAIRED}
        assert got <= sent, "a repaired datagram that was never sent"
        assert alone <= got, (k, len(alone - got))


def test_off_means_off(runs):
    """k_max 0: C1 lines stay UNREPAIRABLE.  Any k_max: the T1 / S1 records, lines, records, bursts and statistics but
    kernel_launches (k3_soft and K4S per gather) and d2h_bytes are those of k_max 0"""
    recs0, lines0, info0, qual0, bursts0, st0 = runs[0]
    assert c1_records(recs0) and all(t[4] == rc.UNREPAIRABLE for t in c1_records(recs0))
    for k in K_MAXES:
        recs, lines, info, qual, bursts, st = runs[k]
        assert [t for t in recs if t not in c1_records(recs)] == [t for t in recs0 if t not in c1_records(recs0)]
        assert lines == lines0
        assert info.tobytes() == info0.tobytes() and qual.tobytes() == qual0.tobytes()
        assert bursts.tobytes() == bursts0.tobytes()
        for name, _t in st._fields_:
            if name in ("kernel_launches", "d2h_bytes") or name.endswith("_ms"):
                continue
            a, b = getattr(st, name), getattr(st0, name)
            if not isinstance(a, (int, float)):
                a, b = bytes(a), bytes(b)
            assert a == b, name
        assert st.kernel_launches - st0.kernel_launches == 2 * (st.batches + 1)
        assert st.d2h_bytes >= st0.d2h_bytes


def test_time_chunks_merge_to_the_sequential_records(hostsim_lib, pkg, runs, weak):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = weak[0]
    parts = []
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_soft=4, max_batch_mib=1) as ctx:
        def push(lo, hi):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
        for rank in range(3):
            out, _ds, _de, _start = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, repairs=True)
            parts.append(out[-1])
    assert [rs.record_tuple(r) for r in shard.merge_repairs(parts)] == runs[4][0]


def test_setter_and_boundary_state(hostsim_lib, pkg, weak):
    lib = hostsim_lib
    cu8 = weak[0]
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        assert lib.wmb_set_repair_soft(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
    with pkg.WmbusB200("-v", lib=lib) as ctx:
        assert lib.wmb_set_soft_bits(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
        assert lib.wmb_set_repair_soft(ctx._ctx, 7) == -1
        assert lib.wmb_set_repair_soft(ctx._ctx, 6) == 0
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert lib.wmb_set_repair_soft(ctx._ctx, 1) != 0 and b"after samples were pushed" in lib.wmb_last_error()
        ctx.reset()
        assert lib.wmb_set_repair_soft(ctx._ctx, 2) == 0
        ctx.seek(0)
        assert lib.wmb_set_repair_soft(ctx._ctx, 0) == 0
    digests = set()
    for k in (0, 1, 6):
        with pkg.WmbusB200("-v", lib=lib, repair=2, repair_soft=k, max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, 3 * rs.MIB)
            digests.add(hashlib.sha256(ctx.boundary_state()).digest())
    assert len(digests) == 3


def test_cli_repaired_file(hostsim_lib, pkg, weak, tmp_path):
    cu8 = weak[0]
    path = tmp_path / "repaired.txt"
    plain = cli(["-v"], cu8, {})
    assert plain.returncode == 0, plain.stderr
    r = cli(["-v"], cu8, {"WMBUS_B200_REPAIRED": str(path), "WMBUS_B200_REPAIR_ERASURES": "2",
                          "WMBUS_B200_REPAIR_SOFT_BITS": "4"})
    assert r.returncode == 0, r.stderr
    assert [blank_ts(l, True) for l in r.stdout.decode().splitlines()] == \
        [blank_ts(l, True) for l in plain.stdout.decode().splitlines()]
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, repair_soft=4, max_batch_mib=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        ctx.poll_flush()
        want = [ctx.repaired_line(x, b"rla;" if x.algo == 0 else b"t2a;") for x in ctx.take_repairs()
                if x.repair.outcome == rc.REPAIRED]
    got = [blank_ts(l, True) for l in path.read_text().splitlines()]
    assert got == want and sum(1 for l in got if ";C1;" in l) >= 20


@pytest.mark.parametrize("env", [{"WMBUS_B200_REPAIR_SOFT_BITS": "2"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_SOFT_BITS": "0"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_SOFT_BITS": "7"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_SOFT_BITS": "x"}])
def test_cli_bad_soft_setting_fails_at_start_up(hostsim_lib, tmp_path, env):
    env = {k: v.replace("{tmp}", str(tmp_path / "r.txt")) for k, v in env.items()}
    r = cli(["-v"], np.zeros(8192, np.uint8), env)
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_REPAIR_SOFT_BITS" in r.stderr, r.stderr
