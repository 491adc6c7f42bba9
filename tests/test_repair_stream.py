"""`not gpu`: erasure repair on the streaming path (wmb_set_repair, wmb_take_repairs; wmbus_b200_framer.h) on the CPU
build.  The records of a context that frames for itself equal, field by field, the restatement from manual framing
(tests/repair_stream_cases.py) at every batching; planted telegrams come back as sent; lines, records, bursts and
statistics do not move; time chunks merge to the sequential records; the setter, the queue and the CLI's file."""
import ctypes as C
import hashlib
import importlib
import os
import subprocess

import numpy as np
import pytest

import receiver_cases
import repair_cases as rc
import repair_stream_cases as rs
from conftest import HOSTSIM_SO

BATCH_M = rs.MIB // 4                  # decimated samples of a 1 MiB batch at -d 2


@pytest.fixture(scope="module")
def flipped():
    return rs.flipped_capture()


@pytest.fixture(scope="module")
def flipped_want(hostsim_lib, pkg, flipped):
    return rs.restated(pkg, hostsim_lib, flipped[0], "-v", (1, 2, 3))


@pytest.fixture(scope="module")
def plain_runs(hostsim_lib, pkg, flipped):
    """the capture decoded once per e_max (1 MiB batches) with quality and bursts on, and once with repair off"""
    return {e: rs.stream(pkg, hostsim_lib, flipped[0], "-v", e, quality=True, burst_level=(14, 14)) for e in (0, 1, 2, 3)}


@pytest.mark.parametrize("e_max", (1, 2, 3))
def test_records_equal_the_restatement_1mib(plain_runs, flipped_want, e_max):
    got = plain_runs[e_max][0]
    assert got == flipped_want[e_max]
    assert sum(1 for t in got if t[4] == rc.REPAIRED) >= 20


@pytest.mark.parametrize("e_max,batching", [(1, "one"), (2, "uneven"), (3, "one"), (3, "uneven")])
def test_records_equal_the_restatement_other_batchings(hostsim_lib, pkg, flipped, flipped_want, e_max, batching):
    got = rs.stream(pkg, hostsim_lib, flipped[0], "-v", e_max, batching, batch_mib=8 if batching == "one" else 1)[0]
    assert got == flipped_want[e_max]


def test_dense_false_matches(hostsim_lib, pkg, flipped):
    """access-code errors (3, 6): many false S1 matches abort.  The sync-error capture holds no damaged telegram, so
    REPAIRED comes from the flipped-emitter capture at the same setting; TOO_MANY and UNREPAIRABLE from both"""
    kw = dict(access_code_errors=(3, 6))
    seen = set()
    for cu8 in (receiver_cases.cached_capture("sync_errors_1m6"), flipped[0]):
        want = rs.restated(pkg, hostsim_lib, cu8, "-v", (1, 3), **kw)
        for e_max in (1, 3):
            for batching, mib in (("1mib", 1), ("one", 8)):
                got = rs.stream(pkg, hostsim_lib, cu8, "-v", e_max, batching, batch_mib=mib, **kw)[0]
                assert got == want[e_max], (e_max, batching, len(got), len(want[e_max]))
        seen |= {t[4] for t in want[3]}
        if len(seen) == 2:
            assert seen == {rc.TOO_MANY, rc.UNREPAIRABLE}, seen
    assert {rc.REPAIRED, rc.TOO_MANY, rc.UNREPAIRABLE} <= seen, seen


def test_waiting_s1_repair_crosses_batches(hostsim_lib, pkg):
    """S1 REPAIRED records whose abort bit (where the framer books the candidate) and bit P - 1 lie in different 1 MiB
    batches: a flipped S1 emitter timed so that a telegram straddles the first batch boundary"""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    em = synth.Emitter("S1", 0x19131290, amp=80.0, offset_hz=2e3, l_field=0x19, period_s=0.29, start_s=0.316, seed=32,
                       data_flips=(16 * 5 + 1, 16 * 20 + 6))
    cu8, _plan = synth.synth_capture(2 << 20, emitters=[em], seed=0xB2000008)
    cu8 = np.ascontiguousarray(cu8.numpy())
    lib = hostsim_lib
    lib.wmb_frame_decode.argtypes = [C.c_void_p, C.c_void_p]
    abort_at = {}
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        ctx.push(cu8.ctypes.data, len(cu8))
        arr, k = ctx.poll(flush=True)
        for i in range(k):
            d = pkg.WmbDecoded()
            lib.wmb_frame_decode(C.addressof(arr[i]), C.addressof(d))
            if d.status == 0:
                abort_at[(arr[i].algo, arr[i].sync_sample)] = d.end_sample
    want = rs.restated(pkg, lib, cu8, "-v", (2,))[2]
    got = rs.stream(pkg, lib, cu8, "-v", 2)[0]
    assert got == want
    crossing = [t for t in got if t[2] == 1 and t[4] == rc.REPAIRED and not t[7]
                and abort_at[(t[3], t[0])] // BATCH_M != t[1] // BATCH_M]
    assert len(crossing) == 2, got                   # rla and t2a


def test_planted_telegrams_come_back_as_sent(plain_runs, flipped):
    _, plan, ems = flipped
    flipped_sent = {ems[p.emitter].payload(p.k): p for p in plan if ems[p.emitter].data_flips}
    alone = {d for d, p in flipped_sent.items()
             if not any(q is not p and q.start_iq < p.start_iq + p.n_iq and p.start_iq < q.start_iq + q.n_iq for q in plan)}
    assert len(alone) >= 15
    for e_max in (1, 2, 3):
        got = [t[-1] for t in plain_runs[e_max][0] if t[4] == rc.REPAIRED]
        assert set(got) <= set(flipped_sent), "a repaired datagram that was never sent"
        assert alone <= set(got), (e_max, len(alone - set(got)))


def test_nothing_else_moves(plain_runs):
    _, lines0, info0, qual0, bursts0, st0 = plain_runs[0]
    assert plain_runs[0][0] == []
    for e_max in (1, 2, 3):
        _, lines, info, qual, bursts, st = plain_runs[e_max]
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
        assert st.kernel_launches - st0.kernel_launches == st.batches + 1      # one K4R per gather (the flush's too)
        assert st.d2h_bytes > st0.d2h_bytes


# ---- time chunks -----------------------------------------------------------------------------------------------------

def test_time_chunks_merge_to_the_sequential_records(hostsim_lib, pkg, plain_runs, flipped):
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    cu8 = flipped[0]
    parts = []
    with pkg.WmbusB200("-v", lib=hostsim_lib, repair=2, max_batch_mib=1) as ctx:
        def push(lo, hi):
            ctx.push(cu8.ctypes.data + lo, hi - lo)
        for rank in range(3):
            out, _ds, _de, _start = shard.decode_time_chunk(ctx, push, len(cu8), 2, rank, 3, repairs=True)
            parts.append(out[-1])
    merged = [rs.record_tuple(r) for r in shard.merge_repairs(parts)]
    assert merged == plain_runs[2][0]


def test_pending_before_counts_a_waiting_repair(hostsim_lib, pkg, plain_runs, flipped):
    cu8 = flipped[0]
    _, plan, ems = flipped
    # an S1 telegram repaired from an abort, alone on the air; its record's sync and end sample
    s1 = [t for t in plain_runs[2][0] if t[2] == 1 and t[4] == rc.REPAIRED and not t[7]]
    starts = sorted(p.start_iq // 2 for p in plan)
    pick = None
    for t in s1:
        sync, end = t[0], t[1]
        others = [m for m in starts if sync - 40000 < m < end + 4000 and abs(m - sync) > 30000]
        if not others and end - sync > 6000:
            pick = t
            break
    assert pick is not None
    sync, end = pick[0], pick[1]
    gran = 4096 * 2                                      # bytes of one batch granule at -d 2 (1024 decimated samples)
    cut = ((sync + end) // 2 * 4) // gran * gran          # a push that ends between the abort and bit P - 1
    got = {}
    for e_max in (0, 2):
        with pkg.WmbusB200("-v", lib=hostsim_lib, repair=e_max, max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, cut)
            got[e_max] = ctx.pending_before(sync + 1)
    assert got[2] >= 1 and got[0] == 0, got


def test_boundary_state_tells_e_max_apart(hostsim_lib, pkg, flipped):
    cu8 = flipped[0]
    digests = set()
    for e_max in (0, 1, 2, 3):
        with pkg.WmbusB200("-v", lib=hostsim_lib, repair=e_max, max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, 3 * rs.MIB)
            digests.add(hashlib.sha256(ctx.boundary_state()).digest())
    assert len(digests) == 4


# ---- setter, queue, CLI ----------------------------------------------------------------------------------------------

def test_setter_and_queue(hostsim_lib, pkg, flipped):
    lib = hostsim_lib
    cu8 = flipped[0]
    n = 4 * rs.MIB
    assert lib.wmb_set_repair(None, 1) == -1
    with pkg.WmbusB200("-v", lib=lib, manual_frames=1) as ctx:
        assert lib.wmb_set_repair(ctx._ctx, 1) == -1 and b"manual_frames" in lib.wmb_last_error()
    with pkg.WmbusB200("-v", lib=lib, max_batch_mib=1) as ctx:
        assert lib.wmb_set_repair(ctx._ctx, 4) == -1                   # WMB_E_INVAL
        assert lib.wmb_set_repair(ctx._ctx, 3) == 0
        ctx.push(cu8.ctypes.data, n)
        assert lib.wmb_set_repair(ctx._ctx, 1) != 0 and b"after samples were pushed" in lib.wmb_last_error()
        out = (pkg.WmbRepairRecord * 4)()
        k = C.c_size_t(0)
        assert lib.wmb_take_repairs(ctx._ctx, out, 1, C.byref(k)) == 0 and k.value == 1       # a partial take
        rest = ctx.take_repairs()
        assert len(rest) >= 2
        first = rs.record_tuple(out[0])
        ctx.reset()                                                    # the setting survives, the queue is emptied
        ctx.push(cu8.ctypes.data, n)
        ctx.reset()
        assert ctx.take_repairs() == []
        ctx.push(cu8.ctypes.data, n)
        again = ctx.take_repairs()
        assert [rs.record_tuple(r) for r in again[:1 + len(rest)]] == [first] + [rs.record_tuple(r) for r in rest]
        ctx.seek(0)
        assert lib.wmb_set_repair(ctx._ctx, 3) == 0                    # valid right after a seek
        ctx.push(cu8.ctypes.data, n)
        assert len(ctx.take_repairs()) == len(again)


def cli(args, cu8, env_extra):
    exe = os.path.join(os.path.dirname(HOSTSIM_SO), "rtl_wmbus_hostsim")
    env = dict(os.environ, WMBUS_B200_BATCH_MIB="1")
    env.update(env_extra)
    return subprocess.run([exe] + args, input=cu8.tobytes(), capture_output=True, env=env, timeout=300)


def blank_ts(line, prefixed):
    f = line.split(";")
    f[4 if prefixed else 3] = "TS"
    return ";".join(f)


def test_cli_repaired_file(hostsim_lib, pkg, flipped, tmp_path):
    cu8 = flipped[0]
    path = tmp_path / "repaired.txt"
    plain = cli(["-v"], cu8, {})
    assert plain.returncode == 0, plain.stderr
    for e_max in ("1", "3"):
        r = cli(["-v"], cu8, {"WMBUS_B200_REPAIRED": str(path), "WMBUS_B200_REPAIR_ERASURES": e_max})
        assert r.returncode == 0, r.stderr
        assert [blank_ts(l, True) for l in r.stdout.decode().splitlines()] == \
            [blank_ts(l, True) for l in plain.stdout.decode().splitlines()]
        recs, *_ = rs.stream(pkg, hostsim_lib, cu8, "-v", int(e_max))
        with pkg.WmbusB200("-v", lib=hostsim_lib, repair=int(e_max), max_batch_mib=1) as ctx:
            ctx.push(cu8.ctypes.data, len(cu8))
            ctx.poll_flush()
            want = [ctx.repaired_line(x, b"rla;" if x.algo == 0 else b"t2a;") for x in ctx.take_repairs()
                    if x.repair.outcome == rc.REPAIRED]
        got = [blank_ts(l, True) for l in path.read_text().splitlines()]
        assert got == want and len(got) >= 20
    r = cli([], cu8[:1 << 20], {"WMBUS_B200_REPAIRED": str(path)})       # without -v: no prefix; default e_max 1
    assert r.returncode == 0


@pytest.mark.parametrize("env", [{"WMBUS_B200_REPAIR_ERASURES": "2"},
                                 {"WMBUS_B200_REPAIRED": "/nonexistent-dir/x", "WMBUS_B200_REPAIR_ERASURES": "1"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_ERASURES": "0"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_ERASURES": "4"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_ERASURES": "x"},
                                 {"WMBUS_B200_REPAIRED": "{tmp}", "WMBUS_B200_REPAIR_ERASURES": ""}])
def test_cli_bad_environment_fails_at_start_up(hostsim_lib, tmp_path, env):
    env = {k: v.replace("{tmp}", str(tmp_path / "r.txt")) for k, v in env.items()}
    r = cli(["-v"], np.zeros(8192, np.uint8), env)
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_" in r.stderr, r.stderr
