"""`not gpu`: telegram records (wmb_group_telegrams, wmb_set_telegrams / wmb_take_telegrams) on the CPU-simulation build
of the library: every record against the restatement (tests/telegram_cases.py) on the committed captures under six flag
sets and three repair settings, the invariants, made-up records at the rule's edges, independence from batch size,
push size, thread order, seek and time chunks, off means off, setter rules and the CLI's file."""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import orc
import receiver_cases as rc
import telegram_cases as tc
from conftest import ROOT

CAPTURES = sorted(rc.COMMITTED)


@pytest.mark.parametrize("name", CAPTURES)
def test_parity_committed(hostsim_lib, pkg, name):
    """every record equals the rule over the run's own lines and repairs, under each flag set and repair setting; a
    -r 0 run's decoded datagrams are a subset of the default run's"""
    cu8 = rc.cached_capture(name)
    n_dec = 0
    for rname, rp in tc.REPAIRS.items():
        runs = {}
        for flags in tc.capture_flags(name):
            recs, data, *_ = tc.check_parity(pkg, hostsim_lib, cu8, flags, repair=rp, max_batch_mib=1)
            runs[flags] = tc.decoded_set(recs, data)
            n_dec += len(runs[flags])
        base = "-d 3" if "-d 3" in rc.COMMITTED[name][0] else ""
        assert runs[(base + " -r 0").strip()] <= runs[base], (name, rname)
    assert n_dec > 0


# ---- wmb_group_telegrams on made-up records ------------------------------------------------------------------------

def made_up(cands):
    """cands: (chain, sync, algo, kind, ok, mode, datagram) with kind "line" or "repair" -> (info, lines, repairs)"""
    info = np.zeros(sum(1 for c in cands if c[3] == "line"), _info_dtype())
    lines, reps, i = [], [], 0
    for ch, s, algo, kind, ok, mode, data in cands:
        d = _pkg().WmbDecoded()
        d.status, d.mode, d.crc_ok, d.len = 1, mode.encode(), int(ok), len(data)
        C.memmove(d.datagram, data, len(data))
        if len(data) >= 8:
            d.serial = int.from_bytes(data[4:8], "little")
        if kind == "line":
            info[i]["sync_sample"], info[i]["chain"], info[i]["algo"], info[i]["crc_ok"] = s, ch, algo, int(ok)
            lines.append(d)
            i += 1
        else:
            r = _pkg().WmbRepairRecord()
            r.sync_sample, r.chain, r.algo = s, ch, algo
            r.repair.outcome = 1 if ok else 4                                   # REPAIRED / UNREPAIRABLE
            r.repair.line = d
            reps.append(r)
    return info, lines, reps


def _pkg():
    return importlib.import_module("rtl-wmbus_b200")


def _info_dtype():
    return _pkg().line_info_dtype()


def group(lib, cands):
    """the library's records of made-up candidates, checked against the restatement"""
    info, lines, reps = made_up(cands)
    recs, data = _pkg().group_telegrams(lib, info, lines, reps)
    want = tc.restate([(c[0], c[1], {("line", 1): 1, ("line", 0): 2, ("repair", 1): 4, ("repair", 0): 8}[(c[3], c[2])],
                        bool(c[4]), c[5], c[6]) for c in cands if c[3] == "line" or c[4]])
    assert tc.as_tuples(recs) == [w[0] for w in want] and data == [w[1] for w in want]
    return recs, data


HDR = bytes.fromhex("2c446850230020717007")          # L C M M A A A A V T
A = HDR + bytes([0x7A]) + bytes(range(20))
B = HDR[:4] + bytes.fromhex("39873320") + HDR[8:] + bytes([0x72]) + bytes(range(30, 50))


def test_group_collision(hostsim_lib):
    """two meters on one chain within W: one group, two decoded records sharing its first match, in byte order"""
    recs, data = group(hostsim_lib, [(0, 1000, 1, "line", 1, "T1", B), (0, 1007, 0, "line", 1, "T1", B),
                                     (0, 1050, 1, "line", 1, "T1", A), (0, 1060, 0, "line", 0, "T1", A[:5])])
    assert len(recs) == 2 and set(recs["sync_sample"]) == {1000} and (recs["failed"] == 1).all()
    assert data == [A, B] and list(recs["sources"]) == [1, 3]
    assert [hex(x) for x in recs["id"]] == [hex(0x71200023), hex(0x20338739)] and list(recs["ci"]) == [0x7A, 0x72]


def test_group_long_failed_span(hostsim_lib):
    """a failed candidate whose (wrong) end lies past the next telegram does not swallow it: only matches link"""
    info, lines, reps = made_up([(0, 1000, 1, "line", 0, "T1", A), (0, 1000 + tc.W[0] + 500, 1, "line", 1, "T1", A)])
    info[0]["end_sample"] = 1000 + 50000
    recs, data = _pkg().group_telegrams(hostsim_lib, info, lines, reps)
    assert list(recs["decoded"]) == [0, 1] and list(recs["failed"]) == [1, 0] and data == [b"", A]
    assert recs[0]["valid"] == 0 and recs[0]["len"] == 0 and recs[0]["mode"] == b""


def test_group_repair_beside_failed_twin(hostsim_lib):
    """a repaired line beside its CRC-failed twin and the other bit sync's good line: one record, failed 1"""
    recs, data = group(hostsim_lib, [(0, 500, 1, "line", 0, "C1", A), (0, 500, 1, "repair", 1, "C1", A),
                                     (0, 508, 0, "line", 1, "C1", A), (0, 508, 0, "repair", 0, "C1", A)])
    assert len(recs) == 1 and recs[0]["sources"] == 2 | 4 and recs[0]["failed"] == 1 and data == [A]


@pytest.mark.parametrize("chain", [0, 1])
def test_group_w_edge(hostsim_lib, chain):
    """matches exactly W apart link, W + 1 apart do not"""
    m = "T1" if chain == 0 else "S1"
    w = tc.W[chain]
    recs, _ = group(hostsim_lib, [(chain, 10000, 1, "line", 1, m, A), (chain, 10000 + w, 0, "line", 1, m, A)])
    assert len(recs) == 1 and recs[0]["sources"] == 3
    recs, _ = group(hostsim_lib, [(chain, 10000, 1, "line", 1, m, A), (chain, 10001 + w, 0, "line", 1, m, A)])
    assert len(recs) == 2 and list(recs["sync_sample"]) == [10000, 10001 + w]
    # a chain of matches each W apart is one group (transitive closure); the other chain never joins
    recs, _ = group(hostsim_lib, [(chain, 0, 1, "line", 1, m, A), (chain, w, 0, "line", 0, m, A),
                                  (chain, 2 * w, 1, "line", 1, m, B), (1 - chain, w, 1, "line", 1, "C1", A)])
    assert list(recs["chain"]) == [chain, chain, 1 - chain] and list(recs["sync_sample"]) == [0, 0, w]
    assert list(recs["failed"]) == [1, 1, 0]


def test_group_short_datagrams(hostsim_lib):
    """a datagram too short for a header field clears that field's valid bit and leaves it 0"""
    cands = [(0, 100000 * (k + 1), 1, "line", 1, "T1", A[:k]) for k in (0, 1, 3, 4, 7, 8, 9, 10, 11)]
    recs, data = group(hostsim_lib, cands)
    want = {0: 0, 1: 1, 3: 3, 4: 7, 7: 7, 8: 15, 9: 31, 10: 63, 11: 127}
    assert [int(r["valid"]) for r in recs] == list(want.values())
    assert recs[2]["manuf"] == b"" and recs[3]["manuf"] == bytes([((0x5068 >> 10) & 31) + 64, ((0x5068 >> 5) & 31) + 64,
                                                                   (0x5068 & 31) + 64])
    assert recs[4]["id"] == 0 and recs[5]["id"] == 0x71200023 and recs[0]["decoded"] == 1 and recs[0]["len"] == 0


def test_group_bounds(hostsim_lib):
    """out must hold lines + repairs records and data the verified bytes; a chain outside 0..1 is refused"""
    info, lines, reps = made_up([(0, 5, 1, "line", 1, "T1", A), (1, 9, 0, "line", 1, "S1", B)])
    out = np.zeros(2, _pkg().telegram_dtype())
    buf = np.zeros(len(A) + len(B), np.uint8)
    n = C.c_size_t(0)
    dec = (_pkg().WmbDecoded * 2)(*lines)
    f = hostsim_lib.wmb_group_telegrams
    assert f(info.ctypes.data, dec, 2, None, 0, out.ctypes.data, 1, buf.ctypes.data, len(buf), C.byref(n)) == -1
    assert f(info.ctypes.data, dec, 2, None, 0, out.ctypes.data, 2, buf.ctypes.data, len(buf) - 1, C.byref(n)) == -1
    assert f(info.ctypes.data, dec, 2, None, 0, out.ctypes.data, 2, buf.ctypes.data, len(buf), C.byref(n)) == 0
    assert n.value == 2
    assert f(None, None, 0, None, 0, None, 0, None, 0, C.byref(n)) == 0 and n.value == 0
    info[1]["chain"] = 2
    assert f(info.ctypes.data, dec, 2, None, 0, out.ctypes.data, 2, buf.ctypes.data, len(buf), C.byref(n)) == -1


# ---- the streaming path --------------------------------------------------------------------------------------------

def test_batches_pushes_seek(hostsim_lib, pkg):
    """one batch or many, ragged pushes, one batch granule (4096 d bytes) per push, a seek: the same records"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    rp = tc.REPAIRS["soft"]
    base = tc.check_parity(pkg, hostsim_lib, cu8, "-v", repair=rp, max_batch_mib=256)
    runs = [tc.check_parity(pkg, hostsim_lib, cu8, "-v", repair=rp, max_batch_mib=1),
            tc.check_parity(pkg, hostsim_lib, cu8, "-v", repair=rp, pushes=[12345, 1 << 19, 4096 * 3 + 17, 777777],
                            max_batch_mib=1),
            tc.check_parity(pkg, hostsim_lib, cu8, "-v", repair=rp, pushes=[8192] * (len(cu8) // 8192), max_batch_mib=1)]
    for r in runs:
        assert tc.as_tuples(r[0]) == tc.as_tuples(base[0]) and r[1] == base[1]
    seek = 2048 * 2 * 37
    r = tc.check_parity(pkg, hostsim_lib, cu8, "-v", repair=rp, seek=seek, max_batch_mib=1)
    shifted = [(t[0] - seek // 2,) + t[1:] for t in tc.as_tuples(r[0])]
    assert shifted == tc.as_tuples(base[0]) and r[1] == base[1]
    cu8 = rc.cached_capture("excerpt_issue48_2m4.cu8")
    a = tc.check_parity(pkg, hostsim_lib, cu8, "-v -d 3 -s", repair=rp, pushes=[12288] * 40, max_batch_mib=1)
    b = tc.check_parity(pkg, hostsim_lib, cu8, "-v -d 3 -s", repair=rp, max_batch_mib=256)
    assert tc.as_tuples(a[0]) == tc.as_tuples(b[0]) and len(a[0])


@pytest.mark.parametrize("order", ["1", "2"])
def test_thread_orders(order):
    """the simulated threads of every phase backwards / scrambled: the same records as in the default order"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, telegram_cases as tc, receiver_cases as rc;"
            "from conftest import HOSTSIM_SO; pkg = importlib.import_module('rtl-wmbus_b200'); lib = pkg.load_library(HOSTSIM_SO);"
            "r = tc.check_parity(pkg, lib, rc.cached_capture('synth_mixed_1m6.cu8'), '-v', repair=tc.REPAIRS['soft'], max_batch_mib=1);"
            "print(repr(tc.as_tuples(r[0])))" % (ROOT, os.path.join(ROOT, "tests")))
    out = {}
    for o in ("0", order):
        env = dict(os.environ, WMB_HOSTSIM_ORDER=o)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0, r.stderr[-3000:]
        out[o] = r.stdout
    assert out["0"] == out[order] and len(out["0"]) > 100


def test_waits_for_telegram_in_flight(hostsim_lib, pkg):
    """a run-length telegram cut by dead air is in flight: its group is not handed out until it ends, and neither is
    any later group"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1) as ctx:
        lines, info = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
    r = [x for l, x in zip(lines, info) if x["crc_ok"] and x["chain"] == 0 and l.startswith("rla;")][2]
    mid = (int(r["sync_sample"]) + int(r["end_sample"])) // 2
    cut = mid * 4 // 4096 * 4096
    dead = np.full(1 << 20, 127, np.uint8)
    cap = np.ascontiguousarray(np.concatenate([cu8[:cut], dead, cu8[cut:]]))
    whole = tc.check_parity(pkg, hostsim_lib, cap, "-v", max_batch_mib=1)
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, telegrams=True) as ctx:
        ctx.push(cap.ctypes.data, cut + len(dead))
        assert ctx.pending_before(int(r["sync_sample"]) + 1) > 0
        early, _ = ctx.take_telegrams()
        assert len(early) and (early["sync_sample"] < r["sync_sample"]).all()
        ctx.push(cap.ctypes.data + cut + len(dead), len(cap) - cut - len(dead))
        ctx.poll_flush()
        late, _ = ctx.take_telegrams()
    assert tc.as_tuples(early) + tc.as_tuples(late) == tc.as_tuples(whole[0])


def test_time_chunks(hostsim_lib, pkg):
    """three time chunks: merge_telegrams over the merged lines and repairs gives the sequential records"""
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    rp = tc.REPAIRS["soft"]
    for name, flags, d in (("synth_mixed_1m6.cu8", "-v", 2), ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s", 3)):
        cu8 = rc.cached_capture(name)
        seq = tc.product(pkg, hostsim_lib, cu8, flags, repair=rp, max_batch_mib=1)
        parts, infos, reps = [], [], []
        for rank in range(3):
            with pkg.WmbusB200(flags, lib=hostsim_lib, max_batch_mib=1, **rp) as ctx:
                out, *_ = shard.decode_time_chunk(ctx, lambda a, b: ctx.push(cu8.ctypes.data + a, b - a), len(cu8), d,
                                                  rank, 3, info=True, repairs=True)
            parts.append(out[0])
            infos.append(out[1])
            reps.append(out[2])
        lines, info = shard.merge_lines(parts, infos)
        recs, data = shard.merge_telegrams(lines, info, shard.merge_repairs(reps), lib=hostsim_lib)
        assert tc.as_tuples(recs) == tc.as_tuples(seq[0]) and data == seq[1] and len(recs)


def test_off_means_off(hostsim_lib, pkg):
    """off is a context that never heard of telegrams; on, lines, records, repairs and every statistic are the same:
    the feature launches and copies nothing"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    out = []
    for kw in ({}, dict(telegrams=False), dict(telegrams=True)):
        with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, repair=3, **kw) as ctx:
            lines, info = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            reps = ctx.take_repairs()
            t, _ = ctx.take_telegrams()
            st = ctx.stats()
        out.append((lines, info, [bytes(r) for r in reps], t, st))
    base = out[0]
    for i, (lines, info, reps, t, st) in enumerate(out):
        assert lines == base[0] and np.array_equal(info, base[1]) and reps == base[2]
        for f, _ in st._fields_:
            if f.endswith("_ms"):
                continue
            v, b = getattr(st, f), getattr(base[4], f)
            assert (list(map(list, v)) == list(map(list, b))) if hasattr(v, "__len__") else v == b, f
        assert bool(len(t)) == (i == 2)


def test_setter_rules(hostsim_lib, pkg):
    L = hostsim_lib
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    with pkg.WmbusB200("-v", lib=L) as ctx:
        assert L.wmb_set_telegrams(ctx._ctx, 2) == -1 and L.wmb_set_telegrams(ctx._ctx, -1) == -1
        ctx.set_telegrams(True)
        ctx.push(cu8.ctypes.data, 1 << 20)
        assert L.wmb_set_telegrams(ctx._ctx, 0) == -6                       # after a push
        ctx.reset()                                                          # the setting survives reset
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        a, _ = ctx.take_telegrams()
        ctx.seek(0)
        ctx.set_telegrams(False)                                             # allowed again after a seek
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        b, _ = ctx.take_telegrams()
    assert len(a) and not len(b)
    with pkg.WmbusB200("-v", lib=L, manual_frames=1) as ctx:
        assert L.wmb_set_telegrams(ctx._ctx, 1) == -1 and L.wmb_set_telegrams(ctx._ctx, 0) == -1
        assert b"manual_frames" in L.wmb_last_error()


def test_partial_take(hostsim_lib, pkg):
    """take stops at cap records or when the next record's bytes do not fit; the rest stay queued, in order"""
    cu8 = rc.cached_capture("synth_mixed_1m6.cu8")
    want, wdata, *_ = tc.product(pkg, hostsim_lib, cu8, "-v", max_batch_mib=1)
    with pkg.WmbusB200("-v", lib=hostsim_lib, max_batch_mib=1, telegrams=True) as ctx:
        ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        r = np.zeros(8, pkg.telegram_dtype())
        buf = np.zeros(4096, np.uint8)
        n = C.c_size_t(0)
        assert hostsim_lib.wmb_take_telegrams(ctx._ctx, r.ctypes.data, 3, buf.ctypes.data, 4096, C.byref(n)) == 0
        assert n.value == 3
        got = [buf[:int(r["len"][:3].sum())].tobytes()]
        assert hostsim_lib.wmb_take_telegrams(ctx._ctx, r[3:].ctypes.data, 5, buf.ctypes.data, int(want["len"][3]),
                                              C.byref(n)) == 0 and n.value == 1
        got.append(buf[:int(r["len"][3])].tobytes())
        rest, rdata = ctx.take_telegrams()
    assert tc.as_tuples(r[:4]) + tc.as_tuples(rest) == tc.as_tuples(want)
    assert b"".join(got) + b"".join(rdata) == b"".join(wdata)


# ---- the CLI -------------------------------------------------------------------------------------------------------

def _cli(env_extra, stdin_bytes, flags="-v"):
    exe = os.path.join(ROOT, "tests", "hostsim", "_build", "rtl_wmbus_hostsim")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WMBUS_B200_")}
    env.update(env_extra)
    return subprocess.run([exe] + flags.split(), input=stdin_bytes, capture_output=True, env=env, timeout=600)


def cli_lines(recs, data):
    """the CLI's lines of records: MODE;DECODED;SOURCES;FAILED;SYNC_SAMPLE;MANUF;ID;VERSION;TYPE;CI;0xDATAGRAM"""
    out = []
    for r, b in zip(recs, data):
        v = int(r["valid"])
        f = lambda bit, s: s if v & bit else "-"
        mode = r["mode"].decode() if r["decoded"] else ("T1C1" if r["chain"] == 0 else "S1")
        out.append(";".join([mode, str(r["decoded"]), str(r["sources"]), str(r["failed"]), str(r["sync_sample"]),
                             f(4, r["manuf"].decode()), f(8, "%08X" % r["id"]), f(16, "%02X" % r["version"]),
                             f(32, "%02X" % r["type"]), f(64, "%02X" % r["ci"]), "0x" + b.hex() if b else "-"]))
    return out


@pytest.mark.parametrize("name,flags,repair", [("synth_mixed_1m6.cu8", "-v", False), ("synth_mixed_1m6.cu8", "", True),
                                               ("synth_mixed_2m4_shift.cu8", "-d 3 -s", True)])
def test_cli_telegrams(hostsim_lib, pkg, tmp_path, name, flags, repair):
    """the file equals take_telegrams(); stdout is byte-identical with and without it (but the wall-clock column)"""
    cu8 = rc.cached_capture(name)
    env = {"WMBUS_B200_REPAIRED": str(tmp_path / "rep.txt"), "WMBUS_B200_REPAIR_ERASURES": "3",
           "WMBUS_B200_REPAIR_SOFT_BITS": "6", "WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS": "6",
           "WMBUS_B200_REPAIR_S1_SOFT_BITS": "6"} if repair else {}
    r0 = _cli(env, cu8.tobytes(), flags)
    r1 = _cli(dict(env, WMBUS_B200_TELEGRAMS=str(tmp_path / "tlg.txt")), cu8.tobytes(), flags)
    assert r1.returncode == 0 and r0.returncode == 0, (r1.stderr, r0.stderr)
    blank = lambda txt: [orc.blank_ts(l) for l in txt.decode().splitlines()]
    assert blank(r1.stdout) == blank(r0.stdout)
    rp = tc.REPAIRS["soft"] if repair else None
    recs, data, *_ = tc.product(pkg, hostsim_lib, cu8, flags, repair=rp, max_batch_mib=64)
    want = cli_lines(recs, data)
    assert (tmp_path / "tlg.txt").read_text().splitlines() == want and len(want) >= 3


def test_cli_bad_path(hostsim_lib):
    r = _cli({"WMBUS_B200_TELEGRAMS": "/nonexistent-dir/x"}, rc.cached_capture("synth_mixed_1m6.cu8").tobytes())
    assert r.returncode == 1 and r.stdout == b"" and b"WMBUS_B200_TELEGRAMS" in r.stderr
