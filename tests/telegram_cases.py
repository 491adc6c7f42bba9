"""Telegram records (wmb_group_telegrams / wmb_set_telegrams / wmb_take_telegrams): the rule of
include/wmbus_b200_framer.h restated in plain Python, and the checks shared by the CPU-simulation tests
(test_telegrams.py) and the GPU tests (test_telegrams_gpu.py).

The restatement takes the lines the library printed (their text: mode, CRC_OK, LINK_LAYER_IDENT_NO and the datagram
column), their line records (sync_sample, chain, algo) and the repair records, and builds the records from those alone."""
from bisect import bisect_right

import numpy as np

import receiver_cases as rc

W = {0: 128, 1: 256}                      # WMB_TLG_W_T1C1, WMB_TLG_W_S1
T2A_LINE, RLA_LINE, T2A_REPAIR, RLA_REPAIR = 1, 2, 4, 8
FIELDS = ("sync_sample", "chain", "decoded", "sources", "failed", "mode", "len", "valid", "l", "c", "m", "manuf", "id",
          "version", "type", "ci")

# repair settings of the capture cases: off, erasure repair only, erasure repair and all three soft repairs
REPAIRS = {"off": {}, "erasure": dict(repair=3), "soft": dict(repair=3, repair_soft=6, repair_t1_soft=6, repair_s1_soft=6)}
FLAGS = ["", "-s", "-r 0", "-t 0", "-v", "-d 3 -s"]


def capture_flags(name):
    """the flag sets a committed capture runs under: a 2.4 MS/s capture always with -d 3"""
    d3 = "-d 3" in rc.COMMITTED[name][0]
    out = []
    for f in FLAGS:
        if d3 and "-d" not in f:
            f = ("-d 3 " + f).strip()
        if f not in out:
            out.append(f)
    return out


def line_fields(line):
    """(mode, crc_ok, ident, datagram bytes) of a datagram line"""
    f = line.split(";")
    if f[0] in ("rla", "t2a"):
        f = f[1:]
    return f[0], int(f[1]), int(f[6], 16), bytes.fromhex(f[7][2:])


def candidates(lines, info, repairs=()):
    """[(chain, sync, source bit, verified, mode, bytes)]: every line and every REPAIRED repair record"""
    out = []
    for l, r in zip(lines, info):
        mode, ok, _, data = line_fields(l)
        out.append((int(r["chain"]), int(r["sync_sample"]), T2A_LINE if int(r["algo"]) == 1 else RLA_LINE, bool(ok),
                    mode, data))
    for r in repairs:
        if int(r.repair.outcome) != 1:
            continue
        d = r.repair.line
        out.append((int(r.chain), int(r.sync_sample), T2A_REPAIR if int(r.algo) == 1 else RLA_REPAIR, True,
                    d.mode.decode(), bytes(d.datagram[:d.len])))
    return out


def header(data):
    """(valid, l, c, m, manuf, id, version, type, ci) of a datagram"""
    n = len(data)
    valid = sum(bit for bit, need in ((1, 1), (2, 2), (4, 4), (8, 8), (16, 9), (32, 10), (64, 11)) if n >= need)
    m = int.from_bytes(data[2:4], "little") if n >= 4 else 0
    manuf = bytes([((m >> 10) & 31) + 64, ((m >> 5) & 31) + 64, (m & 31) + 64]).decode() if n >= 4 else ""
    return (valid, data[0] if n >= 1 else 0, data[1] if n >= 2 else 0, m, manuf,
            int.from_bytes(data[4:8], "little") if n >= 8 else 0, data[8] if n >= 9 else 0, data[9] if n >= 10 else 0,
            data[10] if n >= 11 else 0)


def restate(cands):
    """[(record tuple in FIELDS order, bytes)] in record order"""
    out = []
    for ch in (0, 1):
        c = sorted((x for x in cands if x[0] == ch), key=lambda x: x[1])
        groups = []
        for x in c:
            if groups and x[1] - groups[-1][-1][1] <= W[ch]:
                groups[-1].append(x)
            else:
                groups.append([x])
        for g in groups:
            s0 = g[0][1]
            failed = sum(1 for x in g if not x[3])
            recs = {}
            for x in g:
                if x[3]:
                    recs[(x[4], x[5])] = recs.get((x[4], x[5]), 0) | x[2]
            if not recs:
                out.append(((s0, ch, 0, 0, failed, "", 0) + (0,) * 4 + ("",) + (0,) * 4, b""))
            for (mode, data), src in recs.items():
                valid, l, cc, m, manuf, ident, ver, typ, ci = header(data)
                out.append(((s0, ch, 1, src, failed, mode, len(data), valid, l, cc, m, manuf, ident, ver, typ, ci), data))
    out.sort(key=lambda r: (r[0][0], r[0][1], r[0][5], r[0][6], r[1]))
    return out


def as_tuples(recs):
    return [tuple(r[f].decode() if isinstance(r[f], bytes) else int(r[f]) for f in FIELDS) for r in recs]


def product(pkg, lib, cu8, flags, pushes=None, seek=0, device=None, repair=None, **tuning):
    """the library's telegram records (records, data), taken after every push and at the end, with its lines, line
    records and repair records.  pushes: host push sizes (None: one process call); device: torch, to run the capture
    through process_device"""
    repair = repair or {}
    with pkg.WmbusB200(flags, lib=lib, telegrams=True, **repair, **tuning) as ctx:
        if seek:
            ctx.seek(seek)
        recs, data, lines, info, reps = [], [], [], [], []

        def take():
            r, b = ctx.take_telegrams()
            recs.append(r)
            data.extend(b)

        if device is not None:
            t = device.from_numpy(np.ascontiguousarray(cu8)).cuda()
            l, i = ctx.process_device(t.data_ptr(), len(cu8) - len(cu8) % 4096, flush=True, info=True)
            lines += l
            info.append(i)
        elif pushes is None:
            l, i = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
            lines += l
            info.append(i)
        else:
            off = 0
            for n in pushes + [len(cu8)]:
                n = min(n, len(cu8) - off)
                ctx.push(cu8.ctypes.data + off, n)
                take()
                l, i = ctx.take_lines(info=True)
                lines += l
                info.append(i)
                off += n
            ctx.poll_flush()
            l, i = ctx.take_lines(info=True)
            lines += l
            info.append(i)
        take()
        if repair:
            reps = ctx.take_repairs()
        st = ctx.stats()
    return np.concatenate(recs), data, lines, np.concatenate(info), reps, st


def check_invariants(recs, data, lines, info, reps):
    """every CRC-ok line and repaired line is in exactly one decoded record of its group, with its bit; the ID of a
    record equals the LINK_LAYER_IDENT_NO of every line it came from"""
    by = {}
    for r, b in zip(recs, data):
        if int(r["decoded"]):
            by.setdefault((int(r["chain"]), r["mode"].decode(), b), []).append(r)
    starts = {ch: sorted(int(r["sync_sample"]) for r in recs if int(r["chain"]) == ch) for ch in (0, 1)}
    for ch, s, src, ok, mode, b in candidates(lines, info, reps):
        if not ok:
            continue
        g = starts[ch][bisect_right(starts[ch], s) - 1]          # the group's earliest match
        hit = [r for r in by.get((ch, mode, b), []) if int(r["sync_sample"]) == g]
        assert len(hit) == 1 and int(hit[0]["sources"]) & src, (ch, s, src, mode, b.hex())
    for l, r in zip(lines, info):
        mode, ok, ident, b = line_fields(l)
        if not ok or len(b) < 8:
            continue
        st = starts[int(r["chain"])]
        g = st[bisect_right(st, int(r["sync_sample"])) - 1]
        hit = [x for x in by[(int(r["chain"]), mode, b)] if int(x["sync_sample"]) == g]
        assert int(hit[0]["id"]) == ident, (l, int(hit[0]["id"]))


def check_parity(pkg, lib, cu8, flags, **kw):
    """the records equal the restatement of the run's own lines and repairs, in order; the invariants hold"""
    recs, data, lines, info, reps, st = product(pkg, lib, cu8, flags, **kw)
    want = restate(candidates(lines, info, reps))
    got = as_tuples(recs)
    assert got == [w[0] for w in want], (flags, kw, len(got), len(want),
                                         next(((i, a, b) for i, (a, b) in enumerate(zip(got, [w[0] for w in want]))
                                               if a != b), None))
    assert data == [w[1] for w in want], (flags, kw)
    check_invariants(recs, data, lines, info, reps)
    return recs, data, lines, info, reps, st


def decoded_set(recs, data):
    return {(int(r["chain"]), r["mode"].decode(), b) for r, b in zip(recs, data) if int(r["decoded"])}
