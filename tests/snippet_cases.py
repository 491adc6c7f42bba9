"""Burst snippets (wmb_set_snippets / wmb_take_snippets): the restatement of include/wmbus_b200.h points 2-4 in plain
Python, and the checks shared by the CPU-simulation tests (test_snippets.py) and the GPU tests (test_snippets_gpu.py).

The restatement takes the burst records the library handed out, the access-code matches of its CRC-ok lines and
REPAIRED repair records, and the input bytes.  Granule g covers decimated samples [2048 g, 2048 g + 2048) and input
bytes [4096 d g, 4096 d (g + 1)) of the capture; a piece [s, e) keeps the granules [max(g_first, s // 2048 - PRE),
min(ceil(e / 2048) + POST, end)), end the end of the input consumed (whole 4096-byte items at the end of input)."""
import numpy as np

import burst_cases as bc

PRE, POST = 2, 2            # WMB_SNIPPET_PRE / WMB_SNIPPET_POST
FIELDS = ("start_sample", "end_sample", "start_iq", "nbytes", "chain", "decoded", "flags", "lost")


def decimation(flags):
    t = flags.split()
    return int(t[t.index("-d") + 1]) if "-d" in t else 2


def matches_ok(info, repairs=()):
    """{chain: sorted access-code matches} of the CRC-ok lines and the REPAIRED repair records"""
    ok = {0: set(), 1: set()}
    for r in info:
        if int(r["crc_ok"]):
            ok[int(r["chain"])].add(int(r["sync_sample"]))
    for r in repairs:
        if int(r.repair.outcome) == 1:
            ok[int(r.chain)].add(int(r.sync_sample))
    return ok


def restate(cu8, d, bursts, ok, mode, seek_iq=0, pre=PRE, post=POST):
    """[(record tuple, bytes)] in burst order"""
    gi, gb = 2048 * d, 4096 * d
    consumed = len(cu8) - len(cu8) % 4096
    g_first = seek_iq // gi
    g_end = -(-(seek_iq + consumed // 2) // gi)
    out = []
    for b in sorted(bursts, key=lambda r: (int(r["start_sample"]), int(r["chain"]))):
        s, e, ch = int(b["start_sample"]), int(b["end_sample"]), int(b["chain"])
        dec = int(any(s <= m < e for m in ok[ch]))
        if mode == 2 and dec:
            continue
        lo = max(g_first, s // 2048 - pre)
        hi = min(-(-e // 2048) + post, g_end)
        a = lo * gb - seek_iq * 2
        z = min(hi * gb - seek_iq * 2, consumed)
        out.append(((s, e, lo * gi, z - a, ch, dec, int(b["flags"]), 0), bytes(cu8[a:z])))
    return out


def as_tuples(recs):
    return [tuple(int(r[f]) for f in FIELDS) for r in recs]


def product(pkg, lib, cu8, flags, mode, level=bc.DEFAULT_LEVEL, pushes=None, seek=0, device=None, repair=0, **tuning):
    """the library's snippets (records, bytes) taken after every push and at the end, with its lines, line records,
    bursts, repair records and statistics.  pushes: host push sizes (None: one process call); device: a torch module
    to run the capture through process_device"""
    with pkg.WmbusB200(flags, lib=lib, burst_level=level, snippets=mode, repair=repair, **tuning) as ctx:
        if seek:
            ctx.seek(seek)
        recs, data, bursts = [], [], []

        def take():
            r, b = ctx.take_snippets()
            recs.append(r)
            data.extend(b)
            bursts.append(ctx.take_bursts())

        if device is not None:
            t = device.from_numpy(np.ascontiguousarray(cu8)).cuda()
            lines, info = ctx.process_device(t.data_ptr(), len(cu8) - len(cu8) % 4096, flush=True, info=True)
        elif pushes is None:
            lines, info = ctx.process(cu8.ctypes.data, len(cu8), flush=True, info=True)
        else:
            off = 0
            for n in pushes + [len(cu8)]:
                n = min(n, len(cu8) - off)
                ctx.push(cu8.ctypes.data + off, n)
                take()
                off += n
            ctx.poll_flush()
            lines, info = ctx.take_lines(info=True)
        take()
        reps = ctx.take_repairs() if repair else []
        st = ctx.stats()
    return np.concatenate(recs), data, lines, info, np.concatenate(bursts), reps, st


def check_parity(pkg, lib, cu8, flags, mode=1, level=bc.DEFAULT_LEVEL, pushes=None, seek=0, device=None, repair=0,
                 **tuning):
    """every snippet's record and bytes equal the restatement, in order, and none is lost"""
    recs, data, lines, info, bursts, reps, st = product(pkg, lib, cu8, flags, mode, level, pushes, seek, device, repair,
                                                        **tuning)
    want = restate(cu8, decimation(flags), bursts, matches_ok(info, reps), mode, seek)
    got = as_tuples(recs)
    assert got == [w[0] for w in want], (flags, tuning, len(got), len(want), bc.first_diff(got, [w[0] for w in want]))
    for i, (x, w) in enumerate(zip(data, want)):
        assert x == w[1], (flags, tuning, i, got[i])
    return recs, data, lines, info, bursts


def check_replay(pkg, lib, cu8, flags, level=bc.DEFAULT_LEVEL, seek=True, **tuning):
    """every CRC-ok line's piece, replayed into a fresh context (after wmb_seek(start_iq), or without a seek), gives
    that line with the same text and sync_sample.  Returns the number of lines replayed"""
    recs, data, lines, info, _ = check_parity(pkg, lib, cu8, flags, 1, level, **tuning)
    n = 0
    cache = {}
    for line, r in zip(lines, info):
        if not int(r["crc_ok"]):
            continue
        m, ch = int(r["sync_sample"]), int(r["chain"])
        hit = [i for i, x in enumerate(recs) if int(x["chain"]) == ch and x["start_sample"] <= m < x["end_sample"]]
        if not hit:
            continue                                   # no burst at this level (e.g. a weak telegram): out of scope
        i = hit[0]
        if i not in cache:
            with pkg.WmbusB200(flags, lib=lib, burst_level=level, **tuning) as ctx:
                if seek:
                    ctx.seek(int(recs[i]["start_iq"]))
                buf = np.frombuffer(data[i], np.uint8).copy()
                cache[i] = ctx.process(buf.ctypes.data, len(buf), flush=True, info=True)
        rl, ri = cache[i]
        shift = 0 if seek else int(recs[i]["start_iq"]) // decimation(flags)
        got = [(l, int(x["sync_sample"]) + shift) for l, x in zip(rl, ri)]     # timestamp_mode 1: the literal TS
        assert (line, m) in got, (flags, i, line, m, got)
        n += 1
    return n



def s_capture(n_bytes=4 << 20, seed=0xB20000A1):
    """T1, C1 frame A and B and S1 meters 325 kHz above / below the centre: the reference's -s scenario"""
    E = bc.synth_mod().Emitter
    em = [E("T1", 0x71200031, amp=80.0, period_s=0.21, start_s=0.010, seed=31),
          E("C1A", 0x71200032, amp=80.0, l_field=0x2C, period_s=0.23, start_s=0.060, seed=32),
          E("C1B", 0x71200033, amp=80.0, period_s=0.27, start_s=0.110, seed=33),
          E("S1", 0x19131294, amp=70.0, period_s=0.29, start_s=0.160, seed=34)]
    buf, _ = bc.synth_mod().synth_capture(n_bytes, fs=1.6e6, emitters=em, seed=seed, center_shift_hz=325e3)
    return np.ascontiguousarray(buf.numpy())


# the replay corpus: the committed captures with their flags, and s_capture() with -s
CORPUS = [("excerpt_samples2_a.cu8", "-v"), ("excerpt_issue47_c1.cu8", "-v"), ("excerpt_issue48_2m4.cu8", "-v -d 3 -s"),
          ("synth_mixed_1m6.cu8", "-v"), ("synth_mixed_2m4_shift.cu8", "-v -d 3 -s"), ("s_capture", "-v -s")]


def sass_digests(so_path):
    """{kernel (mangled name): sha256 of its SASS} of a built library (cuobjdump -sass)"""
    import hashlib
    import subprocess
    txt = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", so_path], capture_output=True, text=True,
                         check=True).stdout
    out, name, body = {}, None, []
    for line in txt.splitlines():
        s = line.strip()
        if s.startswith("Function : "):
            if name:
                out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            name, body = s[len("Function : "):], []
        elif name and s:
            body.append(s)
    if name:
        out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
    return out


def resource_usage(so_path):
    """{kernel (mangled name): {REG, STACK, SHARED, LOCAL, ...}} of a built library (cuobjdump -res-usage)"""
    import re
    import subprocess
    txt = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", so_path], capture_output=True, text=True,
                         check=True).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            out[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    return out
