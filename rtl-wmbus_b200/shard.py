"""Multi-GPU sharding rules of the path (DESIGN.md section 6).

* Independent captures (BASELINE config 5): one capture per rank, no data-path collective; the only exchange is
  the all-reduce of the packet counters.  Used by bench.py (NCCL) and by the world_size-2 gloo test on CPU.
* Time chunks of ONE capture (config 4, SURVEY.md 8e): rank g owns the decimated samples [S_g, S_g+1), warm-starts a
  halo earlier and proves that it re-joined the sequential run by comparing `wmb_boundary_state()` with its left
  neighbour's (an all-gather of two digests); a rank whose halo was too short repeats with a longer one."""
from __future__ import annotations

import torch
import torch.distributed as dist

COUNTER_FIELDS = ("lines", "crc_ok", "t1", "c1", "s1")


def capture_seed(config_index: int, rank: int) -> int:
    """Seed of rank `rank`'s capture (SURVEY.md 8d: 0xB200_0000 + config*16 + rank)."""
    return 0xB2000000 + 16 * config_index + rank


def count_lines(lines) -> torch.Tensor:
    """Packet counters of one rank from its datagram lines (with or without the -v prefix)."""
    c = dict.fromkeys(COUNTER_FIELDS, 0)
    for l in lines:
        f = l.split(";")
        if f[0] in ("rla", "t2a"):
            f = f[1:]
        c["lines"] += 1
        c["crc_ok"] += f[1] == "1"
        c[f[0].lower()] += 1
    return torch.tensor([c[k] for k in COUNTER_FIELDS], dtype=torch.int64)


def reduce_counts(counts: torch.Tensor, device=None) -> dict:
    """Sum the counters over all ranks (NCCL over NVLink on GPUs, gloo in the CPU test)."""
    t = counts.to(device) if device is not None else counts.clone()
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return dict(zip(COUNTER_FIELDS, (int(v) for v in t.cpu())))


# ---- time chunks of one capture ---------------------------------------------------------------------

# right halo, decimated samples.  The run-length tracker of the S1 chain accepts up to just under 36 samples per chip
# (rtl_wmbus.c:659; nominal 24.4), so the longest telegram it can deliver -- (16 * 290 + 17) chips -- spans up to
# 4657 * 36 = 167,652 samples; T1/C1: (12 * 290 + 13) chips * 8 * 1.25 < 35,000.
MAX_TELEGRAM_M = 1 << 18


def line_key(line: str):
    """(end sample, stream priority) of a line taken with timestamp_mode=2 ("@<sample>.<prio>" in the TIMESTAMP
    column): the position at which the reference prints it (rtl_wmbus.c:1354-1355)."""
    f = line.split(";")
    ts = f[4 if f[0] in ("rla", "t2a") else 3]
    a, b = ts[1:].split(".")
    return int(a), int(b)


def blank_position(line: str) -> str:
    f = line.split(";")
    f[4 if f[0] in ("rla", "t2a") else 3] = "TS"
    return ";".join(f)


def merge_lines(parts, infos=None, quals=None):
    """Lines of several time chunks (each taken with timestamp_mode=2) -> the sequential run's print order, with the
    TIMESTAMP column blanked.  Within one chunk the order is already right; across chunks a telegram that started in
    chunk g may finish after one that started in chunk g+1, so the merge is by print position (stable).
    infos: the chunks' line records (numpy arrays of wmb_line_info, one per line): returns (lines, records) then, the
    records in the same order.  quals: the chunks' wmb_line_quality records, likewise: (lines[, records], quality)."""
    flat = [l for part in parts for l in part]
    order = sorted(range(len(flat)), key=lambda i: line_key(flat[i]))
    lines = [blank_position(flat[i]) for i in order]
    if infos is None and quals is None:
        return lines
    import numpy as np
    out = [lines]
    for arrs in (infos, quals):
        if arrs is None:
            continue
        recs = np.concatenate(arrs)
        assert len(recs) == len(flat), "one record per line"
        out.append(recs[np.asarray(order, np.int64)])
    return tuple(out)


def chunk_bounds(n_bytes: int, d: int, world: int):
    """IQ-sample boundaries [k_0 .. k_world] of `world` time chunks, multiples of the batch granule."""
    gran = 2048 * d                                   # IQ samples per 4096*d input bytes
    n_iq = (n_bytes // 2) // gran * gran
    return [min(n_iq, (n_iq * g // world) // gran * gran) for g in range(world)] + [n_iq]


def merge_bursts(parts, quals=None):
    """Burst records (wmb_burst arrays) of several time chunks, each holding the pieces that start in its chunk ->
    the sequential run's records, ordered by (start_sample, chain).  quals: the chunks' wmb_burst_quality records, one
    per burst: returns (records, quality) then."""
    import numpy as np
    recs = np.concatenate(parts)
    order = np.lexsort((recs["chain"], recs["start_sample"]))
    if quals is None:
        return recs[order]
    q = np.concatenate(quals)
    assert len(q) == len(recs), "one quality record per burst"
    return recs[order], q[order]


def merge_snippets(parts, infos=None, repairs=None, undecoded=False):
    """Snippets ((records, data) of take_snippets()) of several time chunks, each holding those of the pieces that start
    in its chunk -> the sequential run's, in burst order.  A line whose match lies after a chunk's end belongs to the next
    chunk, so a chunk cannot decide `decoded` for a piece that runs past its end: with infos (the merged line records,
    merge_lines(..., infos)) and repairs (the merged repair records, when repair is on) it is decided here, and
    undecoded=True keeps the pieces that did not decode (the chunks take every piece, mode 1)."""
    import numpy as np
    recs = np.concatenate([p[0] for p in parts])
    data = [x for p in parts for x in p[1]]
    order = np.lexsort((recs["chain"], recs["start_sample"]))
    recs, data = recs[order], [data[i] for i in order]
    if infos is None:
        assert not undecoded, "deciding which pieces decoded needs the merged line records"
        return recs, data
    ok = {0: [], 1: []}
    for r in infos:
        if r["crc_ok"]:
            ok[int(r["chain"])].append(int(r["sync_sample"]))
    for r in repairs or []:
        if r.repair.outcome == 1:                        # WMB_REP_REPAIRED
            ok[int(r.chain)].append(int(r.sync_sample))
    ok = {ch: np.sort(np.asarray(v, np.uint64)) for ch, v in ok.items()}
    for i, r in enumerate(recs):
        m = ok[int(r["chain"])]
        recs[i]["decoded"] = int(np.searchsorted(m, r["end_sample"]) > np.searchsorted(m, r["start_sample"]))
    if undecoded:
        keep = recs["decoded"] == 0
        recs, data = recs[keep], [x for x, k in zip(data, keep) if k]
    return recs, data


def merge_spectrum(parts):
    """Band-survey records (rows, sum, peak) of several time chunks -> the sequential run's records: sum and blocks
    added, peak the max, over the rows of one record (a record that straddles a chunk border has a row in each)."""
    import numpy as np
    full = [p for p in parts if len(p[0])]                # (a chunk may hold no record)
    if not full:
        return parts[0]
    rows = np.concatenate([p[0] for p in full])
    sums = np.concatenate([p[1] for p in full])
    peaks = np.concatenate([p[2] for p in full])
    recs, inv = np.unique(rows["record"], return_inverse=True)
    out = np.zeros(len(recs), rows.dtype)
    first = np.full(len(recs), -1)
    for i in range(len(rows)):
        if first[inv[i]] < 0:
            first[inv[i]] = i
    out[:] = rows[first]
    out["blocks"] = np.bincount(inv, weights=rows["blocks"], minlength=len(recs)).astype(np.uint32)
    s = np.zeros((len(recs), sums.shape[1]), np.uint64)
    p = np.zeros((len(recs), peaks.shape[1]), np.float32)
    np.add.at(s, inv, sums)
    np.maximum.at(p, inv, peaks)
    return out, s, p


def repair_key(r):
    """(end_sample, chain * 2 + (algo == t2a), sync_sample): the order of the repair records (wmb_repair_record)"""
    return r.end_sample, r.chain * 2 + (1 if r.algo == 1 else 0), r.sync_sample


def merge_repairs(parts):
    """Repair records (lists of WmbRepairRecord) of several time chunks, each holding those whose match lies in its
    chunk -> the sequential run's records, in repair_key() order."""
    return sorted((r for part in parts for r in part), key=repair_key)


def line_decoded(line: str):
    """a datagram line ("[rla;|t2a;]MODE;CRC_OK;3OUTOF6OK;TIMESTAMP;PACKET_RSSI;CURRENT_RSSI;IDENT;0xHEX") -> the
    WmbDecoded that wmb_format_line prints as it"""
    import ctypes
    from .capi import WmbDecoded
    f = line.split(";")
    if f[0] in ("rla", "t2a"):
        f = f[1:]
    d = WmbDecoded()
    d.status = 1                                      # WMB_DEC_LINE
    d.mode = f[0].encode()
    d.crc_ok, d.ok_3of6 = int(f[1]), int(f[2])
    d.packet_rssi, d.current_rssi = int(f[4]), int(f[5])
    d.serial = int(f[6], 16)
    data = bytes.fromhex(f[7][2:])
    d.len = len(data)
    ctypes.memmove(d.datagram, data, len(data))
    return d


def merge_telegrams(lines, infos, repairs=(), lib=None):
    """Telegram records of a time-sharded run: wmb_group_telegrams (of lib, default the product library) over the merged
    lines and line records (merge_lines(..., infos)) and the merged repair records (merge_repairs(), when repair is on)
    -> (records, data) as WmbusB200.take_telegrams() gives them in the sequential run.  The chunks need no telegram
    records of their own."""
    from .capi import group_telegrams, load_library
    return group_telegrams(lib or load_library(), infos, [line_decoded(l) for l in lines], list(repairs))


def find_carriers(rows, sum, peak, fs: float, threshold_db: float = 15.0, bridge_hz: float = 110e3,
                  tone_hz: float = 20e3):
    """Carriers worth decoding in a band survey (take_spectrum / merge_spectrum output, or a CLI spectrum file read
    with tools/find_carriers.py), fs the capture's sample rate (0.8 d MHz).  The bins' frequencies come from the rows'
    hz_low and hz_step; fs is checked against them (a survey of another capture rate raises ValueError).
      mean[k] = sum of sum / sum of blocks, hold[k] = max peak, floor = the median over k of mean;
      a bin is hot when hold >= floor * 10^(T / 10), T = 15 dB: in the tests' captures a meter's FSK tones stand 30 dB
        and more above the floor in the peak hold, while noise alone stays below 12 dB there (its hold over 16384 blocks
        is about ln(16384) = 9.7 times, 9.9 dB, the mean);
      hot bins within 110 kHz of each other are one region: S1's two tones lie 100 kHz apart (T1/C1's 80-100 kHz);
      a region's carrier is its hold-weighted mean frequency -- between the two FSK tones -- rounded to the 25 kHz grid
        of the mixer (rtl_wmbus.c:974-993); a region narrower than 20 kHz is a tone (a CW carrier, a spur), not a meter.
    Returns (carriers, tones): carriers a list [(offset_khz, "T"), (offset_khz, "S"), ...] for decode_carriers() -- the
    kind cannot be read off the spectrum, so each carrier gets a context with both chains on it -- and tones a list of
    their frequencies in Hz."""
    import numpy as np
    rows = np.asarray(rows)
    if not len(rows):
        return [], []
    if abs(-2.0 * float(rows["hz_low"][0]) - fs) > 1e-6 * fs:
        raise ValueError(f"the survey covers {-2.0 * float(rows['hz_low'][0]):.0f} Hz, not fs = {fs:.0f} Hz")
    n = rows["bins"][0]
    mean = np.asarray(sum, np.float64).sum(axis=0) / float(rows["blocks"].sum())
    hold = np.asarray(peak, np.float64).max(axis=0)
    floor = float(np.median(mean))
    freq = rows["hz_low"][0] + rows["hz_step"][0] * np.arange(n)
    hot = np.flatnonzero(hold >= floor * 10 ** (threshold_db / 10))
    carriers, tones = [], []
    if not len(hot):
        return carriers, tones
    regions = np.split(hot, np.flatnonzero(np.diff(freq[hot]) >= bridge_hz) + 1)
    step = float(rows["hz_step"][0])
    for reg in regions:
        width = freq[reg[-1]] - freq[reg[0]] + step
        f = float((freq[reg] * hold[reg]).sum() / hold[reg].sum())
        if width < tone_hz:
            tones.append(f)
            continue
        off = int(round(f / 25e3)) * 25
        if (off, "T") not in carriers:
            carriers += [(off, "T"), (off, "S")]
    return carriers, tones


def decode_time_chunk(ctx, push, n_bytes: int, d: int, rank: int, world: int, halo_m: int = 1 << 18, info=False,
                      bursts=False, spectrum=False, quality=False, repairs=False, snippets=False):
    """Decode rank `rank`'s chunk of a capture of n_bytes cu8 bytes.  `push(byte_lo, byte_hi)` feeds that byte
    range of the capture to ctx (host or device memory: the caller's business).
    Returns (lines, digest_start, digest_end, halo_start_iq): digest_start is None for a chunk that starts at 0.
    The lines carry their print position in the TIMESTAMP column (timestamp_mode 2) for merge_lines().
    info=True: lines is (lines, records), the records (wmb_line_info) of the lines.  A line's carrier-offset window lies
    in the chunk that holds its match, far behind the halo's start, so the records are the sequential run's.
    bursts=True (ctx made with a burst level): lines is (lines[, records], bursts), bursts the chunk's burst pieces -- those
    that start in [lo, hi) of decimated samples.  A piece depends on its samples and at most 2^17 + 2^16 + 196 before it
    (DESIGN.md §8), inside the left halo, and one that starts before hi is closed within as many samples after hi, inside
    the right halo, so they are the sequential run's pieces.
    spectrum=True (ctx made with spectrum=...): the band survey's records (rows, sum, peak) come last in lines.  The line
    window counts the chunk's blocks only, so merge_spectrum() over the chunks gives the sequential records.
    quality=True (ctx made with quality=True): the lines' wmb_line_quality records follow the line records, and with
    bursts=True the bursts' wmb_burst_quality records follow the bursts: (lines[, records], quality[, bursts,
    burst_quality][, spectrum]).  Their windows are the offset windows, so they are the sequential run's as well.
    repairs=True (ctx made with repair=e_max, repair_soft=k_max for the C1, repair_t1_soft=s_max for the T1 and
    repair_s1_soft=s_max for the S1 soft repair; the settings survive the chunk's seek): the repair records (take_repairs()) of the candidates matched in the chunk
    come last; merge_repairs() over the chunks gives the sequential records.  A candidate that waits for its repair
    counts in pending_before(), so the right halo goes on until its record is made.
    snippets=True (ctx made with a burst level and snippets=1): the snippets (take_snippets(): records, data) of the pieces
    that start in the chunk come after the bursts and the survey's records.  The left halo holds their PRE granules, and
    the right halo (MAX_TELEGRAM_M = 2^18 samples) holds the rest: a piece that starts before hi ends at most 2^17 + 2^16
    samples later, its end is decided 196 after that, and its POST granules follow within 3 x 2048.  merge_snippets() joins them; it decides `decoded` from the merged line
    records, since a line whose match lies past hi belongs to the next chunk."""
    import hashlib
    recs = []
    qrecs = []
    brecs = []
    bqrecs = []
    srecs = []
    rrecs = []
    snrecs, sndata = [], []

    def take_s():
        if snippets:
            r, b = ctx.take_snippets()
            snrecs.append(r)
            sndata.extend(b)
        if spectrum:
            srecs.append(ctx.take_spectrum())

    def take_b():
        if bursts and quality:
            b, q = ctx.take_bursts(quality=True)
            brecs.append(b)
            bqrecs.append(q)
        elif bursts:
            brecs.append(ctx.take_bursts())

    def take():
        if repairs:
            rrecs.extend(ctx.take_repairs())
        if quality:
            got = ctx.take_lines(2, info=True, quality=True)
            recs.append(got[1])
            qrecs.append(got[2])
            return got[0]
        if not info:
            return ctx.take_lines(2)
        got, r = ctx.take_lines(2, info=True)
        recs.append(r)
        return got
    k = chunk_bounds(n_bytes, d, world)
    lo, hi = k[rank], k[rank + 1]
    gran = 2048 * d
    start = max(0, lo - (halo_m * d + gran - 1) // gran * gran)
    ctx.seek(start)
    ctx.set_line_window(lo // d, hi // d if rank + 1 < world else (1 << 63))
    lines = []
    dig_start = None
    if start < lo:
        push(2 * start, 2 * lo)
        lines += take()
        take_b()
        take_s()
    if lo > 0:
        dig_start = hashlib.sha256(ctx.boundary_state()).digest()
    push(2 * lo, 2 * hi)
    lines += take()
    take_b()
    take_s()
    dig_end = hashlib.sha256(ctx.boundary_state()).digest()
    if rank + 1 < world:                              # finish the telegrams that started in the chunk
        step = (MAX_TELEGRAM_M * d + gran - 1) // gran * gran
        tail = min(k[world], hi + step)
        push(2 * hi, 2 * tail)
        # MAX_TELEGRAM_M bounds a telegram whose samples carry edges.  One that runs into a gap in the input (dead air:
        # the run-length tracker emits nothing until the next edge, then all the missing bits at once) ends arbitrarily
        # late: go on while a telegram matched in the chunk is still in flight
        while tail < k[world] and ctx.pending_before(hi // d) > 0:
            nxt = min(k[world], tail + step)
            push(2 * tail, 2 * nxt)
            tail = nxt
        ctx.poll_flush()
    else:
        if n_bytes > 2 * hi:
            push(2 * hi, n_bytes)                     # the ragged end of the capture (the reference drops a short item)
        ctx.poll_flush()
    lines += take()
    take_b()
    take_s()
    import numpy as np
    out = [lines]
    if info:
        out.append(np.concatenate(recs))
    if quality:
        out.append(np.concatenate(qrecs))
    if bursts:
        b = np.concatenate(brecs)
        m_lo, m_hi = lo // d, (hi // d if rank + 1 < world else 1 << 63)
        keep = (b["start_sample"] >= m_lo) & (b["start_sample"] < m_hi)
        out.append(b[keep])
        if quality:
            out.append(np.concatenate(bqrecs)[keep])
    if spectrum:
        srecs = [x for x in srecs if len(x[0])] or srecs[:1]
        out.append((np.concatenate([x[0] for x in srecs]), np.concatenate([x[1] for x in srecs]),
                    np.concatenate([x[2] for x in srecs])))
    if snippets:
        r = np.concatenate(snrecs)
        m_lo, m_hi = lo // d, (hi // d if rank + 1 < world else 1 << 63)
        keep = (r["start_sample"] >= m_lo) & (r["start_sample"] < m_hi)
        out.append((r[keep], [x for x, kk in zip(sndata, keep) if kk]))
    if repairs:
        out.append(rrecs)
    lines = tuple(out) if len(out) > 1 else lines
    return lines, dig_start, dig_end, start


def decode_time_sharded(ctx, push, n_bytes: int, d: int, halo_m: int = 1 << 18, info=False, bursts=False,
                        spectrum=False, quality=False):
    """All ranks: decode one capture in time chunks, exact by construction (see module docstring).
    Returns (my_lines, rounds); info=True / bursts=True: my_lines carries the records / burst pieces as in
    decode_time_chunk."""
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    rounds = 0
    lines = None
    redo = True
    while True:
        rounds += 1
        if redo:
            lines, ds, de, start = decode_time_chunk(ctx, push, n_bytes, d, rank, world, halo_m, info=info, bursts=bursts,
                                                        spectrum=spectrum, quality=quality)
        mine = torch.zeros(65, dtype=torch.uint8)
        mine[:32] = torch.frombuffer(bytearray(ds or bytes(32)), dtype=torch.uint8)
        mine[32:64] = torch.frombuffer(bytearray(de), dtype=torch.uint8)
        mine[64] = 1 if (ds is None or start == 0) else 0          # started from the true beginning: exact
        if world > 1:
            backend = dist.get_backend()
            dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
            allv = [torch.zeros(65, dtype=torch.uint8, device=dev) for _ in range(world)]
            dist.all_gather(allv, mine.to(dev))
            allv = [v.cpu() for v in allv]
        else:
            allv = [mine]
        bad = [g for g in range(1, world)
               if not allv[g][64] and not torch.equal(allv[g][:32], allv[g - 1][32:64])]
        if not bad:
            return lines, rounds
        redo = rank in bad
        if redo:
            halo_m *= 4                                 # too short: the neighbour's state was not reached yet


# ---- many carriers in one capture (SURVEY.md 8f N3) --------------------------------------------------

def plan_carriers(carriers):
    """carriers: [(offset_khz, "T" | "S"), ...] -- the carriers of one capture, as offsets from its centre frequency
    (multiples of 25 kHz, the grid of the reference's mixer table, rtl_wmbus.c:974-993) and the chain that listens to
    each: "T" = the T1/C1 chain, "S" = the S1 chain.  A context has one chain of each kind (the reference's -s is one
    context with {+325 "T", -325 "S"}), so the carriers are dealt out two per context.
    Returns [(t_offset_khz | None, s_offset_khz | None), ...]."""
    for off, kind in carriers:
        if kind not in ("T", "S"):
            raise ValueError(f"carrier kind {kind!r}: 'T' (T1/C1 chain) or 'S' (S1 chain)")
        if off % 25:
            raise ValueError(f"carrier offset {off} kHz is not on the 25 kHz grid")
    ts = [off for off, kind in carriers if kind == "T"]
    ss = [off for off, kind in carriers if kind == "S"]
    n = max(len(ts), len(ss))
    return [(ts[i] if i < len(ts) else None, ss[i] if i < len(ss) else None) for i in range(n)]


def decode_carriers(make_ctx, run, carriers, flags: str = ""):
    """Decode every carrier of one capture: one context per (T, S) pair of plan_carriers(), all over the same input.
    make_ctx(flags, **opts) -> a WmbusB200; run(ctx) -> its lines for the whole capture (e.g.
    `lambda ctx: ctx.process_device(ptr, n, flush=True)` -- the capture stays where it is, every context reads it).
    Returns {(offset_khz, kind): [lines in print order]}."""
    import ctypes as C
    out = {}
    for t_off, s_off in plan_carriers(carriers):
        carr = (C.c_int32 * 2)(0 if t_off is None else t_off // 25, 0 if s_off is None else s_off // 25)
        opts = dict(simultaneous=2, carrier_25khz=carr, t1c1_enabled=int(t_off is not None), s1_enabled=int(s_off is not None))
        with make_ctx(flags, **opts) as ctx:
            lines = run(ctx)
        if t_off is not None:
            out[(t_off, "T")] = []
        if s_off is not None:
            out[(s_off, "S")] = []
        for l in lines:
            f = l.split(";")
            mode = f[1] if f[0] in ("rla", "t2a") else f[0]
            out[(s_off, "S") if mode == "S1" else (t_off, "T")].append(l)
    return out
