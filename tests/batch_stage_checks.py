"""Batch-by-batch parity of the bit-sync stages, shared by the CPU-simulation tests (tests/test_batch_stages.py) and the
GPU tests (tests/test_zz_stages_at_scale_gpu.py).

pipeline_checks.check_bitsync_stages and receiver_cases.check_stages compare the stage taps of a capture that fits one
batch.  What crosses a batch boundary -- the time2 shift register (StreamDev.t2_sr), the run-length carries, the clock
IIR states, the dphi history prefix, the -s mixer phase, the event rings' write positions -- is seen there only at the
start of the stream.  Here a capture goes through many batches and every batch's taps are compared with the slice of
the oracle's whole-capture stages that the batch covers:
  * serialized: one batch per push (push / push_device), taps read after each; at the end every stream's events,
    batch after batch, are the oracle's whole event arrays and the lines are the oracle's;
  * pipelined: one process / process_device call over many batches, which overlap on the device as in the benchmark;
    the last batch's taps and the lines are compared (a missing cross-batch stream dependency shows only here).
The reference is the oracle (tests/orc.py) with the receiver settings restated by tests/receiver_oracle.py."""
import ctypes as C

import numpy as np

import orc
import receiver_oracle as ro

# (clock lock (T1/C1, S1), access-code errors (T1/C1, S1)): the reference's constants, and the densest strobes together
# with the most access-code flags (about 1 % of random bits on either chain), so that a wrong shift register or
# run-length reset carry shows within a few events of nearly every boundary instead of only where a real code sits
DEFAULT = ((2, 2), (0, 0))
DENSE = ((1, 1), (3, 6))
SETTINGS = (DEFAULT, DENSE)

GRANULE_M = 2048                      # decimated samples of a batch granule (4096 * d bytes) at every decimation
CODE_BITS = {0: 16, 1: 24}            # access-code register bits per chain


def setting_name(s):
    return f"L{s[0][0]}-{s[0][1]}_E{s[1][0]}-{s[1][1]}"


def chains_of(o):
    return [ch for ch, on in ((0, o.t1c1_enabled), (1, o.s1_enabled)) if on]


def algos_of(o):
    return [a for a, on in ((0, o.rla_enabled), (1, o.t2_enabled)) if on]


def geometry(lib):
    """time2 tile geometry of the library (wmb_bitsync.cuh: T2_THREADS, T2_WARP, T2_WPT, SCAN_TILE); the CPU build uses
    tiny tiles and "warps" so that small captures cross every boundary"""
    hostsim = "hostsim" in getattr(lib, "_name", "")
    threads, warp, scan_tile = (8, 4, 4 * 2) if hostsim else (256, 32, 256 * 16)
    return dict(tile_words=threads * 4, warp=warp, warp_words=warp * 4, scan_tile=scan_tile)


class Reference:
    """The oracle's stages of a whole capture, computed one chain at a time (each chain's full stage arrays are freed
    before the next), kept as what the taps compare with: dphi bit patterns, rssi, packed data / clock / strobe bits,
    every stream's events and the lines, per receiver setting."""

    def __init__(self, cu8, flags, settings=SETTINGS, lines=True):
        self.flags = flags
        self.o = o = orc.opts_from_flags(flags)
        self.settings = list(settings)
        self.chains = chains_of(o)
        self.algos = algos_of(o)
        self.taps, self.events = {}, {}
        found = {s: [] for s in self.settings}
        for chain in self.chains:
            st = orc.stages(cu8, o, chain)
            self.M = st["M"]
            pack = lambda a: np.packbits(np.asarray(a, np.uint8), bitorder="little")
            t = dict(dphi=st["fir"].view(np.uint32).copy(), rssi=st["rssi"].astype(np.uint32).astype(np.uint8),
                     bit=pack(st["bit"]), clk=pack(st["clk"]), strobe={})
            for s in self.settings:
                lock, errors = s[0][chain], s[1][chain]
                if lock not in t["strobe"]:
                    t["strobe"][lock] = pack(ro.strobes(st["clk"], lock))
                for algo in self.algos:
                    ev = ro.stream_events(st, chain, algo, lock, errors)
                    self.events[(chain, algo, s)] = ev
                    if lines:
                        found[s] += ro.stream_lines(ev, chain, algo)
            self.taps[chain] = t
            del st
        self.lines = {}
        if lines:
            for s, f in found.items():
                f.sort(key=lambda x: (x[0], x[1], x[2]))
                ls = [l for _, _, _, l in f]
                self.lines[s] = [orc.blank_ts(l if o.show_algorithm else l[4:]) for l in ls]

    def bits(self, chain, name, m0, n, lock=None):
        """unpacked oracle bits [m0, m0 + n) (m0 a multiple of 8: batches start on granules)"""
        assert m0 % 8 == 0
        packed = self.taps[chain]["strobe"][lock] if name == "strobe" else self.taps[chain][name]
        return np.unpackbits(packed[m0 // 8:(m0 + n + 7) // 8], bitorder="little")[:n]

    def sync_counts(self, s):
        return {(ch, a): int(self.events[(ch, a, s)]["sync"].sum()) for ch in self.chains for a in self.algos}


def where(m, m0, M, batch, geo, ev_m=None):
    """where a sample lies in the device's geometry: batch, global and batch-relative index, time2 tile, scan tile and
    32-word round; with the stream's event samples ev_m, how many of its events precede it since each boundary"""
    rel = int(m) - int(m0)
    word = rel // 32
    tile, wt = divmod(word, geo["tile_words"])
    warp, ww = divmod(wt, geo["warp_words"])
    rnd = ww // geo["warp"]
    out = (f"batch {batch} [{m0}, {m0 + M}): sample {m} (batch-relative {rel}), time2 tile {tile} (scan tile "
           f"{tile // geo['scan_tile']}), warp {warp} round {rnd}")
    if ev_m is not None:
        ev_m = np.asarray(ev_m, np.int64)
        i = np.searchsorted(ev_m, m)
        firsts = []
        for name, b in (("batch", m0), ("scan tile", m0 + (tile // geo["scan_tile"]) * geo["scan_tile"] * geo["tile_words"] * 32),
                        ("tile", m0 + tile * geo["tile_words"] * 32)):
            k = int(i - np.searchsorted(ev_m, b))
            if k < 32:
                firsts.append(f"event #{k} after the {name} boundary")
        out += "; " + (", ".join(firsts) if firsts else "not among the first events after a boundary")
    return out


def _compare_taps(ctx, ref, s, m0, M, batch, geo, cbits):
    """dphi, rssi, data bits, strobes (and clock signs) of the context's last batch against the oracle's [m0, m0 + M)"""
    for chain in ref.chains:
        t = ref.taps[chain]
        dphi, rssi = ctx.debug_stage(chain, M)
        assert len(dphi) == M, (batch, chain, len(dphi), M)
        for name, got, want in (("dphi", dphi.view(np.uint32), t["dphi"][m0:m0 + M]), ("rssi", rssi, t["rssi"][m0:m0 + M])):
            bad = np.nonzero(got != want)[0]
            assert len(bad) == 0, (f"chain {chain} {name}: {len(bad)} samples differ, first at "
                                   + where(m0 + bad[0], m0, M, batch, geo), got[bad[:4]], want[bad[:4]])
        taps = [(0, "bit", None)]
        if ref.o.t2_enabled:
            taps.append((1, "strobe", s[0][chain]))
            if cbits:
                taps.append((2, "clk", None))
        for which, name, lock in taps:
            got = ctx.debug_bits(chain, which, M)
            want = ref.bits(chain, name, m0, M, lock)
            bad = np.nonzero(got != want)[0]
            assert len(bad) == 0, f"chain {chain} {name}: {len(bad)} samples differ, first at " + where(m0 + bad[0], m0, M, batch, geo)


def _compare_events(ctx, ref, s, m0, M, batch, geo, pos=None):
    """every stream's events of the context's last batch against the oracle's events with m in [m0, m0 + M); pos: the
    per-stream count of events of the batches before (serialized mode: the batches' events, one after another, must
    be the oracle's whole arrays) -- returns the new counts"""
    out = {}
    for chain in ref.chains:
        for algo in ref.algos:
            want = ref.events[(chain, algo, s)]
            lo, hi = np.searchsorted(want["m"], [m0, m0 + M])
            if pos is not None:
                assert pos[(chain, algo)] == lo, (batch, chain, algo, "events before the batch", pos[(chain, algo)], lo)
            cap = int(hi - lo) + 4096
            got = ctx.debug_events(chain, algo, cap)
            n = len(got["m"])
            assert n < cap, (batch, chain, algo, "the tap returned the whole buffer: more events than the batch has", n)
            assert n == hi - lo, (f"chain {chain} algo {algo}: {n} events, the oracle {hi - lo} in "
                                  + where(m0, m0, M, batch, geo))
            if n:
                assert m0 <= int(got["m"].min()) and int(got["m"].max()) < m0 + M, (batch, chain, algo, "event outside the batch")
            for f in ("m", "bit", "sync", "reset", "rssi"):
                w = want[f][lo:hi].astype(np.uint64)
                bad = np.nonzero(got[f] != w)[0]
                if len(bad):
                    k = bad[0]
                    raise AssertionError(
                        f"{setting_name(s)} chain {chain} algo {algo} field {f}: {len(bad)} of {n} events differ, first "
                        f"the batch's event {k} (ordinal {lo + k}, got {int(got[f][k])}, want {int(w[k])}) at "
                        + where(want["m"][lo + k], m0, M, batch, geo, want["m"]))
            out[(chain, algo)] = int(hi)
    return out


def context(pkg, lib, flags, s, reserved1=0, **tuning):
    """a context with these receiver settings that keeps the clock-sign tap (opts.reserved[1] & 1: one more store)"""
    return pkg.WmbusB200(flags, lib=lib, clock_lock=s[0], access_code_errors=s[1],
                         reserved=(C.c_uint32 * 2)(0, 1 | reserved1), **tuning)


def check_lines(ref, s, lines, overflow_batches):
    """lines against the oracle's: at the default settings always (and nothing may overflow); at the dense ones false
    candidates may legitimately fill the gather tables, which costs lines (pipeline_checks.check_overflow_degrades), so
    the lines are compared when nothing overflowed.  Returns whether they were compared."""
    if s == DEFAULT:
        assert overflow_batches == 0
    if overflow_batches:
        return False
    want = ref.lines[s]
    assert lines == want, (setting_name(s), len(lines), len(want),
                           next((i for i, (a, b) in enumerate(zip(lines, want)) if a != b), None))
    return True


def run_serialized(pkg, lib, ref, data, pushes, s, device_ptr=None, reserved1=0, **tuning):
    """One batch per push: the push sizes in bytes (whole granules; only the last may be ragged, it is then handed to the
    flush).  device_ptr: push from device memory at this address (data is then the capture's length).
    Returns a report: per batch (m0, M) and per stream the cumulative event counts, overflow_batches, lines compared."""
    o = ref.o
    gran = 4096 * max(1, o.decimation)
    assert sum(pushes) == (data if device_ptr is not None else len(data)) and all(n % gran == 0 for n in pushes[:-1])
    geo = geometry(lib)
    batches, totals = [], {(ch, a): [0] for ch in ref.chains for a in ref.algos}
    with context(pkg, lib, ref.flags, s, reserved1, **tuning) as ctx:
        off, pos, m_prev = 0, {k: 0 for k in totals}, 0
        for i, n in enumerate(pushes):
            before = ctx.stats().batches
            if device_ptr is not None:
                ctx.push_device(device_ptr + off, n)
            else:
                ctx.push(data.ctypes.data + off, n)
            if i == len(pushes) - 1:
                ctx.poll_flush()
            off += n
            st = ctx.stats()
            assert st.batches == before + 1, ("one batch per push", i, n, st.batches - before)
            M = int(st.decimated_samples) - m_prev
            m0 = m_prev
            _compare_taps(ctx, ref, s, m0, M, i, geo, cbits=True)
            pos = _compare_events(ctx, ref, s, m0, M, i, geo, pos)
            for k in totals:
                totals[k].append(pos[k])
            batches.append((m0, M))
            m_prev += M
        assert m_prev == ref.M
        for k, v in pos.items():
            assert v == len(ref.events[k + (s,)]["m"]), (k, v, "the batches' events end before the oracle's")
        lines = ctx.take_lines()
        ovf = int(ctx.stats().overflow_batches)
    return dict(batches=batches, totals=totals, overflow_batches=ovf, lines_compared=check_lines(ref, s, lines, ovf))


def run_pipelined(pkg, lib, ref, data, s, device_ptr=None, reserved1=0, min_batches=2, **tuning):
    """One process call over the whole capture (many batches in flight at once); the last batch's taps and events, and
    the lines.  Returns (batches, overflow_batches, lines compared).  data: the capture, or with device_ptr its length."""
    geo = geometry(lib)
    n_bytes = data if device_ptr is not None else len(data)
    with context(pkg, lib, ref.flags, s, reserved1, **tuning) as ctx:
        if device_ptr is not None:
            lines = ctx.process_device(device_ptr, n_bytes, flush=True)
        else:
            lines = ctx.process(data.ctypes.data, n_bytes, flush=True)
        st = ctx.stats()
        assert st.batches >= min_batches, "the capture is meant to take several batches"
        assert int(st.decimated_samples) == ref.M
        M = len(ctx.debug_stage(ref.chains[0], ref.M)[0])
        m0 = ref.M - M
        _compare_taps(ctx, ref, s, m0, M, int(st.batches) - 1, geo, cbits=True)
        _compare_events(ctx, ref, s, m0, M, int(st.batches) - 1, geo)
        ovf = int(st.overflow_batches)
        return int(st.batches), ovf, check_lines(ref, s, lines, ovf)


def code_windows(ref, chains=None, algos=None):
    """(first, last) sample of every real access code: the samples of the register's CODE_BITS events that end in a
    sync event at the default settings (E = 0).  A batch boundary b with first < b <= last splits the code between
    two batches, so that the carried register decides a real line."""
    out = []
    for (chain, algo, s), ev in ref.events.items():
        if s != DEFAULT or (chains and chain not in chains) or (algos and algo not in algos):
            continue
        nb = CODE_BITS[chain]
        for i in np.nonzero(ev["sync"])[0]:
            if i >= nb - 1:
                out.append((int(ev["m"][i - nb + 1]), int(ev["m"][i]), chain, algo))
    return sorted(out)


def boundaries_in_codes(windows, lo=0, hi=None):
    """the granule multiples that fall inside an access code: {boundary sample: (chain, algo)}"""
    out = {}
    for first, last, chain, algo in windows:
        b = (first // GRANULE_M + 1) * GRANULE_M
        if b <= last and b > lo and (hi is None or b < hi):
            out.setdefault(b, (chain, algo))
    return out


def pushes_through(boundaries, M, d, max_m, first_m=None):
    """push sizes (bytes) whose batch boundaries include `boundaries` (decimated samples, granule multiples), no batch
    longer than max_m samples; first_m: also cut there"""
    cuts = sorted(set(int(b) for b in boundaries if 0 < b < M) | ({first_m} if first_m else set()))
    out, at = [], 0
    for b in cuts + [M]:
        while b - at > max_m:
            step = max_m - (max_m % GRANULE_M) - GRANULE_M * ((len(out) * 7) % 5)   # uneven sizes
            out.append(step)
            at += step
        if b > at:
            out.append(b - at)
            at = b
    return [m * 2 * d for m in out]


def wraps_inside(totals, ring):
    """batches in which a ring of `ring` events wrapped strictly inside the batch (not at its first event)"""
    return [i for i in range(1, len(totals)) if totals[i] - 1 >= totals[i - 1] and
            (totals[i] - 1) // ring > totals[i - 1] // ring and totals[i - 1] % ring != 0]


def ring_events(max_batch_mib, d):
    """the time2 ring (and with opts.reserved[1] & 2 the run-length ring) of a context: wmb_context.cu ctx_alloc,
    next_pow2(M_max / 4 + 65536 + WMB_MAXBITS), WMB_MAXBITS = 1 + 16 + 290 * 16"""
    m_max = (max_batch_mib << 20) // (2 * d)
    need = m_max // 4 + 65536 + (1 + 16 + 290 * 16)
    p = 1
    while p < need:
        p <<= 1
    return p


FIRST_LINE_PREFIX = 4096              # candidates a gather's first prefix copy fetches before their count is known


def dense_8mib_capture():
    """48 MiB of mixed traffic for 8 MiB batches: at DENSE each batch has more candidates than FIRST_LINE_PREFIX, so a
    pipelined call grows the prefix while later batches are in flight with the one before"""
    import importlib
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    cap, _ = synth.synth_capture(48 << 20, fs=1.6e6, emitters=synth.default_emitters("mixed"), seed=0xB2000077)
    return np.ascontiguousarray(cap.numpy())


def densest_round(ref, lock, words=32):
    """(the most strobes any warp round -- an aligned run of `words` 32-sample words -- holds, per word; the most any
    one word holds): the time2 staging of a round is sized for 11 per word (T2_MAX_PER_WORD)"""
    best, best_word = 0.0, 0
    for chain in ref.chains:
        s = np.unpackbits(ref.taps[chain]["strobe"][lock], bitorder="little")[:ref.M]
        per_word = s[:len(s) // 32 * 32].reshape(-1, 32).sum(axis=1, dtype=np.int64)
        n = len(per_word) // words * words
        if n:
            best = max(best, float(per_word[:n].reshape(-1, words).sum(axis=1).max()) / words)
        if len(per_word):
            best_word = max(best_word, int(per_word.max()))
    return best, best_word
