"""Captures and settings of the receiver-setting tests (wmb_set_receiver: clock-lock threshold and access-code errors),
shared by the tests and tests/golden/make_golden.py, which records what reference builds with those constants changed
print for them (tests/golden/reference_runs_receiver.json)."""
import importlib
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FIXTURE = os.path.join(GOLDEN, "reference_runs_receiver.json")

# (clock lock T1/C1, S1), (access-code errors T1/C1, S1): the reference builds of oracle/Makefile RX_VARIANTS
VARIANTS = [((2, 2), (0, 0)), ((1, 1), (0, 0)), ((3, 3), (0, 0)), ((4, 4), (0, 0)), ((2, 2), (1, 1)), ((2, 2), (2, 2)),
            ((2, 2), (3, 6)), ((1, 3), (2, 4)), ((2, 2), (3, 0)), ((2, 2), (0, 6))]

# the committed captures and the flags each is recorded with
COMMITTED = {"excerpt_samples2_a.cu8": ["-v", "-v -o"], "excerpt_issue47_c1.cu8": ["-v"],
             "excerpt_issue48_2m4.cu8": ["-v -d 3 -s", "-v -d 3 -s -o"], "synth_mixed_1m6.cu8": ["-v", "-v -o"],
             "synth_mixed_2m4_shift.cu8": ["-v -d 3 -s"]}


def variant_name(lock, errors):
    return f"L{lock[0]}-{lock[1]}_E{errors[0]}-{errors[1]}"


def sync_error_emitters():
    """Telegrams whose access codes carry 1-3 (T1/C1) or 2-5 (S1) inverted chips beside clean ones: the reference's
    defaults print only the clean ones, E >= flips prints the others too."""
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    E = synth.Emitter
    return [E("T1", 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x29, period_s=0.13, start_s=0.004, seed=31),
            E("T1", 0x64700082, amp=80.0, offset_hz=-6e3, l_field=0x19, period_s=0.17, start_s=0.040, seed=32, sync_flips=(2,)),
            E("C1A", 0x20338739, amp=60.0, offset_hz=-5e3, l_field=0x19, period_s=0.19, start_s=0.070, seed=33, sync_flips=(1, 6)),
            E("T1", 0x20210116, amp=70.0, offset_hz=4e3, l_field=0x19, period_s=0.23, start_s=0.100, seed=34, sync_flips=(0, 4, 9)),
            E("S1", 0x19131290, amp=70.0, offset_hz=2e3, l_field=0x19, period_s=0.29, start_s=0.020, seed=35, sync_flips=(3, 10)),
            E("S1", 0x02717473, amp=60.0, offset_hz=-3e3, l_field=0x19, period_s=0.31, start_s=0.150, seed=36, sync_flips=(1, 5, 9, 14, 20))]


# name: (bytes, fs, emitters, seed, flags) -- synthesised on the CPU by seed, checked against the recorded sha256
SYNTH = {"sync_errors_1m6": (3 << 20, 1.6e6, "sync_errors", 0xB2000061, ["-v", "-v -o"]),
         "noise_1m6": (4 << 20, 1.6e6, "none", 0xB2000062, ["-v"])}


def synth_capture(name):
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    n, fs, em, seed, _ = SYNTH[name]
    emitters = sync_error_emitters() if em == "sync_errors" else []
    buf, _ = synth.synth_capture(n, fs=fs, emitters=emitters, seed=seed)
    return np.ascontiguousarray(buf.numpy())


def capture(name):
    if name in SYNTH:
        return synth_capture(name)
    return np.fromfile(os.path.join(GOLDEN, name), np.uint8)


def cases():
    """(capture name, flags) pairs the fixture holds lines for"""
    out = [(name, fl) for name, fls in COMMITTED.items() for fl in fls]
    return out + [(name, fl) for name, v in SYNTH.items() for fl in v[4]]


_fixture = None


def load_fixture():
    global _fixture
    if _fixture is None:
        with open(FIXTURE) as f:
            _fixture = json.load(f)
    return _fixture


_captures = {}


def cached_capture(name):
    if name not in _captures:
        cu8 = capture(name)
        if name in SYNTH:
            import orc
            assert orc.capture_sha(cu8) == load_fixture()["capture_sha256"][name], "the generator's capture changed"
        _captures[name] = cu8
    return _captures[name]


def want_lines(lock, errors, name, flags):
    return load_fixture()["lines"][variant_name(lock, errors)][f"{name}|{flags}"]


def check_lines(pkg, lib, name, flags, lock, errors, pushes=None, **tuning):
    """the product's lines, in order, against what the reference built with these settings printed"""
    import pipeline_checks as pc
    got, st = pc.run_lines(pkg, lib, cached_capture(name), flags, pushes=pushes, clock_lock=lock,
                           access_code_errors=errors, **tuning)
    want = want_lines(lock, errors, name, flags)
    assert got == want, (name, flags, lock, errors, pushes, tuning, len(got), len(want))
    assert st.overflow_batches == 0
    return st


def check_stages(pkg, lib, cu8, flags, lock, errors, **tuning):
    """time2 strobes (wmb_debug_copy_bits(.., 1, ..)) and every (chain, algorithm)'s decoder calls
    (wmb_debug_copy_events) of one batch against the oracle with the same settings (receiver_oracle)"""
    import orc
    import receiver_oracle as ro
    o = orc.opts_from_flags(flags)
    gran = 4096 * max(1, o.decimation)
    data = np.ascontiguousarray(cu8[:len(cu8) // gran * gran], np.uint8)
    n_sync = 0
    with pkg.WmbusB200(flags, lib=lib, clock_lock=lock, access_code_errors=errors, **tuning) as ctx:
        ctx.process(data.ctypes.data, len(data), flush=True)
        assert ctx.stats().batches == 1
        for chain in (0, 1):
            st = orc.stages(data, o, chain)
            got = ctx.debug_bits(chain, 1, st["M"])
            bad = np.nonzero(got != ro.strobes(st["clk"], lock[chain]))[0]
            assert len(bad) == 0, (flags, lock, chain, "strobe", len(bad), bad[:5])
            for algo in (0, 1):
                want = ro.stream_events(st, chain, algo, lock[chain], errors[chain])
                ev = ctx.debug_events(chain, algo)
                assert len(ev["m"]) == len(want["m"]), (flags, lock, errors, chain, algo, len(ev["m"]), len(want["m"]))
                for f in ("m", "bit", "sync", "rssi") + (("reset",) if algo == 0 else ()):
                    bad = np.nonzero(ev[f] != want[f].astype(np.uint64))[0]
                    assert len(bad) == 0, (flags, lock, errors, chain, algo, f, len(bad), bad[:5])
                n_sync += int(want["sync"].sum())
    return n_sync


def check_time_chunks(pkg, lib, cu8, flags, lock, errors, world=3, halo_m=1 << 18, d=2, **tuning):
    """time-chunk sharding (shard.decode_time_chunk, one context per chunk) with these settings: the merged lines are
    the oracle's sequential run"""
    import receiver_oracle as ro
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    want = ro.run_lines(cu8, flags, lock, errors)
    got, ends = [], []
    for rank in range(world):
        h = halo_m
        while True:
            with pkg.WmbusB200(flags, lib=lib, clock_lock=lock, access_code_errors=errors, **tuning) as ctx:
                push = lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo)
                lines, ds, de, start = shard.decode_time_chunk(ctx, push, len(cu8), d, rank, world, h)
            if rank == 0 or start == 0 or ds == ends[rank - 1]:
                break
            h *= 4
        ends.append(de)
        got.append(lines)
    assert shard.merge_lines(got) == want
    assert len(want) > 10 and all(len(part) > 0 for part in got)
