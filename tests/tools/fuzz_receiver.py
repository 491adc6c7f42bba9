"""Differential fuzzing of the receiver settings (wmb_set_receiver) on the CPU build (tests/hostsim) against the oracle
with the same settings (tests/receiver_oracle.py): the random captures, flags, lane geometry and push patterns of
tests/fuzz_cases.py, plus a clock lock (1..16) and access-code errors (up to 3 / 6) per chain from a generator of their
own, so the cases of fuzz_hostsim.py / fuzz_time_chunks.py with the same seed keep their numbers.
    python tests/tools/fuzz_receiver.py [seconds] [seed] [chunks]     prints one line per case; exits 1 at the first mismatch
`chunks` decodes each case in 2-4 time chunks (fuzz_cases.draw_time_chunk_case, shard.decode_time_chunk) instead."""
import importlib, sys, time
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import numpy as np
import fuzz_cases, pipeline_checks as pc, receiver_oracle as ro
from conftest import HOSTSIM_SO
pkg = importlib.import_module("rtl-wmbus_b200"); shard = importlib.import_module("rtl-wmbus_b200.shard")
lib = pkg.load_library(HOSTSIM_SO)
budget = float(sys.argv[1]) if len(sys.argv) > 1 else 600.0
seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1
chunks = len(sys.argv) > 3 and sys.argv[3] == "chunks"
rng = np.random.default_rng(seed)
rng_rx = np.random.default_rng(seed + 2000003)


def draw_receiver(r):
    """clock lock and access-code errors per chain; about a third of the cases keep the defaults of one of them"""
    lock = tuple(int(r.choice([1, 1, 2, 3, 4, int(r.integers(5, 17))])) for _ in range(2))
    errors = (int(r.integers(0, 4)), int(r.integers(0, 7)))
    if r.random() < 0.33:
        if r.random() < 0.5:
            lock = (2, 2)
        else:
            errors = (0, 0)
    return lock, errors


def decode_chunks(c, cu8, rx):
    world, halo = c["world"], c["halo"]
    geom = {k: v for k, v in c["tuning"].items() if k in ("chunk_samples", "warmup_samples")}
    got, ends, overflow = [], [], 0
    for rank in range(world):
        h = halo
        while True:
            with pkg.WmbusB200(c["flags"], lib=lib, max_batch_mib=1, **geom, **rx) as ctx:
                lines, ds, de, start = shard.decode_time_chunk(ctx, lambda lo, hi: ctx.push(cu8.ctypes.data + lo, hi - lo),
                                                               len(cu8), c["d"], rank, world, h)
                overflow += ctx.stats().overflow_batches
            if rank == 0 or start == 0 or ds == ends[rank - 1] or h > (1 << 24):
                break
            h *= 4
        ends.append(de); got.append(lines)
    return shard.merge_lines(got), overflow


t_end = time.time() + budget
k = 0
while time.time() < t_end:
    k += 1
    c = fuzz_cases.draw_time_chunk_case(rng) if chunks else fuzz_cases.draw_case(rng)
    if c is None or c.get("prefilter"):
        continue
    lock, errors = draw_receiver(rng_rx)
    rx = dict(clock_lock=lock, access_code_errors=errors)
    print("start %d flags=%r d=%d n=%d sigma=%g rx=%r tuning=%r pushes=%r" % (k, c["flags"], c["d"], c["n"], c["sigma"], rx,
                                                                            c["tuning"], c.get("pushes")), flush=True)
    cu8 = fuzz_cases.build_capture(c)
    want = ro.run_lines(cu8, c["flags"], lock, errors)
    if chunks:
        got, overflow = decode_chunks(c, cu8, rx)
    else:
        got, st = pc.run_lines(pkg, lib, cu8, c["flags"], pushes=c["pushes"], **c["tuning"], **rx)
        overflow = st.overflow_batches
    ok = got == want
    lost = 0
    if not ok and overflow:                                  # a device table was full: lines may be missing, none may be invented
        it = iter(want)
        ok = all(any(l == w for w in it) for l in got)
        lost = len(want) - len(got)
    print("case %d (seed %d) %s lines=%d overflow_batches=%d lost=%d" % (k, seed, "ok" if ok else "MISMATCH", len(want),
                                                                        overflow, lost), flush=True)
    if not ok:
        print("got", len(got), "want", len(want)); sys.exit(1)
print("done", k, "cases")
