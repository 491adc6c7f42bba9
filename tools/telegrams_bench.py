"""Host cost of telegram records on the benchmark's default step: the 1 GiB `-p S` t1x2 capture, device-resident, one
process_device per step at the benchmark's batch size (1 GiB).  Three contexts -- telegrams off, on, and a second off
context (the spread between two identical sides) -- alternate step by step in one process.  A step is the wall time of
process_device plus wmb_take_telegrams into preallocated arrays (both end in a device synchronise, so this is the host's
view of the step); wmb_take_telegrams is also timed alone.  The records are handed out through the C call directly, so
the numbers hold the library's host work and not the Python wrapper's per-record loop.
    python tools/telegrams_bench.py [steps] [out.json]   prints the device, its power limit and each side's numbers"""
import ctypes as C
import importlib
import json
import subprocess
import sys
import time

sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import numpy as np
import torch

pkg = importlib.import_module("rtl-wmbus_b200")
synth = importlib.import_module("rtl-wmbus_b200.synth")
shard = importlib.import_module("rtl-wmbus_b200.shard")
lib = pkg.load_library()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 8
n = 1 << 30
cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=shard.capture_seed(2, 0),
                             device="cuda")
torch.cuda.synchronize()
try:
    power = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                   # the query is informational
    power = f"unknown ({e})"
dev = torch.cuda.get_device_name()
print(f"device: {dev}  power limit: {power}")
ctxs = {"off": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024),
        "on": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024, telegrams=True),
        "off2": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024)}
recs = np.zeros(1 << 14, pkg.telegram_dtype())
buf = np.zeros(len(recs) * 292, np.uint8)


def take_all(ctx):
    """wmb_take_telegrams until it hands out nothing; returns the records' count and decoded count"""
    n, total, dec = C.c_size_t(0), 0, 0
    while True:
        ctx._check(lib.wmb_take_telegrams(ctx._ctx, recs.ctypes.data, len(recs), buf.ctypes.data, len(buf), C.byref(n)))
        if not n.value:
            return total, dec
        total += n.value
        dec += int(recs["decoded"][:n.value].sum())


times = {k: [] for k in ctxs}
take_ms = []
out = {}
for rep in range(steps + 2):                             # the first two rounds warm up
    for k, ctx in ctxs.items():
        ctx.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lines = ctx.process_device(cap.data_ptr(), n, flush=True, raw=True)
        t1 = time.perf_counter()
        got = take_all(ctx)
        t2 = time.perf_counter()
        if rep >= 2:
            times[k].append((t2 - t0) * 1e3)
            if k == "on":
                take_ms.append((t2 - t1) * 1e3)
        out[k] = (lines, ctx.stats(), got)
res = {"device": dev, "power_limit": power, "steps": steps}
for k in ctxs:
    t = sorted(times[k])
    lines, st, (n_rec, n_dec) = out[k]
    row = dict(step_ms_median=t[len(t) // 2], step_ms_min=t[0], step_ms_max=t[-1], kernel_launches=st.kernel_launches,
               d2h_bytes=st.d2h_bytes, lines=lines.count(b"\n"), telegrams=n_rec, decoded=n_dec)
    res[k] = row
    print(f"telegrams {k:4s}: step {row['step_ms_median']:.2f} ms median, {t[0]:.2f}-{t[-1]:.2f} ms over {len(t)} steps; "
          f"launches {st.kernel_launches}, d2h {st.d2h_bytes} B, lines {row['lines']}, records {n_rec} "
          f"({row['decoded']} decoded)")
tk = sorted(take_ms)
res["take_telegrams_ms"] = dict(median=tk[len(tk) // 2], min=tk[0], max=tk[-1])
print(f"wmb_take_telegrams alone: {tk[len(tk) // 2]:.3f} ms median, {tk[0]:.3f}-{tk[-1]:.3f} ms")
for k in ("on", "off2"):
    assert out[k][0] == out["off"][0], f"{k} changed the lines"
    assert (out[k][1].kernel_launches, out[k][1].d2h_bytes) == (out["off"][1].kernel_launches, out["off"][1].d2h_bytes)
if len(sys.argv) > 2:
    json.dump(res, open(sys.argv[2], "w"), indent=1)
for ctx in ctxs.values():
    ctx.close()
