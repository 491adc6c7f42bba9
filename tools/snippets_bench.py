"""Cost of burst snippets on the benchmark's default step: the 1 GiB `-p S` t1x2 capture, device-resident, one
process_device per step, the burst report on at level 14.  Four contexts -- snippets off, mode 1, mode 2 and a second
off context (the spread between two identical sides) -- alternate step by step in one process; each step is timed with
CUDA events.
    python tools/snippets_bench.py [steps] [out.json]   prints the device, its power limit and each side's numbers"""
import importlib
import json
import subprocess
import sys

sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
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
level = (14, 14)
ctxs = {"off": pkg.WmbusB200("-p S", lib=lib, burst_level=level),
        "mode1": pkg.WmbusB200("-p S", lib=lib, burst_level=level, snippets=1),
        "mode2": pkg.WmbusB200("-p S", lib=lib, burst_level=level, snippets=2),
        "off2": pkg.WmbusB200("-p S", lib=lib, burst_level=level)}
times = {k: [] for k in ctxs}
out = {}
for rep in range(steps + 2):                             # the first two rounds warm up
    for k, ctx in ctxs.items():
        ctx.reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        lines = ctx.process_device(cap.data_ptr(), n, flush=True, raw=True)
        b.record()
        torch.cuda.synchronize()
        if rep >= 2:
            times[k].append(a.elapsed_time(b))
        recs, data = ctx.take_snippets()
        out[k] = (lines, ctx.take_bursts(), ctx.stats(), recs)
res = {"device": dev, "power_limit": power, "steps": steps}
for k in ctxs:
    t = sorted(times[k])
    lines, bursts, st, recs = out[k]
    row = dict(step_ms_median=t[len(t) // 2], step_ms_min=t[0], step_ms_max=t[-1], kernel_launches=st.kernel_launches,
               d2h_bytes=st.d2h_bytes, batches=st.batches, bursts=len(bursts), snippets=len(recs),
               snippet_bytes=int(recs["nbytes"].sum()) if len(recs) else 0, lost=int(recs["lost"].sum()) if len(recs) else 0,
               overflow_batches=st.overflow_batches)
    res[k] = row
    print(f"snippets {k:5s}: step {row['step_ms_median']:.2f} ms median, {t[0]:.2f}-{t[-1]:.2f} ms over {len(t)} steps; "
          f"launches {st.kernel_launches}, d2h {st.d2h_bytes} B, bursts {len(bursts)}, snippets {len(recs)} "
          f"({row['snippet_bytes']} B, {row['lost']} lost)")
for k in ("mode1", "mode2", "off2"):
    assert out[k][0] == out["off"][0], f"{k} changed the lines"
if len(sys.argv) > 2:
    json.dump(res, open(sys.argv[2], "w"), indent=1)
for ctx in ctxs.values():
    ctx.close()
