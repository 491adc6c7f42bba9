"""Cost of the signal-quality report on the benchmark's default step: the 1 GiB `-p S` t1x2 capture, device-resident, one
process_device per step.  Two contexts, one without the report and one with it, alternate step by step in one process;
each step is timed with CUDA events.
    python tools/quality_bench.py [steps] [clock_lock access_code_errors]
prints the device, its power limit and both sides' step times (e.g. `quality_bench.py 8 1 3`: clock lock 1, access-code
errors 3 on T1/C1, the dense-match case)"""
import importlib
import subprocess
import sys

sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import torch

pkg = importlib.import_module("rtl-wmbus_b200")
synth = importlib.import_module("rtl-wmbus_b200.synth")
shard = importlib.import_module("rtl-wmbus_b200.shard")
lib = pkg.load_library()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 8
rx = {}
if len(sys.argv) > 3:
    rx = dict(clock_lock=(int(sys.argv[2]), 2), access_code_errors=(int(sys.argv[3]), 0))
n = 1 << 30
cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=shard.capture_seed(2, 0),
                             device="cuda")
torch.cuda.synchronize()
try:
    power = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                   # the query is informational
    power = f"unknown ({e})"
print(f"device: {torch.cuda.get_device_name()}  power limit: {power}  receiver: {rx or 'default'}")
ctxs = {"off": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024, **rx),
        "on": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024, quality=True, **rx)}
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
        out[k] = (lines, ctx.stats())
for k in ctxs:
    t = sorted(times[k])
    st = out[k][1]
    print(f"quality {k:3s}: step {t[len(t) // 2]:.2f} ms median, {t[0]:.2f}-{t[-1]:.2f} ms over {len(t)} steps; "
          f"kernel launches {st.kernel_launches}, d2h bytes {st.d2h_bytes}, "
          f"matches {sum(st.candidates[c][a] for c in range(2) for a in range(2))}, overflow batches {st.overflow_batches}")
# a step that overflows a device table loses lines, and which ones depends on the order of the device's atomics
if not out["on"][1].overflow_batches and not out["off"][1].overflow_batches:
    assert out["on"][0] == out["off"][0], "the report changed the lines"
for ctx in ctxs.values():
    ctx.close()
