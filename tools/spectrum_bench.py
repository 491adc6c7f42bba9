"""Cost of the band survey on the benchmark's default step: the 1 GiB `-p S` t1x2 capture, device-resident, one
process_device per step.  Two contexts, one without the survey and one at the CLI's default N = 1024, B = 16384,
alternate step by step in one process; each step is timed with CUDA events.  The survey kernel's own time comes from a
third context with both chains off (`-p T -p S`: the demod kernel has nothing to do), less the same context without the
survey.
    python tools/spectrum_bench.py [steps] [bins] [blocks]
prints the device, its power limit, both sides' step times, the survey's time and its fp32 operation rate."""
import importlib
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

pkg = importlib.import_module("rtl-wmbus_b200")
synth = importlib.import_module("rtl-wmbus_b200.synth")
shard = importlib.import_module("rtl-wmbus_b200.shard")
lib = pkg.load_library()
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 8
N = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
B = int(sys.argv[3]) if len(sys.argv) > 3 else 16384
n = 1 << 30
cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=synth.default_emitters("t1x2"), seed=shard.capture_seed(2, 0),
                             device="cuda")
torch.cuda.synchronize()
try:                                                     # the card and its power limit in one query
    card = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=name,power.limit",
                           "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                   # the query is informational
    card = f"{torch.cuda.get_device_name()}, power limit unknown ({e})"
print(f"device, power limit: {card}")
ctxs = {"off": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024),
        "on": pkg.WmbusB200("-p S", lib=lib, max_batch_mib=1024, spectrum=(N, B)),
        "bare": pkg.WmbusB200("-p T -p S", lib=lib, max_batch_mib=1024),
        "bare+survey": pkg.WmbusB200("-p T -p S", lib=lib, max_batch_mib=1024, spectrum=(N, B))}
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
        out[k] = (lines, ctx.take_spectrum(), ctx.stats())
med = {}
for k in ctxs:
    t = sorted(times[k])
    med[k] = t[len(t) // 2]
    st = out[k][2]
    print(f"survey {k:11s}: step {med[k]:.2f} ms median, {t[0]:.2f}-{t[-1]:.2f} ms over {len(t)} steps; "
          f"kernel launches {st.kernel_launches}, d2h bytes {st.d2h_bytes}, records {len(out[k][1][0])}")
# fp32 operations per block as the definition counts them (every separately rounded operation): per sample 2 converts
# (u - 127.5f) and 2 window products; per butterfly 4 products, 2 sums (the twiddle product) and 4 sums (a +- t); per
# bin 2 products and 1 sum (the power)
blocks = n // (2 * N)
ops = blocks * (4 * N + 10 * (N // 2) * int(math.log2(N)) + 3 * N)
survey_ms = med["bare+survey"] - med["bare"]
print(f"survey cost on the step: {med['on'] - med['off']:.2f} ms; survey kernels alone: {survey_ms:.2f} ms "
      f"({blocks} blocks of {N}, {ops / 1e9:.1f} G fp32 operations, {ops / (survey_ms * 1e-3) / 1e12:.2f} T operations/s)")
assert out["on"][0] == out["off"][0], "the survey changed the lines"
for ctx in ctxs.values():
    ctx.close()
