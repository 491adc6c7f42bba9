"""Kernel-level profile of the device-resident benchmark step (torch.profiler, CUDA activities).

    python tools/profile_step.py [--workload t1x2|s1|both|d3|d3s] [--mib 1024] [--steps 3] [--warmup 2] [--trace FILE]

Runs `--warmup` untimed steps, then `--steps` profiled ones, exactly as bench.py's device-resident leg does (reset,
one push of the whole capture, flush).  Prints, averaged over the profiled steps:
  * every kernel's device time and launch count per step;
  * the stages of the step (demod, clock lanes, their verification, time2, run-length bit sync, gather + framer) with
    their device time and their span on the device clock (first kernel start -> last kernel end, from the step's
    first kernel);
  * how much of the run-length stage's kernel time lies inside the clock lanes' span, and the step's span.
The trace itself goes to --trace (default: a temporary directory) as Chrome JSON.
"""
import argparse
import collections
import importlib
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# stage of a kernel, by the first pattern its name matches
STAGES = [
    ("demod", r"^k1_|k1_demod"),
    ("clock lanes", r"k2a2?_lanes_kernel"),
    ("clock verify", r"k2a_(verify|fixseg|fixup)"),
    ("time2", r"k2t_|t2scan_"),
    ("run-length", r"k2p1_|k2pc_|k2p2_|k2p_fold|k2m_|k2c_|cscan_"),
    ("gather+framer", r"k3_|k4_"),
    ("reset", r"wmb_reset"),
]


def stage_of(name):
    for st, pat in STAGES:
        if re.search(pat, name):
            return st
    return "other"


def short(name):
    name = re.sub(r"^void ", "", name)
    return re.sub(r"\(.*$", "", name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="t1x2")
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--trace", default=None, help="where to write the Chrome trace (default: a temporary directory)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    bench = importlib.import_module("bench")
    pkg = importlib.import_module("rtl-wmbus_b200")
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    lib = pkg.load_library()

    wl = bench.workload_def(args.workload, args.mib)
    n_bytes = args.mib << 20
    cap, _ = synth.synth_capture(n_bytes, fs=wl["fs"], emitters=synth.default_emitters(wl["emitters"]),
                                 seed=shard.capture_seed(2, 0), device="cuda", center_shift_hz=wl.get("shift", 0.0))
    torch.cuda.synchronize()
    ctx = pkg.WmbusB200(wl["flags"], lib=lib, max_batch_mib=min(args.mib, 1024))
    for _ in range(args.warmup):
        ctx.reset()
        ctx.process_device(cap.data_ptr(), n_bytes, flush=True, raw=True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            ctx.reset()
            ctx.process_device(cap.data_ptr(), n_bytes, flush=True, raw=True)
        torch.cuda.synchronize()
    tmpdir = None
    path = args.trace
    if path is None:
        tmpdir = tempfile.mkdtemp(prefix="wmb_profile_")
        path = os.path.join(tmpdir, "step.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    # one step = everything from one wmb_reset kernel to the next
    steps, cur = [], None
    for e in kernels:
        if "wmb_reset" in e["name"]:
            cur = []
            steps.append(cur)
        if cur is not None:
            cur.append(e)
    if len(steps) != args.steps:
        raise SystemExit(f"found {len(steps)} steps in the trace, expected {args.steps}")

    n = len(steps)
    per_kernel = collections.defaultdict(lambda: [0.0, 0])
    stage_time = collections.defaultdict(float)
    stage_span = collections.defaultdict(lambda: [0.0, 0.0])
    rl_inside, step_span, streams = 0.0, 0.0, collections.defaultdict(set)
    for ks in steps:
        t0 = min(e["ts"] for e in ks)
        lo, hi = {}, {}
        for e in ks:
            k = short(e["name"])
            per_kernel[k][0] += e["dur"] / 1e3
            per_kernel[k][1] += 1
            st = stage_of(e["name"])
            stage_time[st] += e["dur"] / 1e3
            streams[st].add(e.get("args", {}).get("stream"))
            lo[st] = min(lo.get(st, e["ts"]), e["ts"])
            hi[st] = max(hi.get(st, e["ts"] + e["dur"]), e["ts"] + e["dur"])
        for st in lo:
            stage_span[st][0] += (lo[st] - t0) / 1e3
            stage_span[st][1] += (hi[st] - t0) / 1e3
        step_span += (max(e["ts"] + e["dur"] for e in ks) - t0) / 1e3
        if "clock lanes" in lo:
            a, b = lo["clock lanes"], hi["clock lanes"]
            for e in ks:
                if stage_of(e["name"]) == "run-length":
                    rl_inside += max(0.0, min(b, e["ts"] + e["dur"]) - max(a, e["ts"])) / 1e3

    dev = torch.cuda.get_device_name(0)
    print(f"{dev}, workload {args.workload} ({wl['flags'] or 'default flags'}), {args.mib} MiB, {n} profiled steps; "
          f"times in ms per step")
    print("\nkernel                                              ms/step  launches/step")
    for k, (t, c) in sorted(per_kernel.items(), key=lambda kv: -kv[1][0]):
        print(f"  {k[:48]:48s} {t / n:9.4f} {c / n:8.1f}")
    print("\nstage              kernel ms   span from step start (ms)   streams")
    for st, _ in STAGES + [("other", "")]:
        if st not in stage_time:
            continue
        a, b = stage_span[st]
        print(f"  {st:16s} {stage_time[st] / n:9.4f}   {a / n:8.4f} -> {b / n:8.4f}        {len(streams[st])}")
    print(f"\nrun-length kernel time inside the clock lanes' span: {rl_inside / n:.4f} ms of "
          f"{stage_time.get('run-length', 0.0) / n:.4f} ms")
    print(f"step span (first to last kernel): {step_span / n:.4f} ms")
    print(f"trace: {path}")


if __name__ == "__main__":
    main()
