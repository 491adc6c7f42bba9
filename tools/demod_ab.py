"""A/B timing of two (or more) builds of the library on one card, alternating between them within one process:
   python tools/demod_ab.py A.so B.so [--workload t1x2] [--rounds 3] [--steps 5] [--warmup 2] [--out ab.json]

Every build gets its own context on the same device-resident capture (bench.py's capture for the workload, 1 GiB by
default).  A round runs each build in turn, --warmup untimed steps and then --steps timed ones, so the builds follow
each other A B A B ... and share whatever the card's clock does.  For each build it prints the median and the range
over all timed steps of
    demod_kernel_ms   the demod kernel alone (device events around the launch)
    batch_device_ms   the batch's device pass
    wall_ms           host clock around process_device(), which ends in a device synchronise
and whether its lines are identical to the first build's.  The card's name, power limit and SM clocks are read before
and after the timed rounds."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        return None
    return out[0] if out else None


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("libs", nargs="+", help="paths of libwmbus_b200.so builds; the first is the reference for the lines")
    ap.add_argument("--workload", default="t1x2")
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", help="also write the per-step samples as JSON")
    args = ap.parse_args()

    import torch
    bench = importlib.import_module("bench")
    pkg = importlib.import_module("rtl-wmbus_b200")
    synth = importlib.import_module("rtl-wmbus_b200.synth")
    shard = importlib.import_module("rtl-wmbus_b200.shard")
    wl = bench.workload_def(args.workload, args.mib)
    n = args.mib << 20
    cap, _ = synth.synth_capture(n, fs=wl["fs"], emitters=synth.default_emitters(wl["emitters"]),
                                 seed=shard.capture_seed(2, 0), device="cuda", center_shift_hz=wl.get("shift", 0.0))
    torch.cuda.synchronize()
    print(f"workload {args.workload}: {wl['desc']}", flush=True)
    print(f"card before: {card_info()}", flush=True)

    ctxs = [pkg.WmbusB200(wl["flags"], device=0, lib=pkg.load_library(p), max_batch_mib=min(args.mib, 1024))
            for p in args.libs]
    samples = [{"demod_kernel_ms": [], "batch_device_ms": [], "wall_ms": []} for _ in args.libs]
    lines = [None] * len(args.libs)
    for rnd in range(args.rounds):
        for i, ctx in enumerate(ctxs):
            for step in range(args.warmup + args.steps):
                ctx.reset()
                t0 = time.perf_counter()
                out = ctx.process_device(cap.data_ptr(), n, flush=True)
                wall = (time.perf_counter() - t0) * 1e3
                if step < args.warmup:
                    continue
                st = ctx.stats()
                samples[i]["demod_kernel_ms"].append(st.demod_kernel_ms)
                samples[i]["batch_device_ms"].append(st.batch_device_ms)
                samples[i]["wall_ms"].append(wall)
                lines[i] = out
    print(f"card after:  {card_info()}", flush=True)
    for ctx in ctxs:
        ctx.close()

    for i, path in enumerate(args.libs):
        parts = []
        for k, v in samples[i].items():
            parts.append(f"{k} {statistics.median(v):.3f} [{min(v):.3f}, {max(v):.3f}]")
        same = "same" if lines[i] == lines[0] else "DIFFERENT"
        print(f"{path}: " + "  ".join(parts) + f"  lines {len(lines[i])} {same}", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"workload": args.workload, "libs": args.libs, "samples": samples,
                       "lines_identical": [l == lines[0] for l in lines]}, f, indent=1)


if __name__ == "__main__":
    main()
