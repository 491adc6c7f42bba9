"""What erasure repair on the streaming path (wmb_set_repair) and the C1 / T1 / S1 soft repairs (wmb_set_repair_soft,
wmb_set_repair_t1_soft, wmb_set_repair_s1_soft) cost and gain.
    python tools/repair_bench.py cost [steps]              GPU: step times, repair off against e_max 3, e_max 3 + k_max 6
                                                           and e_max 3 + s_max 6
    python tools/repair_bench.py gain [--cpu] [MiB]        the noise sweep (GPU library, or the CPU build with --cpu)
    python tools/repair_bench.py gain-soft [--cpu] [MiB]   the same for C1 telegrams and k_max 1 .. 6
    python tools/repair_bench.py gain-t1soft [--cpu] [MiB] the same for T1 telegrams: e_max 1 and 3, then s_max 1 .. 6
                                                           on top of e_max 3
    python tools/repair_bench.py gain-s1soft [--cpu] [MiB] the same for S1 telegrams and the S1 soft rule
    python tools/repair_bench.py cost-s1 [steps]           GPU: as cost, on a 1 GiB capture of the `s1` config with the S1
                                                           chain on: off, e_max 3, e_max 3 + S1 s_max 6, off again

cost: the benchmark's default step -- 1 GiB of synthetic 1.6 MS/s cu8 with two T1 emitters, `-p S`, device-resident, one
process_device per step -- then the same at clock lock 1 with T1/C1 access-code errors 3 (about 486 k matches per
step).  A context with repair off and one at e_max 3 alternate step by step in one process; each step is timed with
CUDA events and the medians are printed, with kernel launches and D2H bytes per step, the device and its power limit.

gain: for each noise sigma, a capture with T1 and S1 emitters whose chips are all sent right (no data_flips), decoded
at e_max 1, 2 and 3: the telegrams sent, those decoded CRC-ok by either algorithm, those recovered only by repair, and
the wrong repairs (a REPAIRED datagram that was never sent).  The counts are exact: the GPU and the CPU build agree.

gain-soft: the same sweep with one C1A (L = 0x29) and one C1B (L = 0x7F: a full 128-byte block) emitter, no planted
errors, at k_max 1 .. 6: the C1 telegrams recovered only by the soft repair, and the wrong repairs, split by frame
format (frame B's 128-byte block has code words of weight 2, DESIGN.md section 8).

gain-t1soft: the same sweep with two T1 emitters only, a short (L = 0x19) and a long (L = 0xC8) telegram, no planted
errors: the telegrams recovered only by erasure repair at e_max 1 and 3, then only by repair at e_max 3 plus the T1 soft
rule at s_max 1 .. 6, and the wrong repairs at each s_max split into erasure / soft by the record's soft_t1.

gain-s1soft: the same with two S1 emitters (L = 0x19 and L = 0xC8) and the S1 soft rule (soft_s1).

cost-s1: the `cost` step runs `-p S`, where the S1 chain is off; this one decodes 1 GiB of the `s1` config (S1 emitters)
with both chains on."""
import importlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

pkg = importlib.import_module("rtl-wmbus_b200")
synth = importlib.import_module("rtl-wmbus_b200.synth")
shard = importlib.import_module("rtl-wmbus_b200.shard")

SIGMAS = (8.0, 56.0, 64.0, 72.0, 80.0, 88.0, 96.0, 112.0)


def power_limit():
    import torch
    try:
        return subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                               # the query is informational
        return f"unknown ({e})"


def cost(steps, s1=False):
    import torch
    lib = pkg.load_library()
    n = 1 << 30
    cap, _ = synth.synth_capture(n, fs=1.6e6, emitters=synth.default_emitters("s1" if s1 else "t1x2"),
                                 seed=shard.capture_seed(3 if s1 else 2, 0), device="cuda")
    torch.cuda.synchronize()
    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    legs = (("s1 config, both chains", {}),) if s1 else (("defaults", {}), ("clock lock 1, T1/C1 access-code errors 3",
                                                         dict(clock_lock=(1, 2), access_code_errors=(3, 0))))
    flags = "" if s1 else "-p S"
    for name, rx in legs:
        # two contexts with repair off: where a step overflows its tables, they show how far the lines of two
        # contexts agree without repair
        ctxs = {"off": pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, **rx),
                "e_max 3": pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, repair=3, **rx)}
        if s1:
            ctxs["e3 S1s6"] = pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, repair=3, repair_s1_soft=6, **rx)
        else:
            ctxs["e3 k6"] = pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, repair=3, repair_soft=6, **rx)
            ctxs["e3 s6"] = pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, repair=3, repair_t1_soft=6, **rx)
        ctxs["off (2)"] = pkg.WmbusB200(flags, lib=lib, max_batch_mib=1024, **rx)
        times = {k: [] for k in ctxs}
        out = {}
        for rep in range(steps + 2):                     # the first two rounds warm up
            for k, ctx in ctxs.items():
                ctx.reset()
                before = ctx.stats()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                lines = ctx.process_device(cap.data_ptr(), n, flush=True, raw=True)
                b.record()
                torch.cuda.synchronize()
                if rep >= 2:
                    times[k].append(a.elapsed_time(b))
                st = ctx.stats()
                out[k] = (lines, ctx.take_repairs(), st.kernel_launches - before.kernel_launches,
                          st.d2h_bytes - before.d2h_bytes, st.candidates[0][0] + st.candidates[0][1],
                          st.overflow_batches - before.overflow_batches)
        print(f"-- {name}: {out['off'][4]} access-code matches per step, overflow batches per step {out['off'][5]}")
        for k in ctxs:
            t = sorted(times[k])
            lines, recs, launches, d2h, _m, _o = out[k]
            print(f"  repair {k:8s}: step {t[len(t) // 2]:.2f} ms median, {t[0]:.2f}-{t[-1]:.2f} ms over {len(t)} steps; "
                  f"kernel launches {launches}, d2h bytes {d2h}, records {len(recs)}, "
                  f"{lines.count(b'\n')} lines, same lines as 'off': {lines == out['off'][0]}")
        for ctx in ctxs.values():
            ctx.close()


def gain(cpu, mib):
    if cpu:
        from conftest import HOSTSIM_SO
        lib = pkg.load_library(HOSTSIM_SO)
    else:
        import torch
        lib = pkg.load_library()
        print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    ems = [synth.Emitter("T1", 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x29, period_s=0.10, start_s=0.004, seed=31),
           synth.Emitter("S1", 0x19131290, amp=90.0, offset_hz=2e3, l_field=0x19, period_s=0.10, start_s=0.054, seed=32)]
    print(f"{mib} MiB of 1.6 MS/s cu8 per sigma, one T1 (L = 0x29) and one S1 (L = 0x19) emitter at amplitude 90, -v, "
          f"{'CPU build' if cpu else 'GPU'}")
    print("sigma  sent  crc_ok  +rep1  +rep2  +rep3  wrong1  wrong2  wrong3")
    for sigma in SIGMAS:
        cu8, plan = synth.synth_capture(mib << 20, emitters=ems, seed=0xB2000100 + int(sigma), noise_sigma=sigma)
        cu8 = np.ascontiguousarray(cu8.numpy())
        sent = {ems[p.emitter].payload(p.k) for p in plan}
        row = [len(plan)]
        ok = None
        for e_max in (1, 2, 3):
            with pkg.WmbusB200("-v", lib=lib, repair=e_max, max_batch_mib=min(mib, 1024)) as ctx:
                lines = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
                recs = ctx.take_repairs()
            if ok is None:
                ok = {bytes.fromhex(l.split(";")[8][2:]) for l in lines if l.split(";")[2] == "1"} & sent
                row.append(len(ok))
            rep = {bytes(r.line.datagram[:r.line.len]) for r in recs if r.repair.outcome == 1}
            row.append(len((rep & sent) - ok))
            row.append(len(rep - sent))
        print(f"{sigma:5.1f}  {row[0]:4d}  {row[1]:6d}  {row[2]:5d}  {row[4]:5d}  {row[6]:5d}  {row[3]:6d}  {row[5]:6d}  "
              f"{row[7]:6d}")


def gain_soft(cpu, mib):
    if cpu:
        from conftest import HOSTSIM_SO
        lib = pkg.load_library(HOSTSIM_SO)
    else:
        import torch
        lib = pkg.load_library()
        print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    ems = [synth.Emitter("C1A", 0x20338739, amp=90.0, offset_hz=-5e3, l_field=0x29, period_s=0.10, start_s=0.004, seed=33),
           synth.Emitter("C1B", 0x20210116, amp=90.0, offset_hz=4e3, l_field=0x7F, period_s=0.10, start_s=0.054, seed=34)]
    print(f"{mib} MiB of 1.6 MS/s cu8 per sigma, one C1A (L = 0x29) and one C1B (L = 0x7F) emitter at amplitude 90, -v, "
          f"e_max 1, {'CPU build' if cpu else 'GPU'}")
    print("sigma  sent  crc_ok  " + "  ".join(f"+k{k}" for k in range(1, 7)) + "   wrong A/B at k 1..6")
    for sigma in SIGMAS:
        cu8, plan = synth.synth_capture(mib << 20, emitters=ems, seed=0xB2000200 + int(sigma), noise_sigma=sigma)
        cu8 = np.ascontiguousarray(cu8.numpy())
        sent = {ems[p.emitter].payload(p.k) for p in plan}
        ok, gained, wrong = None, [], []
        for k in range(1, 7):
            with pkg.WmbusB200("-v", lib=lib, repair=1, repair_soft=k, max_batch_mib=min(mib, 1024)) as ctx:
                lines = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
                recs = ctx.take_repairs()
            if ok is None:
                ok = {bytes.fromhex(l.split(";")[8][2:]) for l in lines if l.split(";")[2] == "1"} & sent
            rep = {bytes(r.line.datagram[:r.line.len]) for r in recs
                   if r.repair.outcome == 1 and bytes(r.line.mode[:2]) == b"C1"}
            gained.append(len((rep & sent) - ok))
            bad = rep - sent
            nb = sum(1 for d in bad if len(d) > 1 and d[0] >= 0x7F - 8)           # by L: the C1B emitter's telegrams
            wrong.append(f"{len(bad) - nb}/{nb}")
        print(f"{sigma:5.1f}  {len(plan):4d}  {len(ok):6d}  " + "  ".join(f"{g:3d}" for g in gained) + "   " + " ".join(wrong))


def gain_t1soft(cpu, mib, mode="T1"):
    if cpu:
        from conftest import HOSTSIM_SO
        lib = pkg.load_library(HOSTSIM_SO)
    else:
        import torch
        lib = pkg.load_library()
        print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    s1 = mode == "S1"
    period = 0.25 if s1 else 0.10                   # an L = 0xC8 S1 telegram lasts 111 ms at 32.768 kchip/s
    ems = [synth.Emitter(mode, 0x71200023, amp=90.0, offset_hz=8e3, l_field=0x19, period_s=period, start_s=0.004, seed=35),
           synth.Emitter(mode, 0x71200024, amp=90.0, offset_hz=-3e3, l_field=0xC8, period_s=period, start_s=0.054, seed=36)]
    print(f"{mib} MiB of 1.6 MS/s cu8 per sigma, two {mode} emitters (L = 0x19, L = 0xC8) at amplitude 90, -v, "
          f"{'CPU build' if cpu else 'GPU'}")
    print("sigma  sent  crc_ok  +e1  +e3  " + "  ".join(f"+s{k}" for k in range(1, 7)) + "   wrong erasure/soft at s 1..6")
    for sigma in SIGMAS:
        cu8, plan = synth.synth_capture(mib << 20, emitters=ems, seed=(0xB2000400 if s1 else 0xB2000300) + int(sigma),
                                        noise_sigma=sigma)
        cu8 = np.ascontiguousarray(cu8.numpy())
        sent = {ems[p.emitter].payload(p.k) for p in plan}
        ok, gained, wrong = None, [], []
        for e_max, s_max in [(1, 0), (3, 0)] + [(3, s) for s in range(1, 7)]:
            soft = dict(repair_s1_soft=s_max) if s1 else dict(repair_t1_soft=s_max)
            with pkg.WmbusB200("-v", lib=lib, repair=e_max, max_batch_mib=min(mib, 1024), **soft) as ctx:
                lines = ctx.process(cu8.ctypes.data, len(cu8), flush=True)
                recs = ctx.take_repairs()
            if ok is None:
                ok = {bytes.fromhex(l.split(";")[8][2:]) for l in lines if l.split(";")[2] == "1"} & sent
            rep = [(bytes(r.line.datagram[:r.line.len]), r.soft_s1 if s1 else r.soft_t1) for r in recs
                   if r.repair.outcome == 1]
            gained.append(len(({d for d, _ in rep} & sent) - ok))
            if s_max:
                wrong.append(f"{sum(1 for d, s in rep if d not in sent and not s)}/{sum(1 for d, s in rep if d not in sent and s)}")
        print(f"{sigma:5.1f}  {len(plan):4d}  {len(ok):6d}  {gained[0]:3d}  {gained[1]:3d}  "
              + "  ".join(f"{g:3d}" for g in gained[2:]) + "   " + " ".join(wrong))


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "cost"
    if what == "cost":
        cost(int(sys.argv[2]) if len(sys.argv) > 2 else 8)
    elif what == "cost-s1":
        cost(int(sys.argv[2]) if len(sys.argv) > 2 else 8, s1=True)
    elif what == "gain-s1soft":
        rest = [a for a in sys.argv[2:] if a != "--cpu"]
        gain_t1soft("--cpu" in sys.argv[2:], int(rest[0]) if rest else 32, "S1")
    elif what == "gain-t1soft":
        rest = [a for a in sys.argv[2:] if a != "--cpu"]
        gain_t1soft("--cpu" in sys.argv[2:], int(rest[0]) if rest else 32)
    elif what == "gain-soft":
        rest = [a for a in sys.argv[2:] if a != "--cpu"]
        gain_soft("--cpu" in sys.argv[2:], int(rest[0]) if rest else 16)
    elif what == "gain":
        rest = [a for a in sys.argv[2:] if a != "--cpu"]
        gain("--cpu" in sys.argv[2:], int(rest[0]) if rest else 32)
    else:
        raise SystemExit(__doc__)
