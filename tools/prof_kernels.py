"""Device time of every kernel in one warmed compression, by torch.profiler with CUDA activities.

usage: prof_kernels.py [--inputs text5,web5] [--lib LIB.so] [--match k_split,k_mb_setup] [--out FILE.json]
  inputs as in tools/variant_time.py (text5 is bench.py's headline C2 stream).  One untimed warm-up call, then one
  profiled call.  Prints the card's name and power limit, then per kernel: launches, total and longest device time, and
  the stage timers of the profiled call (last_stats).  --match: only kernels whose name contains one of the words.
"""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from corpus import synth_binary, synth_text, synth_web
import brotli_b200

INPUTS = {
    "text5": (lambda: synth_text(100_000_000, seed=20250922), 5, 22),
    "web5": (lambda: synth_web(256 << 20, seed=20250923), 5, 22),
    "text6": (lambda: synth_text(100_000_000, seed=20250922), 6, 22),
    "bin9": (lambda: synth_binary(32_000_000, seed=20250924), 9, 24),
}

ap = argparse.ArgumentParser()
ap.add_argument("--inputs", default="text5")
ap.add_argument("--lib", default=None)
ap.add_argument("--match", default="")
ap.add_argument("--out", default=None)
a = ap.parse_args()
if a.lib:
    brotli_b200.LIB_PATH = os.path.join(ROOT, "brotli_b200", a.lib)
import torch
from torch.profiler import ProfilerActivity, profile

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip(), flush=True)
words = [w for w in a.match.split(",") if w]
report = {}
for name in a.inputs.split(","):
    gen, q, w = INPUTS[name]
    d = gen()
    brotli_b200.compress_oneshot(d, q, w)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        brotli_b200.compress_oneshot(d, q, w)
        torch.cuda.synchronize()
    st = brotli_b200.last_stats()
    k = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        kn = ev.name.split("(")[0].split("<")[0].replace("void ", "")
        if words and not any(x in kn for x in words):
            continue
        r = k.setdefault(kn, [0, 0.0, 0.0])
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        r[0] += 1; r[1] += us; r[2] = max(r[2], us)
    print("%s: %d bytes, quality %d, lgwin %d; ms_entropy %.3f ms_total %.3f" % (name, len(d), q, w, st["ms_entropy"],
                                                                                   st["ms_total"]), flush=True)
    for kn, (cnt, tot, mx) in sorted(k.items(), key=lambda x: -x[1][1]):
        print("  %-32s %5d launches  total %9.1f us  longest %9.1f us" % (kn, cnt, tot, mx), flush=True)
    report[name] = {"stats": st, "kernels": {kn: {"launches": c, "total_us": t, "max_us": m} for kn, (c, t, m) in k.items()}}
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(report, f, indent=1)
