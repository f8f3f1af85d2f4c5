"""Times alternative builds of the library against each other in one process (tuning experiments).

usage: variant_time.py [--inputs text5,web5,text6,bin9] [--rounds R] LIB.so [LIB.so ...]
  LIB.so: a build of libbrotlienc_b200.so (a path, or a name under brotli_b200/).
  Every round runs each library once per input, in turn, after one untimed warm-up call per library and input, so
  that clock and thermal drift fall on every build alike.  Prints, per input and library, the median and the min-max
  of ms_walk, ms_index, ms_lz77 - ms_walk (the LZ77 stage outside the walker: chain, commits, snapshot upkeep),
  ms_entropy and ms_total (the library's own stage timers, CUDA events) and whether every build returned the same bytes.
inputs:
  text5  100 MB synthetic text (the headline's synth_text, seed 20250922), quality 5, lgwin 22
  web5   256 MiB of the synthetic web mix (synth_web, seed 20250923: the web config's generator), quality 5, lgwin 22
  text6  the same text at quality 6, lgwin 22
  bin9   32 MB synthetic binary mix (synth_binary, seed 20250924), quality 9, lgwin 24
"""
import argparse, os, statistics, sys
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
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("libs", nargs="+")
a = ap.parse_args()
libs = {}
for so in a.libs:   # load every build once; switching is a pointer swap
    brotli_b200._lib = None
    brotli_b200.LIB_PATH = os.path.join(ROOT, "brotli_b200", so)
    libs[so] = brotli_b200.lib()


def run(so, d, q, w):
    brotli_b200._lib = libs[so]
    out = brotli_b200.compress_oneshot(d, q, w)
    return out, brotli_b200.last_stats()


data = {}
for name in a.inputs.split(","):
    gen, q, w = INPUTS[name]
    if name[:-1] not in data:   # (text5 and text6 share their input)
        data[name[:-1]] = gen()
    d = data[name[:-1]]
    res = {so: [] for so in a.libs}
    outs = {}
    for so in a.libs:
        outs[so] = run(so, d, q, w)[0]
    for _ in range(a.rounds):
        for so in a.libs:
            out, st = run(so, d, q, w)
            if out != outs[so]:
                outs[so] = None
            res[so].append((st["ms_walk"], st["ms_index"], st["ms_lz77"] - st["ms_walk"], st["ms_entropy"], st["ms_total"]))
    same = len({o for o in outs.values()}) == 1 and None not in outs.values()
    print("%s: %d bytes, quality %d, lgwin %d, %d rounds; outputs identical across builds and rounds: %s" % (
        name, len(d), q, w, a.rounds, same), flush=True)
    for so in a.libs:
        cols = []
        for i, label in enumerate(("walk", "index", "lz77-walk", "entropy", "total")):
            v = [r[i] for r in res[so]]
            cols.append("%s median %7.2f ms (%.2f-%.2f)" % (label, statistics.median(v), min(v), max(v)))
        print("  %-40s %s  MB/s %.0f" % (so, "  ".join(cols), len(d) / 1e3 / statistics.median([r[4] for r in res[so]])),
              flush=True)
