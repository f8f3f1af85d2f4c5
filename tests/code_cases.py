"""Histograms built to reach the rarely taken branches of one prefix code's construction (E4: the count smoothing of
BrotliOptimizeHuffmanCountsForRle, the depth-limited Huffman tree, the simple codes, the code-length run writers and the
code-length code's header), in every alphabet of a metablock of quality 4+: literal (256), command (704), distance (64).
Deterministic: every family is seeded.

cases() returns (label, histogram) pairs; expect(family) names the oracle edge counters (oracle/brotli_oracle.c EDGE_FIELDS)
that building the family's codes with oracle_build_code must reach, with the least value each must reach.

Count bound: a metablock holds at most 1 << 24 bytes (setup_hasher's max_mb; MLEN has 24 bits), so no count and no sum of
counts of one histogram exceeds that.  The smoothing's 32-bit `256 * (c0 + c1 + c2)` cannot wrap then: a histogram reaches
it only with 16 or more nonzero counts, so c0 + c1 + c2 <= (1 << 24) - 13.  The large_counts family goes up to that bound."""
import functools

import numpy as np

ALPHABETS = (256, 704, 64)
MAX_TOTAL = 1 << 24
FIB = [1, 2]
while len(FIB) < 40:
    FIB.append(FIB[-1] + FIB[-2])


def _h(A, pairs):
    """A histogram of A counts from {symbol: count}."""
    h = np.zeros(A, np.uint32)
    for s, c in pairs.items():
        h[s] = c
    return h


def _spread(A, counts, rng, lo=0, hi=None):
    """counts placed on distinct random symbols of [lo, hi)."""
    hi = A if hi is None else hi
    syms = rng.choice(np.arange(lo, hi), len(counts), replace=False)
    return _h(A, dict(zip(syms.tolist(), counts)))


# ------------------------------------------------------------------------------------------------------- few_symbols
def few_symbols():
    """No symbol (a metablock without explicit distances has an all-zero distance histogram), one symbol at the first,
    a middle and the last index, 2..4 symbols with equal and skewed counts at the alphabet's ends, and the two shapes of
    four symbols: {1, 2, 3, 3} depths (tree-select 1) and {2, 2, 2, 2} (tree-select 0), with depth ties in both orders of
    the symbols, which decide the order the simple code lists them in."""
    out = []
    for A in ALPHABETS:
        out.append(("zero", np.zeros(A, np.uint32)))
        for s in (0, A // 2 + 3, A - 1):
            out.append(("one@%d" % s, _h(A, {s: 7 + s})))
        for k, syms in ((2, (0, A - 1)), (3, (0, 1, A - 1)), (4, (0, 1, A - 2, A - 1))):
            out.append(("k%d_equal" % k, _h(A, {s: 5 for s in syms})))
            out.append(("k%d_skewed" % k, _h(A, {s: 1 + 1000 * (j == k - 1) for j, s in enumerate(syms)})))
            out.append(("k%d_skewed_first" % k, _h(A, {s: 1 + 1000 * (j == 0) for j, s in enumerate(syms)})))
        # {1, 2, 3, 3}: counts 8, 4, 2, 2 in every order over four symbols (which one gets depth 1, which ties are 3 deep)
        syms = (0, 5, A // 2, A - 1)
        for perm in ((8, 4, 2, 2), (2, 2, 4, 8), (2, 8, 2, 4), (4, 2, 8, 2), (3, 1, 1, 9)):
            out.append(("k4_select1_%s" % "_".join(map(str, perm)), _h(A, dict(zip(syms, perm)))))
        for perm in ((2, 2, 2, 2), (3, 2, 2, 3), (5, 4, 4, 5), (1, 1, 1, 1)):
            out.append(("k4_select0_%s" % "_".join(map(str, perm)), _h(A, dict(zip(syms, perm)))))
        # three symbols: which of the two 2-deep ones is listed first
        for perm in ((1, 1, 5), (5, 1, 1), (1, 5, 1), (2, 2, 2)):
            out.append(("k3_ties_%s" % "_".join(map(str, perm)), _h(A, dict(zip((1, A // 3, A - 2), perm)))))
    return out


# ----------------------------------------------------------------------------------------------------------- smoothing
def smoothing():
    """The exits of the smoothing at 5, 15 | 16, 27 | 28 nonzero counts; one-symbol holes next to a count below 4 with
    fewer than 6 zeros (filled) and with 6 or more (left); runs of 5+ zeros and 7+ equal counts (good_for_rle); strides
    of close counts (averaged)."""
    out = []
    for A in ALPHABETS:
        rng = np.random.default_rng(100 + A)
        for nz in (5, 15, 16, 27, 28):
            out.append(("nz%d" % nz, _spread(A, rng.integers(40, 400, nz).tolist(), rng)))
        # 15 | 16 nonzero counts with one hole beside a count of 2: left below 16 nonzero counts, filled from 16 on
        for nz in (15, 16):
            c = rng.integers(40, 400, nz + 1)
            c[5], c[7] = 2, 0
            out.append(("nz%d_hole" % nz, _h(A, {s: int(v) for s, v in enumerate(c)})))
        # 24 symbols 0..23 with 4 single holes beside counts of 2: zeros < 6, filled
        for zeros, tag in ((4, "holes_filled"), (6, "holes_kept"), (9, "holes_kept9")):
            n = 24 + zeros
            hole = set(rng.choice(np.arange(2, n - 2, 3), zeros, replace=False).tolist())
            h = np.zeros(A, np.uint32)
            for s in range(min(n, A)):
                if s not in hole:
                    h[s] = 2 if (s - 1 in hole or s + 1 in hole) else int(rng.integers(50, 300))
            out.append((tag, h))
        # runs of 5 zeros and of 7 equal counts among 40 nonzero ones
        h = np.zeros(A, np.uint32)
        body = [int(c) for c in rng.integers(100, 900, 12)] + [0] * 5 + [333] * 7 + [int(c) for c in rng.integers(100, 900, 10)] \
            + [0] * 6 + [77] * 9 + [int(c) for c in rng.integers(1, 900, 8)]
        h[:len(body)] = body[:A]
        out.append(("good_runs", h))
        # strides: slowly varying counts (averaged within +-1240 / 256 of the running mean) with jumps between them
        h = np.zeros(A, np.uint32)
        lvl = 200
        for s in range(min(A, 120)):
            if s % 17 == 0:
                lvl = int(rng.integers(20, 2000))
            h[s] = lvl + int(rng.integers(-3, 4))
        out.append(("strides", h))
        # strides of small counts with zeros inside (a sum of 0 over 3+ counts keeps them 0)
        h = np.zeros(A, np.uint32)
        for s in range(min(A, 60)):
            h[s] = 0 if s % 11 in (3, 4, 5) else int(rng.integers(1, 4))
        out.append(("strides_small", h))
    return out


# -------------------------------------------------------------------------------------------------------- depth_limit
def _dyadic(A, depths, scale_bits, rng):
    """A histogram whose Huffman depths are `depths` (a complete prefix code): counts 2 ** (scale_bits - depth), on
    symbols 0..len-1 in an order without two equal neighbours where possible."""
    d = sorted(depths)
    order = []
    while d:                          # deal the depths round-robin so that equal ones do not sit side by side
        vals = sorted(set(d), key=lambda v: -d.count(v))
        for v in vals:
            order.append(v)
            d.remove(v)
    return np.asarray([1 << (scale_bits - v) for v in order] + [0] * (A - len(order)), np.uint32)


def depth_limit():
    """Fibonacci counts (one to several count_limit doublings before the tree fits 15 levels), powers of two (many), and
    trees whose code-length code is deeper than 5 levels (retry_cl): the number of symbols per depth grows like the
    Fibonacci numbers, so the histogram of code lengths is Fibonacci-shaped."""
    out = []
    for A in ALPHABETS:
        rng = np.random.default_rng(200 + A)
        for k in (17, 20, 24, 28):
            out.append(("fib%d" % k, _spread(A, FIB[:k], rng)))
        out.append(("fib24_dense", _h(A, {s: FIB[s] for s in range(24)})))
        out.append(("pow2_24", _spread(A, [1 << j for j in range(24)], rng)))
        out.append(("pow2_20_dense", _h(A, {s: 1 << (19 - s) for s in range(20)})))
        out.append(("pow2_pairs", _spread(A, [1 << (j // 2) for j in range(40)], rng)))
    # symbols per depth 1, 1, 2, 3, 5, 8, 13, 21, 34 from depth 7 on, the rest of the Kraft sum in depths 3..6
    per = {3: 1, 4: 2, 5: 3, 6: 5}
    for j, d in enumerate(range(7, 16)):
        per[d] = FIB[j]
    kraft = sum(n * 2.0 ** -d for d, n in per.items())
    per[15] += int(round((1 - kraft) * 2 ** 15))
    depths = [d for d, n in per.items() for _ in range(n)]
    for A in (256, 704):
        if len(depths) <= A:
            out.append(("cl_deep", _dyadic(A, depths, 20, None)))
    return out


# -------------------------------------------------------------------------------------------------------------- ties
def ties():
    """All counts equal (every alphabet; uniform 256 is 8 levels deep everywhere, which the writer stores as one
    code-length symbol, 16, so the code-length code has one symbol), staircases of long equal runs, and leaf counts
    equal to the sums of merged nodes (the merge takes the leaf first)."""
    out = []
    for A in ALPHABETS:
        for v in (1, 7, 20000):
            out.append(("flat%d" % v, np.full(A, v, np.uint32)))
        st = np.zeros(A, np.uint32)
        for s in range(A):
            st[s] = 1 + (s // 40) * 3
        out.append(("staircase", st))
        st2 = np.asarray([1 << min(s // 32, 15) for s in range(A)], np.uint32)
        out.append(("staircase_pow2", st2))
        for j, base in enumerate(((1, 1, 2, 4, 8, 16, 32, 64), (2, 2, 4, 4, 8, 8, 16, 16), (3, 3, 6, 6, 12, 12, 24, 24, 48),
                                  (1, 1, 2, 2, 4, 4, 8, 8, 16, 16, 32, 32, 64, 64, 128, 128, 256, 256))):
            out.append(("leaf_eq_sum%d" % j, _h(A, {s * (A // len(base)): c for s, c in enumerate(base)})))
        rng = np.random.default_rng(300 + A)
        # counts drawn from the sums of pairs of smaller ones
        vals = [1, 1]
        while len(vals) < min(A, 200):
            vals.append(int(vals[rng.integers(0, len(vals))] + vals[rng.integers(0, len(vals))]) % 5000 + 1)
        out.append(("pair_sums", _spread(A, vals, rng)))
    # 288 equal counts within 704 and 300 in 256: the rank sort's passes of 256 nodes hold ties across them
    out.append(("flat_cross_pass", _h(704, {s: 9 for s in range(0, 704, 2)})))
    out.append(("two_levels_cross_pass", np.asarray([5 if s % 3 else 10 for s in range(704)], np.uint32)))
    return out


# ------------------------------------------------------------------------------------------------------ rle_writer
def rle_writer():
    """Code-length runs: exactly 7 equal nonzero depths behind a different one (reps7) and 11 zeros (reps11); zero and
    nonzero runs long enough to chain several 17s and 16s; trailing zeros; code-length codes without lengths 1, 2 (skip 2)
    and 1, 2, 3 (skip 3); and trimmed code-length codes."""
    out = []
    for A in ALPHABETS:
        rng = np.random.default_rng(400 + A)
        # 8 equal counts (one depth: one symbol + 7 repeats), 11 zeros, 8 more, and a varied tail that keeps the RLE on
        h = np.zeros(A, np.uint32)
        h[0:8] = 300
        h[19:27] = 300
        h[27:40] = rng.integers(1, 3000, 13)
        out.append(("reps7_11", h))
        # long runs: 16 * k nonzero equal and 100+ zeros
        if A >= 256:
            h = np.zeros(A, np.uint32)
            h[0:150] = 50
            h[150:170] = rng.integers(1, 9000, 20)
            h[A - 30:A] = 50
            out.append(("long_runs", h))
        h = np.zeros(A, np.uint32)
        h[:A // 2] = rng.integers(1, 1000, A // 2)
        out.append(("trailing_zeros", h))
        # 16 equal counts apart: depth 4 only (code lengths 0 and 4: skip 3)
        out.append(("skip3", _h(A, {s: 10 for s in range(0, min(A, 64), max(1, min(A, 64) // 16))})))
        # depths 3 and 4 (no 1 or 2): skip 2
        out.append(("skip2", _h(A, {s * 3: (20 if s < 4 else 10) for s in range(12)})))
        # 40 nonzero counts without runs: all lengths 3..8 present, the code-length code trimmed behind them
        out.append(("trim", _spread(A, [int(c) for c in rng.zipf(1.3, 40) % 60000 + 1], rng)))
    return out


# ------------------------------------------------------------------------------------------------------ large_counts
def large_counts():
    """Counts up to what one metablock holds (1 << 24 in total): the three first counts near a third of the bound each,
    one count near the bound, and the smoothing's strides over counts of millions."""
    out = []
    for A in ALPHABETS:
        rest = 28
        big = (MAX_TOTAL - rest) // 3
        h = np.zeros(A, np.uint32)
        h[0:3] = big
        h[3:3 + rest] = 1
        out.append(("c012_bound", h))
        h = np.zeros(A, np.uint32)
        h[:30] = 1
        h[A - 1] = MAX_TOTAL - 30
        out.append(("one_huge", h))
        rng = np.random.default_rng(500 + A)
        h = (rng.random(A) * 65000 + 1).astype(np.uint32)
        h[: A // 2] += np.uint32(MAX_TOTAL // A)
        h = np.minimum(h, (MAX_TOTAL - 1) // A).astype(np.uint32)
        out.append(("millions", h))
    return out


# ------------------------------------------------------------------------------------------------------------ random
def _random_histo(rng, A):
    shape = rng.integers(0, 4)
    used = int(rng.integers(2, A + 1))
    scale = float(10 ** rng.uniform(0, 5))
    if shape == 0:       # Zipf
        v = scale / (np.arange(1, used + 1) ** rng.uniform(0.6, 2.0))
    elif shape == 1:     # geometric
        v = scale * rng.uniform(0.5, 0.99) ** np.arange(used)
    elif shape == 2:     # sparse
        v = scale * rng.random(used) * (rng.random(used) < rng.uniform(0.05, 0.4))
    else:                # flat with noise
        v = scale * (1 + 0.1 * rng.random(used))
    v = np.floor(v).astype(np.int64)
    h = np.zeros(A, np.int64)
    pos = rng.permutation(A)[:used] if rng.random() < 0.5 else np.arange(used)
    h[pos] = v
    if rng.random() < 0.5:          # zero runs
        for _ in range(int(rng.integers(1, 6))):
            a = int(rng.integers(0, A))
            h[a:a + int(rng.integers(3, 40))] = 0
    if h.sum() > MAX_TOTAL:
        h = h * MAX_TOTAL // (h.sum() + 1)
    return h.astype(np.uint32)


def random_histograms(count=3000, seed=600):
    """Zipf, geometric, sparse and flat histograms with zero runs, over every alphabet."""
    rng = np.random.default_rng(seed)
    return [("%d" % i, _random_histo(rng, ALPHABETS[i % 3])) for i in range(count)]


FAMILIES = {
    "few_symbols": (few_symbols, {"simple_nsym1": 12, "simple_nsym2": 6, "simple_nsym3": 15, "simple_nsym4": 27,
                                  "simple_select0": 12, "simple_select1": 15}),
    "smoothing": (smoothing, {"rle_lt16": 6, "rle_lt28": 6, "rle_full": 9, "rle_holes": 1, "rle_good": 3, "rle_stride": 3}),
    "depth_limit": (depth_limit, {"retry_lit": 1, "retry_cmd": 1, "retry_dist": 1, "retry_cl": 1}),
    "ties": (ties, {"cl_single": 1, "rle_use_nz": 3}),
    "rle_writer": (rle_writer, {"reps7": 3, "reps11": 3, "rle_use_z": 3, "cl_skip2": 1, "cl_skip3": 1, "cl_trim": 3}),
    "large_counts": (large_counts, {"rle_full": 3, "rle_stride": 1}),
    "random": (random_histograms, {"retry_lit": 1, "rle_full": 100, "rle_use_nz": 10, "rle_use_z": 10}),
}


@functools.lru_cache(maxsize=None)
def _all():
    res = []
    for fam, (make, _) in FAMILIES.items():
        for label, h in make():
            assert len(h) in ALPHABETS and int(h.sum()) <= MAX_TOTAL, (fam, label)
            res.append(("%s/%s/%d" % (fam, label, len(h)), fam, np.ascontiguousarray(h, np.uint32)))
    labels = [r[0] for r in res]
    assert len(set(labels)) == len(labels), "case labels must be unique"
    return tuple(res)


def cases(family=None):
    """(label, histogram) of every case, or of one family."""
    return [(label, h) for label, fam, h in _all() if family is None or fam == family]


def expect(family):
    """{edge counter: least value} that building the family's codes must reach."""
    return FAMILIES[family][1]


def padding(A, count, seed):
    """count more histograms of alphabet A (random shapes) that fill synthetic metablocks."""
    rng = np.random.default_rng(seed)
    return [("pad%d/%d/%d" % (seed, i, A), _random_histo(rng, A)) for i in range(count)]
