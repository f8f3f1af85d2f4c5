"""Inputs built to reach the entropy stage's rarely taken branches (prefix-code depth limits, the block-type cap, simple
prefix codes, the count smoothing and code-length run writers, the longest insert / block-length / distance codes), which
ordinary text, web and binary data reach only by accident.  Deterministic: every family is seeded.

cases() returns (label, data, quality, lgwin) tuples; expect(label) names the oracle edge counters
(oracle/brotli_oracle.c EDGE_FIELDS) the case was built for, with the least value each must reach."""
import functools

import numpy as np

FIB = [1, 1]
while len(FIB) < 30:
    FIB.append(FIB[-1] + FIB[-2])


def _shuffled(symbols, counts, rng):
    """The multiset {symbols[i] x counts[i]} in random order."""
    a = np.repeat(np.asarray(symbols, np.uint8), counts)
    rng.shuffle(a)
    return a.tobytes()


def _pairs_once(n, values):
    """n bytes over `values` (at least 150 of them) in which no 2-byte string occurs twice: an Eulerian walk through all
    pairs (a de Bruijn sequence of order 2, shuffled per symbol).  LZ77 finds nothing in it, not even the 2- and 3-byte
    matches at cached distances, and at log2(len(values)) < 8 bits a byte it is still worth compressing."""
    k = len(values)
    assert n <= k * k
    rng = np.random.default_rng(k)
    succ = [list(rng.permutation(k)) for _ in range(k)]
    out, v = [], 0
    while len(out) < n:          # a greedy walk (each pair used once) that only gets stuck near the end: 25418 bytes for k = 160
        out.append(v)
        if not succ[v]:
            break
        v = int(succ[v].pop())
    assert len(out) == n, len(out)
    return np.asarray(values, np.uint8)[out].tobytes()


# --------------------------------------------------------------------------------------------------- fib_literals
def fib_literals():
    """Literal counts on a Fibonacci sequence over 20..24 byte values, shuffled: the literal tree is deeper than 15
    levels until count_limit has doubled a few times (BrotliCreateHuffmanTree retries), and the code-length code of such
    trees is deep as well."""
    out = []
    # every other byte is flat noise (0..63), which keeps LZ77 from matching the skewed bytes (64..127) away; all
    # bytes are ASCII, so there is one literal context and the tree sees both halves
    for k, q, w in ((24, 2, 22), (24, 3, 16), (22, 4, 22)):
        rng = np.random.default_rng(1000 + k * 10 + q)
        syms = rng.choice(np.arange(64, 128), k, replace=False)
        skew = np.frombuffer(_shuffled(syms, FIB[:k], rng), np.uint8)
        flat = rng.integers(0, 64, skew.size, dtype=np.uint8)
        d = np.stack([flat, skew], 1).ravel().tobytes()
        out.append(("fib_literals/k%d" % k, d, q, w, {"retry_fast" if q == 2 else "retry_lit": 1}))
    # the skew only in the literals behind a continuation byte: every other byte is 0x80..0xBF (uniform), so context
    # modelling splits the literals into a flat and a Fibonacci-shaped histogram and the latter still retries
    for q, w in ((7, 22), (9, 24), (5, 18)):
        rng = np.random.default_rng(1100 + q)
        k = 24
        syms = rng.choice(np.arange(32, 128), k, replace=False)
        skew = np.frombuffer(_shuffled(syms, FIB[:k], rng), np.uint8)
        lead = rng.integers(0x80, 0xC0, skew.size, dtype=np.uint8)
        d = np.stack([lead, skew], 1).ravel().tobytes()
        out.append(("fib_literals/one_context", d, q, w, {"retry_lit": 1, "ctx_nc2": 1}))
    return out


# ----------------------------------------------------------------------------------------- fib_distances / commands
def _copies(rng, plan, base_len=1 << 17):
    """Incompressible noise of base_len bytes, then for each (insert, copy, distance) of plan: `insert` noise bytes and a
    copy of `copy` bytes from `distance` back.  Noise never matches, so the parser finds exactly the planted copies."""
    out = bytearray(rng.integers(0, 256, base_len, dtype=np.uint8).tobytes())
    noise = rng.integers(0, 256, sum(p[0] for p in plan) + 16, dtype=np.uint8).tobytes()
    o = 0
    for ins, cp, dist in plan:
        out += noise[o:o + ins]; o += ins
        s = len(out) - dist
        for j in range(cp):
            out.append(out[s + j])
    out += noise[o:o + 8]
    return bytes(out)


def _dist_in_code(code, rng):
    """A distance whose prefix code (NPOSTFIX 0, NDIRECT 0) is `code` >= 16 (prefix.h:23)."""
    nbits = (code - 16) // 2 + 1
    prefix = (code - 16) & 1
    lo = ((2 + prefix) << nbits) - 3               # code(dcode) for dcode = distance + 15: 4 + dcode - 16 = distance + 3
    return int(rng.integers(lo, lo + (1 << nbits)))


def _fresh_distances(codes, rng):
    """One distance per entry of codes, never within 3 of the last four: no copy is coded through the distance cache
    (which would add symbols to the distance histogram)."""
    res = []
    for code in codes:
        while True:
            d = _dist_in_code(int(code), rng)
            if all(abs(d - r) > 3 for r in res[-4:]):
                break
        res.append(d)
    return res


def _weighted(weights, rng):
    """Indices i, weights[i] times each, shuffled."""
    a = np.repeat(np.arange(len(weights)), weights)
    rng.shuffle(a)
    return a


def fib_distances():
    """Copies whose distance codes are Fibonacci-weighted (x4, so that the count smoothing keeps them apart) over 20
    codes: the distance tree retries."""
    out = []
    for q, w in ((4, 18),):
        rng = np.random.default_rng(2000 + q)
        codes = rng.permutation(np.arange(26, 46))        # distances 61 .. 128 Ki (inside the noise), 64+ per code
        which = codes[_weighted([4 * f for f in FIB[:20]], rng)]
        dists = _fresh_distances(which, rng)
        plan = [(int(rng.integers(1, 3)), int(rng.integers(5, 9)), d) for d in dists]
        out.append(("fib_distances", _copies(rng, plan), q, w, {"retry_dist": 1}))
    return out


def fib_commands():
    """Copies whose insert-and-copy length codes are Fibonacci-weighted (x4) over 20 codes: the command tree retries."""
    out = []
    pairs = [(i, c) for i in (1, 2, 3, 4, 5, 6, 8, 10) for c in (5, 6, 7, 8, 9, 10, 12, 14)]   # distinct command codes
    for q, w in ((4, 22),):
        rng = np.random.default_rng(3000 + q)
        pick = [pairs[j] for j in rng.choice(len(pairs), 20, replace=False)]
        which = _weighted([4 * f for f in FIB[:20]], rng)
        dists = _fresh_distances(rng.integers(30, 36, which.size), rng)      # 1 .. 16 Ki back: never evicted
        plan = [(pick[j][0], pick[j][1], d) for j, d in zip(which, dists)]
        out.append(("fib_commands", _copies(rng, plan), q, w, {"retry_cmd": 1}))
    return out


# ---------------------------------------------------------------------------------------------------- many_dialects
def _dialect(rng, n, pool):
    """n bytes from a random alphabet of 12..24 values of `pool`, with its own geometric skew."""
    k = int(rng.integers(12, 25))
    syms = rng.choice(pool, k, replace=False)
    p = 0.8 ** np.arange(k)
    return rng.choice(syms, n, p=p / p.sum()).astype(np.uint8).tobytes()


def many_dialects():
    """Segments of 1..4 KiB, each from its own alphabet and skew, all in one metablock (lgwin 24, quality 5..9): the
    greedy literal splitter opens a new block type for nearly every segment until it reaches 256 / nc types, so the
    metablock stores 256 literal trees.  One input per context count the encoder can choose; and two dialects in
    turn, which sends the splitter back to the type before last."""
    out = []
    ascii_ = np.arange(0, 128)
    for label, q, segs, pool, want in (
            ("nc1", 5, 330, ascii_, {"lit_cap_nc1": 1, "max_lit_trees": 256}),
            ("nc1", 9, 330, ascii_, {"lit_cap_nc1": 1, "max_lit_trees": 256}),
            ("nc2", 6, 200, "cont", {"lit_cap_nc2": 1, "max_lit_trees": 256}),
            ("nc3", 8, 150, "utf8", {"lit_cap_nc3": 1, "max_lit_trees": 255})):
        rng = np.random.default_rng(4000 + q + segs)
        parts = []
        for _ in range(segs):
            n = int(rng.integers(1024, 4097))
            if isinstance(pool, str) and pool == "cont":
                # a continuation byte (0x80..0xBF) is always followed by ASCII, ASCII by a continuation byte 6 times in
                # 10: the class of a literal depends on whether the byte before it is a continuation byte (nc 2)
                a = np.frombuffer(_dialect(rng, n, np.arange(0x20, 0x80)), np.uint8)
                c = np.frombuffer(_dialect(rng, n, np.arange(0x80, 0xC0)), np.uint8)
                seq, prev_cont = [], False
                for j, u in enumerate(rng.random(n)):
                    prev_cont = not prev_cont and u < 0.6
                    seq.append(c[j] if prev_cont else a[j])
                parts.append(np.asarray(seq, np.uint8).tobytes())
            elif not isinstance(pool, str):
                parts.append(_dialect(rng, n, pool))
            else:
                # ASCII and two-byte UTF-8 sequences: the literal's class depends on the byte before it
                a = np.frombuffer(_dialect(rng, n // 2, np.arange(0x20, 0x80)), np.uint8)
                lead = np.frombuffer(_dialect(rng, n // 2, np.arange(0xC2, 0xE0)), np.uint8)
                cont = np.frombuffer(_dialect(rng, n // 2, np.arange(0x80, 0xC0)), np.uint8)
                pick = rng.random(n // 2) < (0.5 if label != "nc3" else 0.8)
                parts.append(np.where(pick[:, None], np.stack([lead, cont], 1), np.stack([a, a], 1)).ravel().tobytes())
        out.append(("many_dialects/%s" % label, b"".join(parts), q, 24, want))
    rng = np.random.default_rng(4100)
    a, b = _dialect(rng, 300000, ascii_), _dialect(rng, 300000, np.arange(128, 256))
    d = b"".join((a if i % 2 == 0 else b)[i * 1500:(i + 1) * 1500] for i in range(200))
    for q in (5, 6, 4):
        out.append(("many_dialects/alternating", d, q, 24, {"split_back": 1}))
    return out


# ---------------------------------------------------------------------------------------------------- tiny_alphabets
def tiny_alphabets():
    """One to four distinct literals: simple prefix codes (NSYM 1..4; four even counts take the 2, 2, 2, 2 shape).  A
    run of one byte is one command with one distance: one-symbol codes everywhere.  (Skewed four-symbol literals do not
    keep their skew through LZ77; the 1, 2, 3, 3 shape is met in the many_dialects inputs.)"""
    out = []
    for q, w in ((2, 22), (3, 18), (4, 22), (5, 22), (9, 24)):
        rng = np.random.default_rng(5000 + q)
        out.append(("tiny_alphabets/run", b"\x41" * 5000, q, w, {"simple_nsym1": 1 if q == 2 else 3}))
        for k in (2, 3):
            syms = rng.choice(256, k, replace=False)
            out.append(("tiny_alphabets/k%d" % k, rng.choice(syms, 3000).astype(np.uint8).tobytes(), q, w,
                        {"simple_nsym%d" % k: 1}))
        syms = rng.choice(256, 4, replace=False)
        out.append(("tiny_alphabets/k4_flat", rng.choice(syms, 3000).astype(np.uint8).tobytes(), q, w,
                    {"simple_select0": 1}))
    return out


# ------------------------------------------------------------------------------------------------------- rle_shapes
def rle_shapes():
    """Literal histograms at the exits of BrotliOptimizeHuffmanCountsForRle (5, 15 | 16, 27 | 28, 29 nonzero symbols),
    with one-symbol holes next to counts below 4 (filled when fewer than 6 zeros), and code-length runs of exactly 7
    non-zero depths behind a different one and 11 zeros (the reps == 7 / reps == 11 cases)."""
    out = []
    exits = {5: "rle_lt28", 15: "rle_lt16", 16: "rle_lt28", 27: "rle_lt28", 28: "rle_full", 29: "rle_full"}
    for q, w in ((5, 22), (9, 24), (3, 22), (4, 17)):
        rng = np.random.default_rng(6000 + q)
        for nz in (5, 15, 16, 27, 28, 29) if q != 3 else ():
            counts = rng.integers(40, 400, nz)
            syms = rng.choice(np.arange(0x20, 0x80), nz, replace=False)
            want = {exits[nz]: 1}
            if nz == 5:
                want = {"rle_lt16": 1}      # below 16 nonzero counts the first exit is taken
            out.append(("rle_shapes/nz%d" % nz, _shuffled(syms, counts, rng), q, w, want))
        # dense symbols 0..29 with three holes (zeros < 6) beside counts of 1..3: the holes are filled
        syms = [s for s in range(30) if s not in (7, 15, 22)]
        counts = [2 if s in (6, 8, 14, 16, 21, 23) else int(rng.integers(200, 400)) for s in syms]
        if q != 3:
            out.append(("rle_shapes/holes", _shuffled(syms, counts, rng), q, w, {"rle_holes": 1}))
        # 8 equal counts from symbol 0 (one depth, written as one + 7 repeats), 11 zeros, 8 more
        syms = list(range(8)) + list(range(19, 27))
        out.append(("rle_shapes/reps7_11", _shuffled(syms, [300] * 16, rng), q, w, {"reps7": 1, "reps11": 1}))
    return out


# -------------------------------------------------------------------------------------------------------- long_codes
def long_codes():
    """The longest codes of one metablock: inserts of 6210+ and 22594+ literals in one command (match-free but
    compressible bytes, so the metablock stays compressed), a literal block of more than 16625 symbols between type
    switches (the 24-extra-bit block-length code), and a copy at exactly max_backward = (1 << lgwin) - 16."""
    out = []
    tail = bytes(range(0xE0, 0xFF)) * 3           # (a copy behind the literals)
    for n, code_base in ((24000, 22594), (10000, 6210)):
        ins = _pairs_once(n, list(range(160))) + tail
        for q, w in ((5, 22), (9, 24), (2, 22), (3, 18), (4, 22)):
            out.append(("long_codes/insert%d" % n, ins, q, w, {"max_insert": code_base}))
    # uniform bytes of two disjoint halves in turn (7 bits a byte, next to no matches): literal blocks of 20000 of
    # one type between switches
    rng = np.random.default_rng(7100)
    lo, hi = (rng.integers(a, a + 128, 48000, dtype=np.uint8).tobytes() for a in (0, 128))
    blocks = lo[:20000] + hi[:4000] + lo[20000:42000] + hi[4000:8000]
    for q, w in ((5, 22), (9, 24), (4, 22)):
        out.append(("long_codes/block_len", blocks, q, w, {"max_block_len": 16625}))
    # a unique 64-byte pattern, zeros up to exactly max_backward, the pattern again: its only match is max_backward back
    rng = np.random.default_rng(7000)
    pat = rng.integers(1, 256, 64, dtype=np.uint8).tobytes()
    for w, qs in ((10, (2, 3, 4)), (17, (2, 4, 5, 9)), (18, (3, 6, 8))):
        mb = (1 << w) - 16
        d = bytes(100) + pat + bytes(mb - len(pat)) + pat + bytes(100)
        for q in qs:
            out.append(("long_codes/distance_w%d" % w, d, q, w, {"max_distance": mb}))
    return out


FAMILIES = [fib_literals, fib_distances, fib_commands, many_dialects, tiny_alphabets, rle_shapes, long_codes]


@functools.lru_cache(maxsize=None)
def _all():
    res = []
    for fam in FAMILIES:
        for label, d, q, w, want in fam():
            res.append(("%s-q%d-w%d" % (label, q, w), d, q, w, want))
    labels = [r[0] for r in res]
    assert len(set(labels)) == len(labels), "case labels must be unique"
    return tuple(res)


def cases():
    """(label, data, quality, lgwin) for every case."""
    return [(label, d, q, w) for label, d, q, w, _ in _all()]


def expect(label):
    """{edge counter: least value} that the case `label` was built to reach."""
    return next(want for lab, _, _, _, want in _all() if lab == label)
