"""Seeded inputs for the literal context decision (E2) and the greedy block splitter (E3) of the entropy stage, run on
their own through br_debug_split / sim_debug_split / oracle_split (tests/test_entropy_split.py).

A case is a job: input bytes, a command list that covers them in order, and metablocks over the commands.  Commands are
tuples (insert, copy, dcode) -- copy 0 makes an insert-only command -- that the test turns into the encoder's 16-byte
commands with the oracle's own InitCommand (oracle_make_cmd).  `expect` names the oracle edge counters
(brotli_oracle.c EDGE_FIELDS) the case was built to reach.

The exact ties rest on one identity.  Two blocks of S symbols each (S a power of two) whose histograms share symbols
with equal counts, shared mass m, cost together 2S - 2m bits more than apart (BitsEntropy: the c log c terms of a
shared symbol cancel against 2c log 2c, leaving 2c).  With every count and every sum a power of two, each log2 the
splitter looks up is an integer, so that difference is exact in double precision, and `diff` can be put exactly on a
threshold (2S - 2m = thr) or exactly 20 bits apart between the last two types."""
import numpy as np

CATS = ("literal", "command", "distance")
MIN_BLOCK = (512, 1024, 512)
THR = (400, 500, 100)


class Case:
    def __init__(self, label, quality=5, size_hint=None, disable_ctx=1, expect=None, seed=0):
        self.label, self.quality, self.disable_ctx = label, quality, disable_ctx
        self.size_hint = size_hint
        self.expect = dict(expect or {})
        self.data, self.cmds, self.mbs = bytearray(), [], []
        self.base = 0
        self.rng = np.random.default_rng(seed)

    def stream(self):
        """The metablocks after this belong to a new stream of a batch: their literal contexts start from zeros."""
        self.base = len(self.data)

    def mb(self, parts, compress=1):
        """One metablock of (literal bytes, copy, distance code) parts; copy is a length (the copied bytes are seeded
        noise) or the copied bytes themselves."""
        start, c0 = len(self.data), len(self.cmds)
        for lits, copy, dcode in parts:
            self.data += bytes(lits)
            if isinstance(copy, (bytes, bytearray)):
                self.data += copy
                copy = len(copy)
            elif copy:
                self.data += self.rng.integers(0, 256, copy, dtype=np.uint8).tobytes()
            self.cmds.append((len(lits), copy, dcode))
        self.mbs.append([start, len(self.data), c0, len(self.cmds) - c0, 0, compress, self.base])
        return self

    def done(self):
        self.mbs[-1][4] = 1
        if self.size_hint is None:
            self.size_hint = len(self.data)
        return self


# ---- symbol streams of one category
# commands: insert i (0..5) and copy 2 + c (c in 0..7) with the last distance (code 0) have the insert and copy codes
# (i, c), and CombineLengthCodes maps distinct (insert code < 8, copy code < 16) pairs to distinct command symbols; the
# insert's literals are 'a'.
CMD_SYMS = [(i, 2 + c) for i in range(6) for c in range(8)]


def dist_code(sym):
    """The distance code whose symbol (NPOSTFIX = NDIRECT = 0) is sym, 1..63 (symbol 0 is the last distance, which a
    command with a short copy codes in its command symbol instead)."""
    if sym < 16:
        return sym
    nbits, pre = (sym - 16) // 2 + 1, (sym - 16) % 2
    return ((2 + pre) << nbits) - 4 + 16


def parts_for(cat, syms, rng=None):
    """Command parts that put the symbol stream `syms` into category cat (and whatever follows into the others)."""
    if cat == 0:
        return [(bytes(syms), 0, 0)]
    if cat == 1:
        return [(b"a" * CMD_SYMS[s][0], CMD_SYMS[s][1], 0) for s in syms]
    return [(b"", 4, dist_code(s)) for s in syms]


def windowed(lits, window):
    """Parts of a metablock whose literals are `lits` and whose bytes at every 4 096-byte stride (all that the context
    decision samples, 64 at a time) are the copied bytes `window`: the decision is the window's, the literals are free."""
    assert len(window) == 64
    parts, o = [(b"", window, 0)], 0
    while o < len(lits):
        parts.append((bytes(lits[o:o + 4032]), window if o + 4032 < len(lits) else 0, 0))
        o += 4032
    return parts


# Windows that make the context decision take 2 (quality 5 and 6), 3 (quality 7..9) or 13 (size hint of 1 MiB or more)
# literal contexts; they end in ASCII letters, so that the literal after a window is in context 0 of the 2- and
# 3-context maps when its own previous byte is ASCII too.
def window_utf8():
    return utf8_mix(62, 1) + b"aa"


def window_text():
    return b"the Queen said to Alice, and the March Hare went on: `Take som"[:62].ljust(62, b" ") + b"aa"


def powers(m):
    """m as distinct powers of two, largest first."""
    return [1 << k for k in range(m.bit_length() - 1, -1, -1) if m >> k & 1]


class Syms:
    """Fresh symbol ids of an alphabet, handed out in order."""
    def __init__(self, cat):
        self.next = 1 if cat == 2 else 0
        self.lim = (256, len(CMD_SYMS), 64)[cat]

    def take(self, counts):
        out = {}
        for c in counts:
            assert self.next < self.lim, "alphabet exhausted"
            out[self.next] = c
            self.next += 1
        return out


def block(*hists, rng):
    """A block's symbol stream from {symbol: count} dicts, in a seeded order."""
    s = [k for h in hists for k, c in h.items() for _ in range(c)]
    rng.shuffle(s)
    return s


def exact_diff(a, b):
    """diff of two blocks in exact arithmetic (fractions), for histograms whose counts and sums are powers of two."""
    from fractions import Fraction

    def cost(h):
        tot = sum(h.values())
        lg = lambda v: Fraction(v.bit_length() - 1)
        assert all(c & (c - 1) == 0 for c in h.values()) and tot & (tot - 1) == 0
        r = tot * lg(tot) - sum(c * lg(c) for c in h.values())
        return max(r, Fraction(tot))
    comb = dict(a)
    for k, c in b.items():
        comb[k] = comb.get(k, 0) + c
    return cost(comb) - cost(a) - cost(b)


def tie_split(cat, extra, seed, small=None, nctx=1):
    """Blocks A and B of S symbols sharing mass m with equal counts: diff = 2S - 2m = thr + extra.  extra 0: a tie, the
    block must merge (`>`); extra 2: it must split.  small: counts that replace the shared power of two they sum to;
    counts below 256 that are not powers of two read float-rounded log2 entries, which move diff off the exact tie."""
    S, thr = MIN_BLOCK[cat], THR[cat]
    m = S - (thr + extra) // 2
    ids = Syms(cat)
    sh = powers(m)
    if small:
        sh = [c for c in sh if c != sum(small)] + list(small)
    shared = ids.take(sh)
    A, B = ids.take(powers(S - m)), ids.take(powers(S - m))
    rng = np.random.default_rng(seed)
    syms = block(shared, A, rng=rng) + block(shared, B, rng=rng)
    hist = ({**shared, **A}, {**shared, **B})
    if nctx > 1:
        # ASCII literals behind the window's ASCII ending: every literal is in context 0, the other contexts are
        # empty, so diff (summed over the contexts) is the one-context diff
        c = Case("literal tie split%+d, %d contexts" % (extra, nctx), quality=5 if nctx == 2 else 7, disable_ctx=0,
                 expect={"split_tie": 1, "ctx_nc%d" % nctx: 1} if extra == 0 else {"ctx_nc%d" % nctx: 1}, seed=seed)
        return c.mb(windowed(bytes(0x21 + x for x in syms), window_utf8())).done(), hist
    if not small:
        assert exact_diff(*hist) == thr + extra
        c = Case("%s tie split%+d" % (CATS[cat], extra), expect={"split_tie": 1} if extra == 0 else {}, seed=seed)
    else:
        c = Case("%s tie split%+d, shared counts %s" % (CATS[cat], extra, small), seed=seed)
    return c.mb(parts_for(cat, syms)).done(), hist


# (common, x_A, x_B at the tie) per category: A and B share `common`; C shares common + x_A with A and common + x_B with
# B, with x_A - x_B = 10, so diff[1] = diff[0] - 20, and diff[1] <= thr, so no new type is opened.
BACK = {0: (256, 64, 54), 1: (520, 256, 246), 2: (416, 48, 38)}


def tie_back(cat, extra, seed, xa_parts=None):
    """Blocks A, B (a new type), C: diff[1] == diff[0] - 20 - extra.  extra 0: C must merge into B; 2: C must go back to
    A's type.  xa_parts: the counts of what C shares with A alone, in place of powers of two."""
    S = MIN_BLOCK[cat]
    common, xa, xb = BACK[cat]
    xb -= extra // 2
    ids = Syms(cat)
    com, XA, XB = ids.take(powers(common)), ids.take(xa_parts or powers(xa)), ids.take(powers(xb))
    A = {**com, **XA, **ids.take(powers(S - common - xa))}
    B = {**com, **XB, **ids.take(powers(S - common - xb))}
    C = {**com, **XA, **XB, **ids.take(powers(S - common - xa - xb))}
    rng = np.random.default_rng(seed)
    syms = block(A, rng=rng) + block(B, rng=rng) + block(C, rng=rng)
    if xa_parts:
        assert sum(xa_parts) == xa
        c = Case("%s tie back%+d, C shares %s with A" % (CATS[cat], extra, xa_parts), expect={"split_back": 1}, seed=seed)
        return c.mb(parts_for(cat, syms)).done(), (A, B, C)
    d0, d1 = exact_diff(C, B), exact_diff(C, A)
    assert exact_diff(A, B) > THR[cat] and d1 <= THR[cat] and d1 == d0 - 20 - extra, (d0, d1)
    c = Case("%s tie back%+d" % (CATS[cat], extra), expect={"back_tie": 1} if extra == 0 else {"split_back": 1}, seed=seed)
    return c.mb(parts_for(cat, syms)).done(), (A, B, C)


# Exact ties moved by the float rounding of log2 entries below 256 (br_host.cc, fast_log.c): shared counts 12 and 4 in
# place of 16 lift the split diff of the literal tie by 5.7e-6, so the blocks split; shared counts 5 and 3 in place of 8
# lower diff[1] of the literal go-back tie by 7.2e-7, so the third block goes back.  With every entry in double both
# stay exact ties and merge.
ROUNDING = ((0, (12, 4)), (0, (32, 16, 8, 5, 3)))


def clamp(cat, seed):
    """Two blocks of one symbol each: their costs (0 bits) are raised to their symbol counts, so diff is 0 and the second
    block merges; without the clamp diff would be 2S and it would split."""
    S = MIN_BLOCK[cat]
    ids = Syms(cat)
    a, b = ids.take([S]), ids.take([S])
    c = Case("%s two one-symbol blocks" % CATS[cat], expect={"split_clamp": 1}, seed=seed)
    return c.mb(parts_for(cat, block(a, rng=c.rng) + block(b, rng=c.rng))).done()


def ties():
    out = []
    for cat in range(3):
        for extra in (0, 2):
            out.append(tie_split(cat, extra, 10 + cat)[0])
            out.append(tie_back(cat, extra, 20 + cat)[0])
        out.append(clamp(cat, 30 + cat))
    for nctx in (2, 3):
        for extra in (0, 2):
            out.append(tie_split(0, extra, 40 + nctx, nctx=nctx)[0])
    out.append(tie_split(ROUNDING[0][0], 0, 14, ROUNDING[0][1])[0])
    out.append(tie_back(ROUNDING[1][0], 0, 24, ROUNDING[1][1])[0])
    return out


def block_counts():
    """nsym of 0, 1, min - 1, min, min + 1, exact multiples of the target and a short final block in every category, and
    a run of equal blocks long enough for the target to grow."""
    out = []
    for cat in range(3):
        mn = MIN_BLOCK[cat]
        for n in (1, mn - 1, mn, mn + 1, 2 * mn, 3 * mn + 7, 7 * mn):
            rng = np.random.default_rng(n + cat)
            syms = list(rng.integers(1 if cat == 2 else 0, (256, len(CMD_SYMS), 64)[cat], n))
            exp = {"split_grow": 1} if n == 7 * mn else {"split_pad": 1} if n in (1, mn - 1, 3 * mn + 7) else \
                {"split_pad_empty": 1} if n in (mn, 2 * mn) else {}
            c = Case("%s nsym %d" % (CATS[cat], n), expect=exp, seed=n)
            out.append(c.mb(parts_for(cat, syms)).done())
    # a metablock of copies only (no literals: nsym 0) and of short-copy last-distance commands (no distances)
    out.append(Case("no literals, no distances").mb(parts_for(1, [0] * 50)).done())
    return out


def type_caps():
    """256 literal / command / distance types, then alternation between the last two after the cap."""
    out = []
    for cat, sets, per in ((0, 16, 32), (1, 6, None), (2, 7, None)):
        mn = MIN_BLOCK[cat]
        rng = np.random.default_rng(40 + cat)
        lim = (256, len(CMD_SYMS), 64)[cat]
        lo = 1 if cat == 2 else 0
        width = (lim - lo) // sets
        syms = []
        for b in range(300):
            g = b % sets
            alph = np.arange(lo + g * width, lo + (g + 1) * width)
            syms += list(rng.choice(alph, mn))
        c = Case("%s 300 blocks over %d disjoint alphabets" % (CATS[cat], sets),
                 expect={"lit_cap_nc1": 1} if cat == 0 else {"cmd_cap": 1} if cat == 1 else {"dist_cap": 1}, seed=cat)
        out.append(c.mb(parts_for(cat, syms)).done())
        if cat == 0:   # the literal caps of 2, 3 and 13 contexts: 128, 85 and 19 types
            for nctx, q, hint, win in ((2, 5, None, window_utf8()), (3, 7, None, window_utf8()),
                                       (13, 5, 1 << 20, window_text())):
                c = Case("literal 300 blocks over %d disjoint alphabets, %d contexts" % (sets, nctx), quality=q,
                         size_hint=hint, disable_ctx=0, expect={"lit_cap_nc%d" % nctx: 1}, seed=nctx)
                out.append(c.mb(windowed(bytes(int(x) for x in syms), win)).done())
    return out


def contexts(text):
    """Literal contexts at a stream start, at metablock boundaries, in a second stream of a batch behind nonzero bytes,
    and right after copies, with context modelling on (quality 5..9, size hints on both sides of 1 MiB)."""
    out = []
    for q in (5, 7, 9):
        for hint in ((1 << 20) - 1, 1 << 20):
            c = Case("contexts q%d hint %d" % (q, hint), quality=q, size_hint=hint, disable_ctx=0, seed=q)
            pos = 0
            for k in range(6):
                if k == 3:
                    c.stream()
                parts = []
                for j in range(40):
                    n = 20 + (j * 7) % 50
                    parts.append((text[pos:pos + n], 3 + j % 5, 17 + j))
                    pos += n
                c.mb(parts, compress=0 if k == 4 else 1)
            out.append(c.done())
    return out


def e2_lengths(text):
    """E2 on metablocks of 63/64/65 and 4 159/4 160/4 161 bytes (the stride count (length - 64) / 4096 + 1 changes at
    4 160), quality 5..9, both sides of the 1 MiB size hint, with and without disable_ctx."""
    out = []
    for q in range(5, 10):
        for n in (63, 64, 65, 4159, 4160, 4161):
            for hint in ((1 << 20) - 1, 1 << 20):
                c = Case("E2 q%d length %d hint %d" % (q, n, hint), quality=q, size_hint=hint, disable_ctx=0)
                out.append(c.mb([(text[:n], 0, 0)]).done())
        c = Case("E2 q%d disable_ctx" % q, quality=q, size_hint=1 << 20, disable_ctx=1)
        out.append(c.mb([(text[:5000], 0, 0)]).done())
        c = Case("E2 q%d two-byte UTF-8" % q, quality=q, size_hint=(1 << 20) - 1, disable_ctx=0)
        out.append(c.mb([(utf8_mix(40000, q), 0, 0)]).done())
        # one stride of a constant byte, then two-byte UTF-8 from 4 096 on: 4 159 bytes sample only the first stride,
        # 4 160 the second one too, which changes the choice
        for n in (4159, 4160, 4161):
            c = Case("E2 q%d stride boundary %d" % (q, n), quality=q, size_hint=(1 << 20) - 1, disable_ctx=0)
            out.append(c.mb([((b"a" * 4096 + utf8_mix(200, 1))[:n], 0, 0)]).done())
            # the same on the 13-context side: a constant first stride, text from 4 096 on
            c = Case("E2 q%d 13-context stride boundary %d" % (q, n), quality=q, size_hint=1 << 20, disable_ctx=0)
            out.append(c.mb([((b"a" * 4096 + text[:200])[:n], 0, 0)]).done())
    return out


def utf8_mix(n, seed):
    """ASCII letters and two-byte UTF-8 sequences: the continuation bytes make three literal contexts pay off, which the
    context decision may pick from quality 7 on (below it, ChooseContextMap prices the 3-context model at 10x)."""
    rng = np.random.default_rng(seed)
    lead, cont = rng.integers(0xC2, 0xC6, n), rng.integers(0x80, 0xC0, n)
    asc = rng.integers(0x61, 0x7B, 2 * n)
    pick = rng.random(n) < 0.6
    pairs = np.where(pick[:, None], np.stack([lead, cont], 1), asc.reshape(n, 2))
    return pairs.astype(np.uint8).ravel().tobytes()[:n]


def random_streams(count, seed):
    """Seeded random command streams over a few metablocks each, some raw, context modelling on."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        c = Case("random %d" % k, quality=int(rng.integers(5, 10)), disable_ctx=int(rng.integers(0, 2)), seed=seed + k)
        for m in range(int(rng.integers(1, 5))):
            parts = []
            skew = rng.integers(1, 8)
            for _ in range(int(rng.integers(1, 3000))):
                n = int(rng.geometric(0.2)) - 1
                lits = (rng.integers(0, 256 >> skew, n) * (1 << skew) // 2 + 32).astype(np.uint8).tobytes()
                copy = int(rng.integers(0, 40)) if rng.random() < 0.9 else 0
                parts.append((lits or b"x", copy, int(rng.choice([0, 1, 2, 5, int(rng.integers(16, 5000))]))))
            c.mb(parts, compress=int(rng.random() < 0.85))
        if not any(mb[5] for mb in c.mbs):
            c.mbs[0][5] = 1
        out.append(c.done())
    return out


def large(seed=0):
    """One 16 MiB metablock of one literal: the counts reach 2^24, the last entries of the log2 table."""
    c = Case("16 MiB of one literal", expect={"split_clamp": 1})
    c.mb([(b"\x61" * (1 << 24), 0, 0)])
    return c.done()


# ---- E2 near its thresholds
def e2_quantities(data, log2, ctx_lut, map13):
    """The quantities the context decision compares, for one metablock of `data` sampled as encode.c:341 / :424 sample
    it (64 bytes every 4 096): entropy[1] - entropy[2] and entropy[2] - entropy[3] of ChooseContextMap at qualities 7+,
    and entropy[2] and entropy[1] - entropy[2] of the 13-context test.  log2: the encoder's table (float-rounded below
    256); ctx_lut: the UTF-8 context lookup (512 bytes: previous byte, then the one before)."""
    d = np.frombuffer(bytes(data), np.uint8)
    strides = [d[s:s + 64] for s in range(0, len(d) - 63, 4096)]

    def est(pop):
        tot = int(sum(pop))
        return tot * log2(tot) - sum(int(p) * log2(int(p)) for p in pop) if tot else 0.0
    lut = [0, 0, 1, 2]
    bigram = [0] * 9
    comb, ctxh, total = [0] * 32, [[0] * 32 for _ in range(13)], 0
    for w in strides:
        prev = lut[w[0] >> 6] * 3
        for x in w[1:]:
            bigram[prev + lut[x >> 6]] += 1
            prev = lut[x >> 6] * 3
        p2, p1 = int(w[0]), int(w[1])
        for x in w[2:]:
            c = map13[ctx_lut[p1] | ctx_lut[256 + p2]]
            total += 1; comb[x >> 3] += 1; ctxh[c][x >> 3] += 1
            p2, p1 = p1, int(x)
    mono = [sum(bigram[i] for i in range(9) if i % 3 == k) for k in range(3)]
    two = [sum(bigram[i] for i in range(9) if i % 6 == k) for k in range(6)]
    e0 = 1.0 / sum(mono)
    e1 = est(mono) * e0
    e2 = (est(two[:3]) + est(two[3:])) * e0
    e3 = sum(est(bigram[3 * i:3 * i + 3]) for i in range(3)) * e0
    f0 = 1.0 / total
    f1, f2 = est(comb) * f0, sum(est(h) for h in ctxh) * f0
    return {"e1-e2 (0.2)": e1 - e2, "e1-e3 (0.2)": e1 - e3, "e2-e3 (0.02)": e2 - e3, "13: e2 (3.0)": f2,
            "13: e1-e2 (0.2)": f1 - f2}


THRESHOLDS = {"e1-e2 (0.2)": 0.2, "e1-e3 (0.2)": 0.2, "e2-e3 (0.02)": 0.02, "13: e2 (3.0)": 3.0, "13: e1-e2 (0.2)": 0.2}


def markov_source(rng, strides):
    """A metablock of `strides` sampled strides whose 64 sampled bytes have top two bits that follow a random Markov chain
    (a random 4 x 4 transition matrix, sharpened by a random power) and low six bits random over a random range; the
    bytes between the strides are never sampled."""
    T = rng.random((4, 4)) ** rng.uniform(0.5, 8)
    T = np.cumsum(T / T.sum(1, keepdims=True), 1)
    n = 64 * strides
    u = rng.random(n)
    top = np.zeros(n, np.int64)
    for i in range(1, n):
        top[i] = min(3, int(np.searchsorted(T[top[i - 1]], u[i])))
    low = rng.integers(0, int(rng.integers(1, 65)), n)
    w = (top << 6 | low).astype(np.uint8).tobytes()
    return b"".join(w[64 * k:64 * k + 64] + (b"a" * 4032 if k + 1 < strides else b"") for k in range(strides))


def e2_search(log2, ctx_lut, map13, tries=3000, seed=2024, strides=4):
    """A seeded search over Markov sources of `strides` sampled strides for the cases closest below and above each
    threshold.  Returns {quantity: (below, above)}, each (margin, data)."""
    rng = np.random.default_rng(seed)
    best = {k: [None, None] for k in THRESHOLDS}
    for _ in range(tries):
        data = markov_source(rng, strides)
        for k, v in e2_quantities(data, log2, ctx_lut, map13).items():
            m = v - THRESHOLDS[k]
            side = 0 if m < 0 else 1
            if best[k][side] is None or abs(m) < abs(best[k][side][0]):
                best[k][side] = (m, data)
    return best
