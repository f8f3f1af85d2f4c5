"""The prefix codes of a job (E4 in br_entropy2.h): built and stored by one warp per code when the job has at most
BR_CODE_WARP_MAX (8 192) of them, else by one thread per code, with the metablock headers written in between.

CPU: the device code run on the CPU (tests/sim, which takes the warp workers' functions) equals the oracle for inputs in
which stored-raw metablocks lie between compressed ones (they have no codes).
GPU (-m gpu): the same inputs through BrotliEncoderCompress, and batch jobs of thousands of tiny streams through
BrotliB200CompressBatch, whose codes outnumber what the warps take, so the thread workers build and store them.  The late
uncompressed fallback (encode.c:604), which runs the entropy stage a second time on the same job, is covered by
test_zz_gpu_q234.py at quality 4 and by the batch tests of test_gpu_parity.py.

E4 on its own: the crafted histogram families of code_cases.py, packed into synthetic metablocks, through the hooks
br_debug_codes (the pipeline's own launches on the GPU) and sim_debug_codes (the same worker functions on the CPU, the
thread workers' too, over a pool of tree areas dealt as k_codes deals them).  Every code is compared with the oracle's
oracle_build_code: the smoothed counts, the bit offsets and the stored bits exactly; the depths over the symbols with a
nonzero smoothed count (and 0 elsewhere when there are two or more); the code words where the depth is nonzero.  Checks
that rely on neither (an RFC 7932 reader of the stored code, the Kraft sum, canonical code words, smoothing that keeps
nonzero counts nonzero, the cost of an unconstrained Huffman tree) run on the oracle's outputs on the CPU and on the
device's on the GPU."""
import ctypes as C
import heapq
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import code_cases
from brotli_libs import ROOT, TABLES, Oracle

SIM_SO = os.path.join(ROOT, "tests", "sim", "libbrsim.so")


def _tiny_streams(count, seed):
    """count streams of 300 .. 2 000 bytes cut from text, web and binary data: each is compressed, with at least a literal,
    a command and a distance code, so the job has more than 3 * count codes."""
    from corpus import synth_binary, synth_text, synth_web
    pool = synth_web(1_000_000, seed) + synth_text(500_000, seed + 1) + synth_binary(500_000, seed + 2)
    rnd = np.random.RandomState(seed)
    out = []
    for _ in range(count):
        n = int(rnd.randint(300, 2001))
        o = int(rnd.randint(0, len(pool) - n))
        out.append(pool[o:o + n])
    return out


def _mixed(seed):
    """Text, noise, binary data, noise, text: the noise is stored raw, in metablocks between compressed ones."""
    from corpus import synth_binary, synth_text
    rnd = np.random.default_rng(seed).integers(0, 256, 600_000, dtype=np.uint8).tobytes()
    return synth_text(250_000, seed + 1) + rnd[:350_000] + synth_binary(200_000, seed + 2) + rnd[350_000:] + synth_text(150_000, seed + 3)


MIXED = [(q, w) for q in (4, 5, 6) for w in (18, 22)]


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def sim():
    if not os.path.exists(SIM_SO):
        import __graft_entry__
        __graft_entry__.build_checkers()
    L = C.CDLL(SIM_SO)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    L.sim_compress.restype = C.c_long
    L.sim_compress.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
    L.sim_debug_codes.argtypes = _CODES_ARGS
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    return L


@pytest.mark.parametrize("q,w", MIXED)
def test_sim_raw_metablocks_between_compressed(sim, oracle, q, w):
    d = _mixed(910)
    cap = 2 * len(d) + 100000
    out = C.create_string_buffer(cap)
    st = np.zeros(8, np.uint32)
    r = sim.sim_compress(q, w, d, len(d), out, cap, st.ctypes.data)
    assert r >= 0 and out.raw[:r] == oracle.compress(d, q, w), (q, w)


@pytest.fixture(scope="module")
def b200():
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    return brotli_b200


@pytest.mark.gpu
def test_gpu_raw_metablocks_between_compressed(b200, oracle):
    d = _mixed(910)
    for q, w in MIXED:
        assert b200.compress_oneshot(d, q, w) == oracle.compress(d, q, w), (q, w)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [4, 5])
def test_gpu_batch_of_tiny_streams(b200, oracle, q):
    """8 192 tiny streams, one device job (br_driver.h kBatchGroupStreams): over 24 000 codes for the thread workers."""
    items = _tiny_streams(8192, 920 + q)
    got = b200.compress_batch(items, q, 22, threads=4)
    for k, x in enumerate(items):
        assert got[k] == oracle.compress(x, q, 22), k


# ------------------------------------------------------------------------------------------------ E4 on its own
# br_debug_codes / sim_debug_codes (br_kernels.cu, tests/sim/br_sim.cc): n_mbs, counts, histos, code_ctas, H, depth, bits,
# offsets, out, out_words, info
_CODES_ARGS = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
               C.c_uint32, C.c_void_p]
OUT_WORDS = 1 << 16          # bit buffer words returned per metablock (2 Mbit: 768 codes of 704 symbols fit)
WARP_MAX = 8192              # BR_CODE_WARP_MAX
KIND = {1: "warp", 2: "thread"}


def _pack(codes, seed):
    """Synthetic metablocks for codes [(label, histogram)]: every metablock takes up to 256 codes of each alphabet; an
    alphabet that has run out is filled with one padding code (a metablock has at least one code of each).  Returns a list
    of metablocks, each three lists of (label, histogram) in code order: literal, command, distance codes."""
    q = {A: [c for c in codes if len(c[1]) == A] for A in code_cases.ALPHABETS}
    mbs, k = [], 0
    while any(q.values()):
        mb = []
        for A in code_cases.ALPHABETS:
            take, q[A] = q[A][:256], q[A][256:]
            if not take:
                take = code_cases.padding(A, 1, seed * 1000 + k)
                k += 1
            mb.append(take)
        mbs.append(mb)
    return mbs


def _pad_to(mbs, total, seed):
    """mbs followed by metablocks of padding codes, so that the job has exactly `total` codes."""
    r = total - sum(len(x) for mb in mbs if mb for x in mb)
    assert r == 0 or r >= 3, r
    out, k = list(mbs), 0
    while r:
        n = [min(256, r - 2), 0, 0] if r <= 768 else [256, 256, 256]
        if r > 768 and r - 768 < 3:
            n = [250, 256, 256]
        if r <= 768:
            n[1] = min(256, r - n[0] - 1)
            n[2] = r - n[0] - n[1]
        out.append([code_cases.padding(A, n[j], seed * 1000 + k + j) for j, A in enumerate(code_cases.ALPHABETS)])
        k += 3
        r -= sum(n)
    return out


class _Codes:
    """What one hook call gave, per code in job order: label, alphabet, input, H, depth, bits, bit offset, stored bits."""

    def __init__(self, fn, mbs, ctas):
        n = len(mbs)
        counts = np.zeros(3 * n, np.uint32)
        codes = []
        for i, mb in enumerate(mbs):
            if mb:
                counts[3 * i:3 * i + 3] = [len(x) for x in mb]
                codes += [c for x in mb for c in x]
        lens = np.asarray([len(h) for _, h in codes], np.int64)
        starts = np.concatenate([[0], np.cumsum(lens)])
        histos = np.concatenate([h for _, h in codes]).astype(np.uint32)
        H, depth, bits = np.zeros(len(histos), np.uint32), np.zeros(len(histos), np.uint8), np.zeros(len(histos), np.uint16)
        offsets = np.zeros(len(codes) + n, np.uint32)
        out = np.zeros(n * OUT_WORDS, np.uint32)
        info = np.zeros(3, np.uint32)
        assert fn(n, counts.ctypes.data, histos.ctypes.data, ctas, H.ctypes.data, depth.ctypes.data, bits.ctypes.data,
                  offsets.ctypes.data, out.ctypes.data, OUT_WORDS, info.ctypes.data) == 1
        self.total, self.kind, self.workers = int(info[0]), KIND[int(info[1])], int(info[2])
        assert self.total == len(codes)
        self.labels = [c[0] for c in codes]
        self.inputs = [c[1] for c in codes]
        sl = [slice(int(starts[g]), int(starts[g + 1])) for g in range(len(codes))]
        self.H, self.depth, self.bits = [H[x] for x in sl], [depth[x] for x in sl], [bits[x] for x in sl]
        self.off, self.stored, self.mb_bits, self.mb_ends = [], [], [], []
        o = 0
        for i, mb in enumerate(mbs):
            if not mb:
                assert offsets[o] == 0 and not out[i * OUT_WORDS:(i + 1) * OUT_WORDS].any(), "raw metablock %d" % i
                o += 1
                continue
            nt = sum(len(x) for x in mb)
            offs = offsets[o:o + nt + 1].astype(np.int64)
            o += nt + 1
            assert offs[-1] + 256 <= OUT_WORDS * 32, "metablock %d: the codes end at bit %d" % (i, offs[-1])
            b = np.unpackbits(out[i * OUT_WORDS:(i + 1) * OUT_WORDS].view(np.uint8), bitorder="little")
            assert not b[offs[-1]:offs[-1] + 256].any(), "metablock %d: bits written behind its last code" % i
            self.mb_bits.append(b[:offs[-1]])
            self.mb_ends.append(int(offs[-1]))
            for x in range(nt):
                self.off.append(int(offs[x]))
                self.stored.append(b[offs[x]:offs[x + 1]])


_ORACLE_CODES = {}


def _oracle_code(oracle, label, h):
    """oracle_build_code of one histogram: H, depth, bits, stored bits (a bit array), cached by label."""
    r = _ORACLE_CODES.get(label)
    if r is None:
        H, depth, bits, stored, nbits = oracle.build_code(h)
        sb = np.unpackbits(np.frombuffer(stored, np.uint8), bitorder="little")[:nbits]
        r = _ORACLE_CODES[label] = (H, depth, bits, sb)
    return r


def _first_difference(got, g, want):
    """The first field of code g that differs from want's (H, depth, bits, stored bits), or None.  Depths are compared
    over the used symbols, and must be 0 elsewhere with two or more; a code of at most one symbol leaves the others' depths
    unwritten (as BuildAndStoreHuffmanTree does).  Code words are compared where the depth is nonzero."""
    H, depth, bits, sb = want
    if not np.array_equal(got.H[g], H):
        return "smoothed histogram (first at symbol %d)" % int(np.nonzero(got.H[g] != H)[0][0])
    if len(got.stored[g]) != len(sb):
        return "bit offset: the code takes %d bits, the oracle's %d" % (len(got.stored[g]), len(sb))
    if not np.array_equal(got.stored[g], sb):
        return "stored bits (first at bit %d of the code)" % int(np.nonzero(got.stored[g] != sb)[0][0])
    used = H > 0
    if not np.array_equal(got.depth[g][used], depth[used]):
        return "depth of a used symbol"
    if used.sum() >= 2 and got.depth[g][~used].any():
        return "depth of an unused symbol"
    nz = used & (depth > 0)
    if not np.array_equal(got.bits[g][nz], bits[nz]):
        return "code words"
    return None


def _compare(oracle, got, what):
    """Every code of a hook call against the oracle: fails with the first code that differs."""
    bad = []
    for g in range(got.total):
        d = _first_difference(got, g, _oracle_code(oracle, got.labels[g], got.inputs[g]))
        if d:
            bad.append("code %d (%s), %s worker: %s" % (g, got.labels[g], got.kind, d))
    assert not bad, "%s: %d of %d codes differ; first: %s" % (what, len(bad), got.total, bad[0])


# ---- checks that rely on neither the oracle nor the device
class _Reader:
    def __init__(self, bits):
        self.b, self.p = bits, 0

    def read(self, n):
        if self.p + n > len(self.b):
            raise ValueError("reads past the code's stored size")
        v = 0
        for i in range(n):
            v |= int(self.b[self.p + i]) << i
        self.p += n
        return v


def _canonical(lengths):
    """RFC 7932 section 3.2: the canonical code of every symbol with a nonzero length, {(length, code): symbol}."""
    bl = [0] * 16
    for x in lengths:
        bl[x] += 1
    bl[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    res = {}
    for s, x in enumerate(lengths):
        if x:
            res[s] = nxt[x]
            nxt[x] += 1
    return res


def read_prefix_code(bits, A):
    """RFC 7932 sections 3.4 and 3.5: the code lengths of a prefix code over A symbols stored in `bits` (LSB first).
    Returns (lengths, bits read, NSYM of a simple code or 0)."""
    r = _Reader(bits)
    abits = (A - 1).bit_length()
    lengths = [0] * A
    hskip = r.read(2)
    if hskip == 1:                                   # simple prefix code
        nsym = r.read(2) + 1
        syms = [r.read(abits) for _ in range(nsym)]
        if len(set(syms)) != nsym or max(syms) >= A:
            raise ValueError("simple code symbols %s" % syms)
        ls = {1: [0], 2: [1, 1], 3: [1, 2, 2]}.get(nsym)
        if nsym == 4:
            ls = [1, 2, 3, 3] if r.read(1) else [2, 2, 2, 2]
        for s, x in zip(syms, ls):
            lengths[s] = x
        return lengths, r.p, nsym
    order = (1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    cl, space, num = [0] * 18, 32, 0
    for i in range(hskip, 18):                       # the code-length code, in the fixed code of section 3.5
        b = (r.read(1), r.read(1))
        x = {(0, 0): 0, (0, 1): 3, (1, 0): 4}.get(b)
        if x is None:
            x = 2 if r.read(1) == 0 else (1 if r.read(1) == 0 else 5)
        cl[order[i]] = x
        if x:
            space -= 32 >> x
            num += 1
            if space <= 0:
                break
    if num != 1 and space != 0:
        raise ValueError("code-length code is not complete")
    if num == 1:
        only = next(s for s in range(18) if cl[s])
        table = None
    else:
        table = {(cl[s], c): s for s, c in _canonical(cl).items()}

    def symbol():
        if table is None:
            return only
        code, n = 0, 0
        while True:
            code, n = (code << 1) | r.read(1), n + 1
            if (n, code) in table:
                return table[(n, code)]
            if n > 5:
                raise ValueError("no code-length symbol")

    sym, prev, rep, rep_len, space = 0, 8, 0, 0, 32768
    while sym < A and space > 0:
        c = symbol()
        if c < 16:
            rep = 0
            lengths[sym] = c
            sym += 1
            if c:
                prev = c
                space -= 32768 >> c
            continue
        extra, new_len = (2, prev) if c == 16 else (3, 0)
        if rep_len != new_len:
            rep, rep_len = 0, new_len
        old = rep
        if rep > 0:
            rep = (rep - 2) << extra
        rep += r.read(extra) + 3
        delta = rep - old
        if sym + delta > A:
            raise ValueError("repeat past the alphabet")
        for _ in range(delta):
            lengths[sym] = new_len
            sym += 1
        if new_len:
            space -= delta * (32768 >> new_len)
    if space != 0:
        raise ValueError("code lengths do not form a complete code")
    return lengths, r.p, 0


def _huffman(counts):
    """Cost (sum of count * depth) and depth of an unconstrained Huffman tree of counts (all nonzero, two or more);
    on equal weights the lower subtree is merged first."""
    h = [(int(c), 0, i) for i, c in enumerate(counts)]
    heapq.heapify(h)
    cost, k = 0, len(h)
    while len(h) > 1:
        a, b = heapq.heappop(h), heapq.heappop(h)
        cost += a[0] + b[0]
        heapq.heappush(h, (a[0] + b[0], max(a[1], b[1]) + 1, k))
        k += 1
    return cost, h[0][1]


def independent_check(h_in, H, depth, bits, stored):
    """What one built and stored code must satisfy whatever built it; returns the first violation, or None."""
    A = len(H)
    if np.any((h_in > 0) & (H == 0)):
        return "smoothing turned a nonzero count into 0"
    used = H > 0
    nsym = int(used.sum())
    try:
        lengths, nread, simple = read_prefix_code(stored, A)
    except ValueError as e:
        return "RFC 7932 reader: %s" % e
    if nread != len(stored):
        return "the reader takes %d of the code's %d bits" % (nread, len(stored))
    lengths = np.asarray(lengths)
    if nsym <= 1:
        want = int(np.nonzero(used)[0][0]) if nsym else 0
        if simple != 1 or lengths.any() or nread != 4 + (A - 1).bit_length():
            return "a code of %d symbols is not a one-symbol simple code" % nsym
        if stored[4:].dot(1 << np.arange(len(stored) - 4)) != want:
            return "the one-symbol code names another symbol than %d" % want
        return None
    d = depth.astype(np.int64)
    if d.max() > 15:
        return "depth %d" % d.max()
    if np.any(d[used] == 0) or np.any(d[~used] != 0):
        return "depths do not match the used symbols"
    if int(np.sum(1 << (15 - d[used]))) != 1 << 15:
        return "Kraft sum is not 1"
    if not np.array_equal(lengths, d):
        return "the stored code's lengths are not the depths"
    can = _canonical(d.tolist())
    for s, c in can.items():
        if int(bits[s]) != int("{:0{w}b}".format(c, w=d[s])[::-1], 2):
            return "code word of symbol %d is not the bit-reversed canonical code" % s
    cost, hd = _huffman(H[used])
    if hd <= 15 and int(np.sum(H.astype(np.int64) * d)) != cost:
        return "cost %d, the Huffman tree's %d" % (int(np.sum(H.astype(np.int64) * d)), cost)
    return None


def _independent_all(labels, inputs, H, depth, bits, stored, who):
    bad = []
    for g in range(len(labels)):
        e = independent_check(inputs[g], H[g], depth[g], bits[g], stored[g])
        if e:
            bad.append("code %d (%s), %s: %s" % (g, labels[g], who, e))
    assert not bad, "%d codes fail; first: %s" % (len(bad), bad[0])


# ---- CPU
@pytest.mark.parametrize("family", list(code_cases.FAMILIES))
def test_code_family_reaches_its_edges(oracle, family):
    oracle.edge_stats_reset()
    for _, h in code_cases.cases(family):
        oracle.build_code(h)
    got = oracle.edge_stats()
    miss = {k: (got[k], v) for k, v in code_cases.expect(family).items() if got[k] < v}
    assert not miss, "%s: edge counters below their least values (got, want): %s" % (family, miss)


def test_oracle_codes_pass_independent_checks(oracle):
    cs = code_cases.cases()
    res = [_oracle_code(oracle, label, h) for label, h in cs]
    _independent_all([c[0] for c in cs], [c[1] for c in cs], [r[0] for r in res], [r[1] for r in res], [r[2] for r in res],
                     [r[3] for r in res], "oracle")


def test_independent_checks_catch_a_wrong_code(oracle):
    """The checks reject a code with one stored bit flipped, one depth changed, one code word changed."""
    label, h = next(c for c in code_cases.cases("random") if (c[1] > 0).sum() > 40)
    H, depth, bits, sb = _oracle_code(oracle, label, h)
    assert independent_check(h, H, depth, bits, sb) is None
    flipped = sb.copy()
    flipped[len(sb) // 2] ^= 1
    d2 = depth.copy()
    d2[np.nonzero(depth)[0][0]] += 1
    b2 = bits.copy()
    b2[np.nonzero(depth)[0][0]] ^= 1
    for args in ((H, depth, bits, flipped), (H, d2, bits, sb), (H, depth, b2, sb)):
        assert independent_check(h, *args) is not None


def test_sim_codes_warp_workers(sim, oracle):
    """Every family through the warp workers' functions, with raw metablocks between coded ones."""
    mbs = _pack(code_cases.cases(), 1)
    mbs = mbs[:2] + [None] + mbs[2:5] + [None, None] + mbs[5:] + [None]
    got = _Codes(sim.sim_debug_codes, mbs, 0)
    assert got.kind == "warp" and got.total <= WARP_MAX
    _compare(oracle, got, "sim, warp workers")


@pytest.mark.parametrize("ctas", [1, 3])
def test_sim_codes_thread_workers(sim, oracle, ctas):
    """More than 8 192 codes: the thread workers' functions, each worker building and storing dozens of codes over one
    tree area that the previous code left dirty."""
    mbs = _pad_to(_pack(code_cases.cases(), 2), WARP_MAX + 1, 3)
    got = _Codes(sim.sim_debug_codes, mbs, ctas)
    assert got.kind == "thread" and got.workers == 64 * ctas and got.total == WARP_MAX + 1
    _compare(oracle, got, "sim, %d thread workers" % got.workers)


# ---- GPU
@pytest.fixture(scope="module")
def gpu_codes(b200):
    L = b200.lib()
    L.br_debug_codes.argtypes = _CODES_ARGS
    return L


@pytest.mark.gpu
def test_gpu_codes_warp_workers(gpu_codes, sim, oracle):
    """Every family in one call (a warp per code); the device's codes pass the independent checks, and its bit buffers
    (the headers included) equal the sim's."""
    mbs = _pack(code_cases.cases(), 1)
    got = _Codes(gpu_codes.br_debug_codes, mbs, 0)
    assert got.kind == "warp"
    _compare(oracle, got, "device, warp workers")
    _independent_all(got.labels, got.inputs, got.H, got.depth, got.bits, got.stored, "device")
    ref = _Codes(sim.sim_debug_codes, mbs, 0)
    for i, (a, b) in enumerate(zip(got.mb_bits, ref.mb_bits)):
        assert np.array_equal(a, b), "metablock %d: the device's bit buffer differs from the sim's" % i


@pytest.mark.gpu
def test_gpu_codes_8192_and_8193(gpu_codes, oracle):
    """The families padded to exactly 8 192 codes (warps) and to 8 193 (threads, one code each): identical results."""
    base = _pack(code_cases.cases(), 1)
    a = _Codes(gpu_codes.br_debug_codes, _pad_to(base, WARP_MAX, 4), 0)
    b = _Codes(gpu_codes.br_debug_codes, _pad_to(base, WARP_MAX + 1, 4), 0)
    assert (a.kind, b.kind) == ("warp", "thread") and b.workers >= b.total
    _compare(oracle, b, "device, 8 193 codes")
    where = {label: g for g, label in enumerate(b.labels)}
    last = a.total - sum(len(x) for x in _pad_to(base, WARP_MAX, 4)[-1])    # (only the last padding metablock differs)
    for g in range(a.total):
        gb = where.get(a.labels[g])
        if gb is None:
            continue
        d = _first_difference(a, g, (b.H[gb], b.depth[gb], b.bits[gb], b.stored[gb]))
        assert d is None, "code %d (%s): 8 192 and 8 193 codes differ in the %s" % (g, a.labels[g], d)
        assert g >= last or a.off[g] == b.off[gb], "code %d (%s): bit offset differs" % (g, a.labels[g])
    _compare(oracle, a, "device, 8 192 codes")


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", [1, 3, 0])
def test_gpu_codes_thread_workers(gpu_codes, sim, oracle, ctas):
    """More than 8 192 codes with 1 and 3 CTAs of thread workers (dozens of codes each, over one tree area) and with the
    pipeline's count; raw metablocks between the coded ones."""
    mbs = _pad_to(_pack(code_cases.cases(), 2), WARP_MAX + 1, 3)
    mbs = mbs[:3] + [None] + mbs[3:-1] + [None] + mbs[-1:]
    got = _Codes(gpu_codes.br_debug_codes, mbs, ctas)
    assert got.kind == "thread"
    if ctas:
        assert got.workers == 64 * ctas and got.total >= 24 * got.workers
    print("thread workers: %d codes over %d workers" % (got.total, got.workers))
    _compare(oracle, got, "device, %d thread workers" % got.workers)
    _independent_all(got.labels, got.inputs, got.H, got.depth, got.bits, got.stored, "device")
    ref = _Codes(sim.sim_debug_codes, mbs, ctas)
    for i, (a, b) in enumerate(zip(got.mb_bits, ref.mb_bits)):
        assert np.array_equal(a, b), "metablock %d: the device's bit buffer differs from the sim's" % i


def _many_code_streams(count, seed):
    """count streams of 4 .. 6 KiB, each with many prefix codes: short segments of 32 dialects in turn, each dialect 16
    ASCII bytes and 4 lead bytes of two-byte UTF-8 sequences.  A segment's literals differ enough from the last two block
    types' to open a new one (about 11 literal types a stream), and the sequences make the context model take 2 contexts
    (encode.c ChooseContextMap; 3 need quality 7), so every type has two literal codes: about 16 codes a stream."""
    rng = np.random.default_rng(seed)
    pools = [rng.choice(np.arange(0x21, 0x7F), 16, replace=False).astype(np.uint8) for _ in range(32)]
    leads = [rng.choice(np.arange(0xC2, 0xE0), 4, replace=False).astype(np.uint8) for _ in range(32)]
    out = []
    for _ in range(count):
        n = int(rng.integers(4096, 6145))
        parts, m = [], 0
        while m < n:
            k = int(rng.integers(0, 32))
            seg = int(rng.integers(150, 200))
            a, b = rng.choice(pools[k], seg), rng.choice(pools[k], seg)
            lead, cont = rng.choice(leads[k], seg), rng.integers(0x80, 0xC0, seg).astype(np.uint8)
            pick = rng.random(seg) < 0.7
            parts.append(np.where(pick[:, None], np.stack([lead, cont], 1), np.stack([a, b], 1)).ravel().tobytes())
            m += 2 * seg
        out.append(b"".join(parts)[:n])
    return out


@pytest.mark.gpu
def test_gpu_batch_more_codes_than_thread_workers(b200, oracle):
    """8 192 streams of a few KiB in one device job (br_driver.h: at most 8 192 streams, under 128 MiB, each under 1 MiB)
    with at least 1.5 * 65 536 prefix codes in all: more codes than the job's 65 536 thread workers, so workers build and
    store a second code over their tree area.  Each stream's bytes equal the oracle's."""
    items = _many_code_streams(8192, 930)
    assert sum(len(x) for x in items) < 128 << 20

    def one(x):          # (the oracle's edge counters are per thread)
        oracle.edge_stats_reset()
        return oracle.compress(x, 5, 22), oracle.stored_codes()

    with ThreadPoolExecutor(8) as ex:
        res = list(ex.map(one, items))
    want, codes = [r[0] for r in res], sum(r[1] for r in res)
    print("batch: %d streams, %d prefix codes (oracle)" % (len(items), codes))
    assert codes >= 1.5 * 65536, codes
    got = b200.compress_batch(items, 5, 22, threads=4)
    for k in range(len(items)):
        assert got[k] == want[k], k
