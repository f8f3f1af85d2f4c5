"""The match search on its own: one search per probe, from a fully specified hash-table state.

A probe fixes the search position `cur`, the first position the walker owns (`p0`), the stream start, the block end
(max_length and the stale byte), max_backward, the dictionary distance, the distance cache, the incoming length and
score, and the static-dictionary counters.  Two stored-bit bitmaps are given for the whole input: the snapshot and the
walker's own bits; a position q counts as inserted when (q >= p0 ? own : snapshot) has it.  Three implementations run
the same probes and must agree:
  - the oracle's sequential find_longest_match / quick_find_longest_match over a real bucket table with uint16 counters
    (oracle_search_probe: the stream's inserted positions in front of cur are hashed into a fresh table first);
  - the product's search in the one-lane sim (tests/sim/search_probe.cc);
  - on the GPU, the product's search with a 32-lane warp (br_debug_search), on the index, tags, S-ordered snapshot and
    slot entry points built by the pipeline's own kernels; at quality 7..9 with every row grouping G (1, 4, 8).
At qualities 2..4 every slot read the search records (`saw`, what br_verify_run checks) must equal what numpy derives from
the index and the bitmaps.  The GPU's tagS / storedS / prefS are checked against numpy as well.

Every probe family is built for a branch ordinary parses meet rarely (ring-buffer stop and skip, ties at max_length that
the stale byte decides, wrapped bucket counters, len-2 distance-cache matches, the dictionary gate, full rings, streams of
a batch) and asserts that it reached that branch: through the oracle's edge counters (oracle/brotli_oracle.c
EDGE_FIELDS), or, for full rings, through which candidate won."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from brotli_libs import ROOT, TABLES, Oracle
from corpus import synth_binary, synth_text, synth_web
from golden_cases import make_case

W = 16                      # words per probe and per result (brotli_b200/csrc/br_probe.h)
MIN_SCORE = 2020            # BR_MIN_SCORE: the score every search of a parse starts from
SAW_ABSENT, SAW_SKIP = 0x80000000, 0xFFFFFFFE
U32 = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------- parameters
def derive(q, lgwin, lgblock, hint):
    """what br_derive_params (brotli_b200/csrc/br_params.h) decides for the search"""
    P = dict(q=q, lgwin=lgwin, quick=q < 5, max_backward=(1 << lgwin) - 16)
    if q < 5:
        lgb = 14 if q < 4 else 16
        if q == 4 and lgblock:
            lgb = min(24, max(16, lgblock))
        bits, sb, hl = {2: (16, 0, 5), 3: (16, 1, 5)}.get(q, (20, 2, 7) if hint >= (1 << 20) else (17, 2, 5))
        P.update(bits=bits, sweep_bits=sb, hash_len=hl, htl=8, block_size=1, ndist=1)
    else:
        lgb = 16 if q < 9 else min(lgwin, 18)
        if lgblock:
            lgb = min(24, max(16, lgblock))
        h64 = hint >= (1 << 20) and lgwin >= 19
        P.update(hash64=h64, bits=15 if h64 or q >= 7 else 14, htl=8 if h64 else 4, block_size=1 << (q - 1),
                 ndist=4 if q < 7 else 10 if q < 9 else 16)
    P["rmask"] = (1 << (1 + max(lgwin, lgb))) - 1
    return P


def _load64(d):
    a = np.frombuffer(bytes(d) + bytes(16), np.uint8)
    n = len(d)
    v = np.zeros(n, np.uint64)
    for k in range(8):
        v |= a[k:k + n].astype(np.uint64) << np.uint64(8 * k)
    return v


def index_of(d, bounds, P):
    """numpy restatement of the position index: keys of every position (bucket of H5 / H6 hashed over the whole input, or
    the quick hashers' slot counted from the stream start), S sorted by (key, position), seg"""
    n = len(d)
    v = _load64(d)
    with np.errstate(over="ignore"):
        if P["quick"]:
            base = np.repeat(np.r_[0, bounds[:-1]].astype(np.uint64), np.diff(np.r_[0, bounds]))
            key = ((v << np.uint64(64 - 8 * P["hash_len"])) * np.uint64(0x1FE35A7BD3579BD3)) >> np.uint64(64 - P["bits"])
            pos = np.arange(n, dtype=np.uint64) - base
            key = (key + (pos & np.uint64(((1 << P["sweep_bits"]) - 1) << 3))) & np.uint64((1 << P["bits"]) - 1)
        elif P["hash64"]:
            key = (v * np.uint64((0x1FE35A7BD3579BD3 << 24) & 0xFFFFFFFFFFFFFFFF)) >> np.uint64(49)
        else:
            key = ((v & np.uint64(U32)) * np.uint64(0x1E35A7BD) & np.uint64(U32)) >> np.uint64(32 - P["bits"])
    key = key.astype(np.int64)
    key[max(0, n - P["htl"] + 1):] = 1 << P["bits"]
    S = np.argsort(key, kind="stable").astype(np.int64)
    seg = np.searchsorted(key[S], np.arange((1 << P["bits"]) + 2), side="left")
    return key, S, seg


# ----------------------------------------------------------------------------------------------------------- libraries
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("probe") / "libsearchprobe.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-Wno-unused-function",
                           "-o", so, os.path.join(ROOT, "tests", "sim", "search_probe.cc")])
    L = C.CDLL(so)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    L.sim_debug_search.argtypes = [C.c_int] * 3 + [C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                                   C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def oracle():
    o = Oracle()
    o.lib.oracle_search_probe.argtypes = [C.c_int] * 3 + [C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_char_p,
                                                          C.c_void_p, C.c_size_t, C.c_void_p]
    return o


@pytest.fixture(scope="module")
def gpu():
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    L = brotli_b200.lib()
    L.br_debug_search.argtypes = [C.c_int] * 3 + [C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                                  C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    return L


# ---------------------------------------------------------------------------------------------------------------- inputs
_INPUTS = {}


def data_of(kind, n, seed=1):
    k = (kind, n, seed)
    if k not in _INPUTS:
        if kind == "text":
            d = synth_text(n, seed)
        elif kind == "web":
            d = synth_web(n, seed)
        elif kind == "binary":
            d = synth_binary(n, seed)
        elif kind == "noise":
            d = np.random.RandomState(seed).randint(0, 256, n, dtype=np.uint8).tobytes()
        elif kind == "zeros":
            d = bytes(n)
        elif kind == "dict":
            from fuzz_cases import dict_cases
            d = b"".join(x for _, x, _, _ in dict_cases(seed, 40, TABLES))
            d = (d * (n // len(d) + 1))[:n]
        else:   # golden kinds: heavy (one key > 65536 times), periodic
            d = make_case(dict(kind=kind, n=n, seed=seed, period=997 + seed))
        _INPUTS[k] = d
    return _INPUTS[k]


# ----------------------------------------------------------------------------------------------------------------- state
class Case:
    """one call: an input (a batch when bounds has several streams), parameters, the two bitmaps and sorted probes"""

    def __init__(self, d, q, lgwin, hint=None, lgblock=0, bounds=None, heavy_min=0):
        self.d, self.q, self.lgwin, self.lgblock = d, q, lgwin, lgblock
        self.n = len(d)
        self.bounds = np.array(bounds if bounds is not None else [self.n], np.int64)
        self.hint = hint or int(np.diff(np.r_[0, self.bounds]).max())
        self.heavy_min = heavy_min
        self.P = derive(q, lgwin, lgblock, self.hint)
        starts = np.r_[0, self.bounds[:-1]]
        self.base_of = np.repeat(starts, np.diff(np.r_[0, self.bounds]))
        self.end_of = np.repeat(self.bounds, np.diff(np.r_[0, self.bounds]))
        # positions the reference never inserts: the last HashTypeLength - 1 bytes of every stream
        self.insertable = np.arange(self.n) + self.P["htl"] <= self.end_of

    def set_bits(self, snap, own):
        self.snap = (snap & self.insertable).astype(np.uint8)
        self.own = (own & self.insertable).astype(np.uint8)

    def set_probes(self, pr):
        pr = pr[np.argsort(pr[:, 0], kind="stable")]
        pr = pr[np.r_[True, np.diff(pr[:, 0]) != 0]]          # one search per position
        assert np.all(pr[:, 0] + 8 <= self.end_of[pr[:, 0]]) and np.all(pr[:, 3] <= self.end_of[pr[:, 0]])
        assert np.all(pr[:, 3] > pr[:, 0])
        self.probes = np.ascontiguousarray(pr.astype(np.uint32))

    def words(self, m):
        b = np.packbits(m.astype(np.uint8), bitorder="little")
        b = np.concatenate([b, np.zeros(-len(b) % 4 + 4, np.uint8)])
        return np.ascontiguousarray(b.view(np.uint32))


def bitmaps(rng, n, kind):
    """a stored mask: all, parse-like (stored except runs of 1..40), Bernoulli 0.5 or 0.05"""
    if kind == "all":
        return np.ones(n, bool)
    if kind == "parse":
        m = np.ones(n, bool)
        for s in rng.randint(0, n, n // 60):
            m[s:s + rng.randint(1, 41)] = False
        return m
    return rng.random_sample(n) < {"b50": 0.5, "b05": 0.05}[kind]


def own_of(rng, snap, rate):
    """the walker's own bits: the snapshot with fresh flips (above a probe's p0 they count, below it they are ignored)"""
    return snap ^ (rng.random_sample(len(snap)) < rate)


def probes_for(rng, c, curs, dc=None, pend=None, p0=None, len_in=None, score_in=None, dict_lm=None, dict_distance=None):
    """probe words for positions `curs`; every field not given is drawn the way a parse produces it (with some spread)"""
    curs = np.asarray(curs, np.int64)
    k = len(curs)
    P = c.P
    base, end = c.base_of[curs], c.end_of[curs]
    if pend is None:
        span = rng.choice([8, 20, 300, 5000, 1 << 30], k) + rng.randint(0, 64, k)
        pend = np.minimum(end, curs + span)
    pend = np.maximum(pend, curs + 1)
    if p0 is None:
        # (never in front of the stream: a sweep ends at its stream's last block, br_walk_block, so a walker owns positions
        # of its own stream only -- br_ring_heavy's own-range scan relies on that in a batch)
        mode = rng.randint(0, 3, k)
        p0 = np.where(mode == 0, base, np.where(mode == 1, curs + 1, base + (rng.random_sample(k) * (curs - base + 1)).astype(np.int64)))
    maxb = np.minimum(curs - base, P["max_backward"])
    if dc is None:
        pool = np.array([1, 2, 3, 4, 8, 11, 15, 16, 24, 100, 997, 998, 1994, 4000])
        dc = rng.choice(pool, (k, 4))
        r = rng.random_sample((k, 4)) < 0.3
        dc[r] = (rng.random_sample(r.sum()) * np.repeat(maxb + 1, 4)[r.ravel()]).astype(np.int64)
    if len_in is None:
        len_in = np.zeros(k, np.int64)
        if P["quick"]:
            x = rng.randint(0, 4, k)
            ml = pend - curs
            len_in = np.where(x == 1, np.minimum(rng.randint(1, 12, k), ml), np.where(x == 2, ml, 0))
    if score_in is None:
        score_in = MIN_SCORE + np.where(rng.random_sample(k) < 0.15, rng.randint(0, 1500, k), 0)
    if dict_lm is None:
        dl = rng.randint(0, 1 << 20, k).astype(np.int64)
        dm = np.maximum(0, (dl >> 7) + rng.randint(-3, 60, k))
    else:
        dl, dm = dict_lm
    if dict_distance is None:
        dict_distance = maxb
    pr = np.zeros((k, W), np.int64)
    pr[:, 0], pr[:, 1], pr[:, 2], pr[:, 3], pr[:, 4], pr[:, 5] = curs, p0, base, pend, maxb, dict_distance
    pr[:, 6:10] = np.asarray(dc, np.int64) & U32
    pr[:, 10], pr[:, 11] = len_in, score_in
    pr[:, 12], pr[:, 13], pr[:, 14], pr[:, 15] = dl & U32, dl >> 32, dm & U32, dm >> 32
    return pr


# -------------------------------------------------------------------------------------------------------------- running
def run_sim(L, c):
    res = np.zeros((len(c.probes), W), np.uint32)
    sw, ow = c.words(c.snap), c.words(c.own)
    b = c.bounds.astype(np.uint32)
    assert L.sim_debug_search(c.q, c.lgwin, c.lgblock, c.hint, c.d, c.n, b.ctypes.data, len(b), sw.ctypes.data,
                              ow.ctypes.data, c.heavy_min, c.probes.ctypes.data, len(c.probes), res.ctypes.data)
    return res


def run_oracle(o, c):
    """the oracle runs every stream of a batch on its own"""
    res = np.zeros((len(c.probes), W), np.uint32)
    lo = 0
    for hi in c.bounds:
        sel = np.nonzero((c.probes[:, 0] >= lo) & (c.probes[:, 0] < hi))[0]
        if len(sel):
            pr = np.ascontiguousarray(c.probes[sel])
            r = np.zeros((len(sel), W), np.uint32)
            assert o.lib.oracle_search_probe(c.q, c.lgwin, c.lgblock, c.hint, c.d[lo:hi] + bytes(64), int(hi - lo),
                                             c.snap[lo:hi].tobytes(), c.own[lo:hi].tobytes(), pr.ctypes.data, len(sel),
                                             r.ctypes.data)
            res[sel] = r
        lo = hi
    return res


def run_gpu(L, c, S):
    n = c.n
    res = np.zeros((3, len(c.probes), W), np.uint32)
    tagS = np.zeros(n, np.uint16); storedS = np.zeros((n + 31) // 32, np.uint32); prefS = np.zeros((n + 1023) // 1024, np.uint32)
    sw, ow = c.words(c.snap), c.words(c.own)
    b = c.bounds.astype(np.uint32)
    nvar = L.br_debug_search(c.q, c.lgwin, c.lgblock, c.hint, c.d, n, b.ctypes.data, len(b), sw.ctypes.data, ow.ctypes.data,
                             c.heavy_min, c.probes.ctypes.data, len(c.probes), res.ctypes.data, tagS.ctypes.data,
                             storedS.ctypes.data, prefS.ctypes.data)
    assert nvar == (3 if c.q >= 7 else 1), nvar
    # the index's side arrays, against numpy
    a = np.frombuffer(c.d + bytes(4), np.uint8).astype(np.uint32)
    first4 = a[S] | a[S + 1] << 8 | a[S + 2] << 16 | a[S + 3] << 24
    with np.errstate(over="ignore"):
        assert np.array_equal(tagS, ((first4 * np.uint32(0x9E3779B1)) >> np.uint32(16)).astype(np.uint16)), "tagS"
    bits = c.snap[S].astype(np.uint8)
    want = np.packbits(bits, bitorder="little")
    want = np.concatenate([want, np.zeros(-len(want) % 4, np.uint8)]).view(np.uint32)
    assert np.array_equal(storedS, want[:len(storedS)]), "storedS"
    cnt = np.add.reduceat(bits.astype(np.int64), np.arange(0, n, 1024))
    assert np.array_equal(prefS, (np.cumsum(cnt) - cnt).astype(np.uint32)), "prefS"
    return res[:nvar]


def saw_expected(c, S, seg, key, res):
    """the slot reads of a quality 2..4 search: per slot, the latest inserted position in front of cur in the slot's segment
    of S (its index), or SAW_ABSENT | the index where the backward walk stopped (the segment's start, a position of an
    earlier stream, or one outside the window); SAW_SKIP for slot 0 when H2 took the last distance"""
    P = c.P
    sweep, mask = 1 << P["sweep_bits"], (1 << P["bits"]) - 1
    out = np.zeros((len(c.probes), 4), np.int64)
    for t, pr in enumerate(c.probes.astype(np.int64)):
        cur, p0, base, maxb = pr[0], pr[1], pr[2], pr[4]
        r = res[t]
        if sweep == 1 and r[2] != pr[11] and r[2] == 135 * r[0] + 1935:
            out[t, 0] = SAW_SKIP
            continue
        i_own = ((cur - base) >> 3) & (sweep - 1)
        k0 = (key[cur] - (i_own << 3)) & mask
        for i in range(sweep):
            slot = (k0 + (i << 3)) & mask
            lo, hi = seg[slot], seg[slot + 1]
            j = lo + np.searchsorted(S[lo:hi], cur)
            w = SAW_ABSENT | j
            while j > lo:
                q = S[j - 1]
                if q < base or cur - q > maxb:
                    break
                if (c.own if q >= p0 else c.snap)[q]:
                    w = j - 1
                    break
                j -= 1
                w = SAW_ABSENT | j
            out[t, i] = w
    return out


COUNTERS = ["srch_dc_len2", "srch_ring_break", "srch_ring_skip", "srch_tie_max", "srch_wrap_cut", "srch_dict_hit",
            "srch_gate_closed"]


def check(sim, oracle, c, gpu=None):
    """runs the case through every implementation; returns the oracle's search counters"""
    before = oracle.edge_stats()
    want = run_oracle(oracle, c)
    after = oracle.edge_stats()
    got = run_sim(sim, c)

    def same(a, b, what):
        bad = np.nonzero((a[:, :10] != b[:, :10]).any(axis=1))[0]
        if len(bad):
            t = bad[0]
            raise AssertionError("%s: %d of %d probes differ (q%d lgwin %d hint %d); first: probe %s -> %s, oracle %s" % (
                what, len(bad), len(a), c.q, c.lgwin, c.hint, c.probes[t].tolist(), a[t, :10].tolist(), b[t, :10].tolist()))
    same(got, want, "sim vs oracle")
    assert np.all(got[:, 8] == 1) and np.all(got[:, 9] == 1)
    key, S, seg = index_of(c.d, c.bounds, c.P)
    if c.P["quick"]:
        ws = saw_expected(c, S, seg, key, got)
        sweep = 1 << c.P["sweep_bits"]
        bad = np.nonzero((got[:, 10:10 + sweep] != ws[:, :sweep]).any(axis=1))[0]
        assert not len(bad), ("saw", c.q, c.probes[bad[0]].tolist(), got[bad[0], 10:14].tolist(), ws[bad[0]].tolist())
    if gpu is not None:
        for v, r in enumerate(run_gpu(gpu, c, S)):
            bad = np.nonzero((r != got).any(axis=1))[0]
            if len(bad):
                t = bad[0]
                raise AssertionError("GPU variant %d vs sim: %d of %d probes differ (q%d); first: probe %s -> %s, sim %s" % (
                    v, len(bad), len(r), c.q, c.probes[t].tolist(), r[t].tolist(), got[t].tolist()))
    return {k: after[k] - before[k] for k in COUNTERS}, got


# -------------------------------------------------------------------------------------------------------------- families
def fam_inputs(rng, q):
    """every input kind, both hashes (hints on both sides of 1 MiB, lgwin 18 / 19), every mask, own bits against the
    snapshot"""
    kinds = ["text", "web", "binary", "noise", "zeros", "heavy", "periodic", "dict"]
    for i, kind in enumerate(kinds):
        n = {"zeros": 1 << 16, "heavy": 600000}.get(kind, [1 << 16, 300000, (1 << 20) + 4096][i % 3])
        if kind == "text":
            n = 2 << 20
        d = data_of(kind, n, seed=3 + i)
        for lgwin, hint in ((18, n), (19, max(n, 1 << 20)), (22, min(n, (1 << 20) - 1))):
            c = Case(d, q, lgwin, hint=hint)
            mk = ["all", "parse", "b50", "b05"][rng.randint(4)]
            snap = bitmaps(rng, n, mk)
            c.set_bits(snap, own_of(rng, snap, rng.choice([0.01, 0.3])))
            k = 300 if kind in ("zeros", "heavy") else 2500
            curs = rng.randint(0, n - 8, k)
            c.set_probes(probes_for(rng, c, curs))
            yield c


def fam_ring(rng, q):
    """lgwin 17 with lgblock 16..24: searches whose position, or whose candidates, lie within max_length of the ring
    buffer's end (the stop cur_m + best_len > rmask and the skip prev_m + best_len > rmask)"""
    for lgblock in (16, 17, 18, 20, 24) if q >= 4 else (0,):
        c = Case(data_of("periodic", 1 << 20, seed=lgblock), q, 17, hint=1 << 20, lgblock=lgblock)
        R = c.P["rmask"] + 1
        snap = bitmaps(rng, c.n, ["all", "parse"][lgblock & 1])
        c.set_bits(snap, own_of(rng, snap, 0.02))
        period = 997 + lgblock
        curs = []
        for j in range(1, c.n // R + 1):
            for t in range(0, 6):
                curs += [j * R - dd + t * period for dd in range(1, 48)]
        curs = np.array([x for x in curs if 0 < x < c.n - 8])
        if len(curs) == 0:   # a ring larger than the input: positions at the half ring instead
            curs = np.arange(1, 2000) * 487
        c.set_probes(probes_for(rng, c, curs, pend=np.minimum(c.n, curs + rng.randint(4, 300, len(curs)))))
        yield c


def fam_block_ends(rng, q):
    """pend - cur from 1 to 20 on periodic data: several candidates reach max_length and the stale byte decides"""
    for lgwin, n in ((17, 1 << 20), (22, 300000)):
        d = data_of("periodic", n, seed=5)
        c = Case(d, q, lgwin, hint=n)
        snap = bitmaps(rng, n, "parse")
        c.set_bits(snap, own_of(rng, snap, 0.05))
        curs = np.unique(rng.randint(3000, n - 40, 6000))
        c.set_probes(probes_for(rng, c, curs, pend=curs + rng.randint(1, 21, len(curs))))
        yield c


def fam_dcache(rng, q):
    """distance caches of 0, negative, beyond max_backward, repeated; dc[0] / dc[1] +- 1..3 landing on 0 or on the window
    edge (max_backward and one past it); len-2 matches at k < 2 and k >= 2"""
    for kind, n in (("binary", 300000), ("text", 300000), ("noise", 1 << 16)):
        d = data_of(kind, n, seed=7)
        c = Case(d, q, 18, hint=n)
        snap = bitmaps(rng, n, "all")
        c.set_bits(snap, own_of(rng, snap, 0.1))
        k = 4000
        curs = np.unique(rng.randint(8, n - 8, k))
        k = len(curs)
        maxb = np.minimum(curs, c.P["max_backward"])
        dc = rng.choice([0, -1, -5, 1, 2, 3, 4], (k, 4)).astype(np.int64)
        edge = rng.randint(0, 6, (k, 4))
        dc = np.where(edge == 1, maxb[:, None] + rng.randint(-3, 4, (k, 4)), dc)
        dc = np.where(edge == 2, maxb[:, None] + 1 + rng.randint(0, 1 << 20, (k, 4)), dc)
        dc = np.where(edge == 3, np.repeat(dc[:, :1], 4, axis=1), dc)
        # len-2 candidates: a position with the same two bytes as cur
        a = np.frombuffer(d, np.uint8).astype(np.int64)
        two = a[:-1] | a[1:] << 8
        order = np.argsort(two, kind="stable")
        first = np.searchsorted(two[order], two[curs])
        cand = order[np.minimum(first + rng.randint(0, 3, k), len(order) - 1)]
        ok = (cand < curs) & (two[cand] == two[curs])
        slot = rng.randint(0, 4, k)
        l2 = (edge[np.arange(k), slot] >= 4) & ok
        dc[np.arange(k)[l2], slot[l2]] = (curs - cand)[l2]
        c.set_probes(probes_for(rng, c, curs, dc=dc))
        yield c


def fam_dict(rng, q):
    """dictionary words; dict_l / dict_m one step either side of the gate dict_m < dict_l >> 7; dictionary distances other
    than max_backward (STREAM_OFFSET)"""
    n = 300000
    d = data_of("dict", n, seed=9)
    for lgwin in (18, 22):
        c = Case(d, q, lgwin, hint=n)
        snap = bitmaps(rng, n, "b05")
        c.set_bits(snap, own_of(rng, snap, 0.05))
        curs = np.unique(rng.randint(8, n - 40, 6000))
        k = len(curs)
        dl = rng.randint(128, 1 << 24, k).astype(np.int64) + (rng.random_sample(k) < 0.1) * (1 << 33)
        dm = (dl >> 7) + rng.randint(-1, 2, k)
        maxb = np.minimum(curs, c.P["max_backward"])
        dd = np.where(rng.random_sample(k) < 0.5, maxb, np.minimum(curs + rng.randint(1, 1 << 20, k), c.P["max_backward"]))
        c.set_probes(probes_for(rng, c, curs, dict_lm=(dl, dm), dict_distance=dd))
        yield c


def fam_heavy(rng, q):
    """the heavy golden kind (one key every 8 bytes, > 65536 times): stored counts whose value modulo 65536 sits at 0,
    1, block_size - 1, block_size, block_size + 1 at the probe, from the snapshot and from own bits above p0 far behind cur;
    and ordinary buckets moved onto the heavy path by a lowered heavy_min"""
    n = 1300000
    d = data_of("heavy", n, seed=12)
    bs = 1 << (q - 1)
    for lgwin, hint in ((22, n), (18, n)):
        c = Case(d, q, lgwin, hint=hint)
        snap = bitmaps(rng, n, "all")
        snap[rng.randint(0, n, 3000)] = False
        c.set_bits(snap, own_of(rng, snap, 0.02))
        key = index_of(d, c.bounds, c.P)[0]
        heavy = np.nonzero(key[:n - 8] == key[0])[0]            # the bucket of "abcd" / "abcde", collisions included
        probes = []
        for t in range(30):
            p0 = int(rng.randint(0, 700000))
            ins = np.where(heavy >= p0, c.own[heavy], c.snap[heavy]).astype(np.int64)
            before = np.cumsum(ins) - ins                        # inserted heavy positions in front of each
            target = [0, 1, bs - 1, bs, bs + 1][t % 5]       # (0: the ring looks empty)
            hit = np.nonzero((before >= 65536) & (before % 65536 == target) & (heavy > p0))[0]
            if len(hit):
                cur = int(heavy[hit[rng.randint(len(hit))]])
                probes.append(probes_for(rng, c, [cur], p0=np.array([p0])))
        c.set_probes(np.concatenate(probes))
        yield c
    t = data_of("text", 300000, seed=13)
    c = Case(t, q, 22, heavy_min=int(rng.choice([1, 40, 300])))
    snap = bitmaps(rng, c.n, "parse")
    c.set_bits(snap, own_of(rng, snap, 0.2))
    c.set_probes(probes_for(rng, c, rng.randint(0, c.n - 8, 3000)))
    yield c


def fam_ring_full(rng, q):
    """full rings: a 40-byte string X, then m copies of X's first 8 bytes (m = block_size - 1 .. block_size + 2), then X
    again at the probe.  The ring holds the block_size newest entries: X's first copy is in it only while fewer than
    block_size entries of its bucket lie between it and the probe, and then it is the best match (40 bytes against 8)"""
    bs = 1 << (q - 1)
    parts, curs, first = [], [], []
    pos = 0
    for t in range(max(8, 2048 // bs)):
        m = bs - 1 + t % 4
        x = rng.randint(1, 256, 40).astype(np.uint8).tobytes()
        seg = bytearray(64 * (m + 2) + 64)
        seg[0:40] = x
        for i in range(m):
            seg[64 * (i + 1):64 * (i + 1) + 8] = x[:8]
        seg[64 * (m + 1):64 * (m + 1) + 40] = x
        first.append(pos); curs.append(pos + 64 * (m + 1))
        parts.append(bytes(seg)); pos += len(seg)
    d = b"".join(parts)
    c = Case(d, q, 22)
    snap = np.ones(c.n, bool)
    for k in (5, 6, 7):   # m = block_size .. block_size + 2 without the newest copy: the stored entries straddle a row
        snap[np.array(curs)[k::8] - 64] = False
    c.set_bits(snap, snap.copy())
    curs = np.array(curs)
    c.set_probes(probes_for(rng, c, curs, dc=np.full((len(curs), 4), 3), pend=np.minimum(c.n, curs + 300),
                            dict_lm=(np.zeros(len(curs), np.int64), np.zeros(len(curs), np.int64))))
    key = index_of(d, c.bounds, c.P)[0]
    c.in_ring = np.array([((key[a + 1:b] == key[b]) & (c.snap[a + 1:b] > 0)).sum() < bs for a, b in zip(first, curs)])
    yield c


def fam_batch(rng, q):
    """three streams end to end: probes in the second and third stream (base > 0); the oracle sees each stream alone"""
    parts = [data_of("text", 200000, seed=21), data_of("periodic", 150000, seed=22), data_of("web", 250000, seed=23)]
    d = b"".join(parts)
    bounds = np.cumsum([len(x) for x in parts])
    c = Case(d, q, 18, bounds=bounds, heavy_min=int(rng.choice([0, 64])))
    snap = bitmaps(rng, c.n, "parse")
    c.set_bits(snap, own_of(rng, snap, 0.1))
    curs = rng.randint(bounds[0], c.n, 5000)
    curs = curs[curs + 8 <= c.end_of[curs]]
    near = np.concatenate([bounds[:2] + x for x in (0, 1, 2, 5, 9, 17, 100)])
    c.set_probes(probes_for(rng, c, np.concatenate([curs, near])))
    yield c


def fam_quick(rng, q):
    """qualities 2..4: best_len_in > 0 up to max_length, H2's early returns, empty slots at the stream start and beyond
    a small window"""
    for lgwin, n in ((10, 1 << 16), (16, 300000), (22, (1 << 20) + 100)):
        d = data_of(["binary", "text", "web"][lgwin % 3], n, seed=lgwin)
        c = Case(d, q, lgwin)
        snap = bitmaps(rng, n, ["b50", "parse", "all"][lgwin % 3])
        c.set_bits(snap, own_of(rng, snap, 0.1))
        curs = np.concatenate([np.arange(0, 300), rng.randint(0, n - 8, 5000)])
        dc = rng.choice([1, 4, 8, 16, 1000, 3000], (len(curs), 4))
        c.set_probes(probes_for(rng, c, curs, dc=dc))
        yield c


FAMILIES = {
    "inputs": (fam_inputs, ()),
    "ring": (fam_ring, ("srch_ring_break", "srch_ring_skip")),
    "block_ends": (fam_block_ends, ("srch_tie_max",)),
    "dcache": (fam_dcache, ("srch_dc_len2",)),
    "dict": (fam_dict, ("srch_dict_hit", "srch_gate_closed")),
    "heavy": (fam_heavy, ("srch_wrap_cut",)),
    "ring_full": (fam_ring_full, ()),
    "batch": (fam_batch, ()),
}
QUICK_FAMILIES = {"inputs": (fam_inputs, ()), "quick": (fam_quick, ()), "ring": (fam_ring, ()),
                  "block_ends": (fam_block_ends, ()), "batch": (fam_batch, ())}


def run_family(sim, oracle, q, fam, gpu=None):
    fams = QUICK_FAMILIES if q < 5 else FAMILIES
    fn, want = fams[fam]
    rng = np.random.RandomState(1000 * q + sum(map(ord, fam)))
    total = {k: 0 for k in COUNTERS}
    nprobes = found = 0
    saw_kinds = set()
    for c in fn(rng, q):
        cnt, res = check(sim, oracle, c, gpu)
        for k in cnt:
            total[k] += cnt[k]
        nprobes += len(c.probes)
        found += int((res[:, 0] > 0).sum())
        if fam == "ring_full":   # X's first copy only while it is in the ring
            assert np.array_equal(res[:, 0] >= 40, c.in_ring) and c.in_ring.any() and not c.in_ring.all(), res[:, 0].tolist()
        if q < 5:
            s = res[:, 10:10 + (1 << c.P["sweep_bits"])].ravel()
            saw_kinds |= {"skip" if x == SAW_SKIP else "absent" if x & SAW_ABSENT else "found" for x in s}
    for k in want:
        assert total[k] > 0, (fam, q, k, total)
    assert found > 0, (fam, q)
    if q < 5 and fam == "quick":
        assert saw_kinds >= ({"found", "absent", "skip"} if q == 2 else {"found", "absent"}), saw_kinds
    return nprobes


CPU_PARAMS = [(q, f) for q in (5, 6, 7, 8, 9) for f in FAMILIES] + [(q, f) for q in (2, 3, 4) for f in QUICK_FAMILIES]


@pytest.mark.parametrize("q,fam", CPU_PARAMS)
def test_search_sim_equals_oracle(sim, oracle, q, fam):
    run_family(sim, oracle, q, fam)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [2, 3, 4, 5, 6, 7, 8, 9])
def test_search_gpu_equals_oracle(sim, oracle, gpu, q):
    for fam in (QUICK_FAMILIES if q < 5 else FAMILIES):
        run_family(sim, oracle, q, fam, gpu)
