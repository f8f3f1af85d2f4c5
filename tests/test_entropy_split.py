"""The literal context decision (E2, br_decide_context_modeling in k_mb_setup) and the greedy block splitter (E3,
br_split_cta in k_split) on their own, on the jobs of split_cases.py: exact ties at every threshold, block counts around
the shortest block, type caps, literal contexts at stream, metablock and batch-stream starts, a 16 MiB metablock,
E2's length and size-hint boundaries, random command streams and the oracle's own parse of the corpus.

Three runs of the same job: br_debug_split (the pipeline's own launches on the GPU: the E0 scans, k_expand, launch_split,
launch_codes), sim_debug_split (the same device functions on the CPU, one thread per CTA) and oracle_split (the oracle's
restatement: the split-building half of its metablock store, then the header-and-codes half).  Each returns, per
compressed metablock, the context count, the splits, the histograms before smoothing and the metablock's bits up to the
end of its last prefix code.  A failure names the case, the metablock, the category and the first differing block or bit.

CPU: the sim equals the oracle; the oracle's output passes checks that rely on neither (histograms recounted from the
splits and the symbol stream, the padding rule, the type sequence rules, the shortest block, the type cap); every case
reaches the edge counter it was built for; the exact ties are ties in exact arithmetic.
GPU (-m gpu): every family through br_debug_split against the oracle and the sim; one job mixing the families with raw
metablocks; the oracle's parse of the corpus at qualities 5..9."""
import ctypes as C
import os

import numpy as np
import pytest

import split_cases as sc
from brotli_libs import ROOT, TABLES, Oracle

SIM_SO = os.path.join(ROOT, "tests", "sim", "libbrsim.so")
SPLIT_REF = os.path.join(ROOT, "oracle", "_ref", "split_ref")
SPLIT_REF_CALLS = os.path.join(ROOT, "tests", "golden", "split_reference.json")
# (in, n, cmds, ncmd, mbs, n_mbs, quality, size_hint, disable_ctx, out, out_cap)
_ARGS = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_int,
         C.c_void_p, C.c_size_t]
CMD_DT = np.dtype([("insert", "<u4"), ("copy", "<u4"), ("dist_extra", "<u4"), ("cmd_prefix", "<u2"), ("dist_prefix", "<u2")])


@pytest.fixture(scope="module")
def oracle():
    o = Oracle()
    L = o.lib
    L.oracle_split.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_size_t,
                               C.c_int, C.c_void_p, C.c_size_t]
    L.oracle_split.restype = C.c_size_t
    L.oracle_make_cmd.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p]
    L.oracle_make_insert_cmd.argtypes = [C.c_uint32, C.c_void_p]
    L.oracle_static_context_map.argtypes = [C.c_size_t, C.c_void_p]
    return o


@pytest.fixture(scope="module")
def sim():
    if not os.path.exists(SIM_SO):
        import __graft_entry__
        __graft_entry__.build_checkers()
    L = C.CDLL(SIM_SO)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    L.sim_debug_split.argtypes = _ARGS
    L.sim_debug_split.restype = C.c_long
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 24) + 2)     # the device's table: a 16 MiB metablock's counts reach 2^24
    return L


def _cmds(oracle, case):
    """The case's commands as the encoder's 16-byte commands, built by the oracle's InitCommand."""
    if isinstance(case.cmds, np.ndarray):
        return case.cmds
    out = np.zeros(len(case.cmds), CMD_DT)
    memo = {}
    one = np.zeros(1, CMD_DT)
    for k, t in enumerate(case.cmds):
        if t not in memo:
            ins, copy, dcode = t
            if copy:
                oracle.lib.oracle_make_cmd(ins, copy, 0, dcode, one.ctypes.data)
            else:
                oracle.lib.oracle_make_insert_cmd(ins, one.ctypes.data)
            memo[t] = one[0].copy()
        out[k] = memo[t]
    case.cmds = out
    return out


def _cap(case, cmds):
    """Words the records of the case's compressed metablocks may take."""
    words = 0
    for start, end, c0, nc, _, comp, _ in case.mbs:
        if not comp:
            continue
        nlit = int(cmds["insert"][c0:c0 + nc].sum())
        nb = (nlit // 512 + 2, nc // 1024 + 2, nc // 512 + 2)
        words += 8 + 2 * sum(nb) + min(256, 13 * nb[0]) * 256 + min(256, nb[1]) * 704 + min(256, nb[2]) * 64
        words += (2 * (end - start) + 503) // 4 + 16
    return words


def run(fn, oracle, case):
    """One hook on the case: the parsed records of its compressed metablocks."""
    cmds = _cmds(oracle, case)
    mbs = np.asarray(case.mbs, np.uint32).ravel()
    cap = _cap(case, cmds)
    out = np.zeros(cap, np.uint32)
    data = bytes(case.data)
    r = fn(data, len(data), cmds.ctypes.data, len(cmds), mbs.ctypes.data, len(case.mbs), case.quality, case.size_hint,
           case.disable_ctx, out.ctypes.data, cap)
    assert 0 < r <= cap, (case.label, r, cap)
    return _parse(out[:r])


def _parse(w):
    recs, k = [], 0
    while k < len(w):
        which, nt, nb, nbits = int(w[k]), [int(x) for x in w[k + 1:k + 4]], [int(x) for x in w[k + 4:k + 7]], int(w[k + 7])
        k += 8
        rec = {"which": which, "num_types": nt, "num_blocks": nb, "nbits": nbits, "types": [], "lengths": [], "H": []}
        for cat in range(3):
            rec["types"].append(w[k:k + nb[cat]]); k += nb[cat]
            rec["lengths"].append(w[k:k + nb[cat]]); k += nb[cat]
        for cat, A in enumerate((256, 704, 64)):
            rows = nt[cat] * (which if cat == 0 else 1)
            rec["H"].append(w[k:k + rows * A].reshape(rows, A)); k += rows * A
        nw = (nbits + 31) // 32
        rec["bits"] = w[k:k + nw]; k += nw
        recs.append(rec)
    return recs


def _first_bit(a, b):
    x = np.nonzero(a != b)[0][0]
    return 32 * int(x) + int(np.nonzero([(int(a[x] ^ b[x]) >> j) & 1 for j in range(32)])[0][0])


def compare(got, want, label, what):
    assert len(got) == len(want), "%s: %s returned %d compressed metablocks, the oracle %d" % (label, what, len(got), len(want))
    for m, (g, o) in enumerate(zip(got, want)):
        where = "%s, metablock %d (%s vs oracle)" % (label, m, what)
        assert g["which"] == o["which"], "%s: %d literal contexts, oracle %d" % (where, g["which"], o["which"])
        for cat in range(3):
            cw = "%s, %s" % (where, sc.CATS[cat])
            gt, ot, gl, ol = g["types"][cat], o["types"][cat], g["lengths"][cat], o["lengths"][cat]
            n = min(len(gt), len(ot))
            d = np.nonzero((gt[:n] != ot[:n]) | (gl[:n] != ol[:n]))[0]
            assert not len(d), "%s: block %d is (type %d, length %d), oracle (%d, %d)" % (cw, d[0], gt[d[0]], gl[d[0]], ot[d[0]], ol[d[0]])
            assert g["num_types"][cat] == o["num_types"][cat] and len(gt) == len(ot), \
                "%s: %d types / %d blocks, oracle %d / %d" % (cw, g["num_types"][cat], len(gt), o["num_types"][cat], len(ot))
            if not np.array_equal(g["H"][cat], o["H"][cat]):
                r, s = np.argwhere(g["H"][cat] != o["H"][cat])[0]
                raise AssertionError("%s: histogram row %d symbol %d is %d, oracle %d" % (cw, r, s, g["H"][cat][r, s], o["H"][cat][r, s]))
        if g["nbits"] != o["nbits"] or not np.array_equal(g["bits"], o["bits"]):
            n = min(len(g["bits"]), len(o["bits"]))
            fb = _first_bit(g["bits"][:n], o["bits"][:n]) if not np.array_equal(g["bits"][:n], o["bits"][:n]) else None
            raise AssertionError("%s: header and codes take %d bits, oracle %d; first differing bit %s" % (where, g["nbits"], o["nbits"], fb))


# ---- oracle-free checks
def symbols(case, cmds, mb):
    """The symbol stream of each category of a metablock, from the data and the 16-byte commands."""
    start, end, c0, nc = mb[:4]
    c = cmds[c0:c0 + nc]
    lit, pos = [], start
    for k in range(nc):
        ins, copy = int(c["insert"][k]), int(c["copy"][k]) & 0x1FFFFFF
        lit.append(np.frombuffer(bytes(case.data[pos:pos + ins]), np.uint8))
        pos += ins + copy
    lit = np.concatenate(lit) if lit else np.zeros(0, np.uint8)
    hasd = ((c["copy"] & 0x1FFFFFF) != 0) & (c["cmd_prefix"] >= 128)
    return lit.astype(np.int64), c["cmd_prefix"].astype(np.int64), (c["dist_prefix"][hasd] & 0x3FF).astype(np.int64)


def check_record(case, cmds, mb, rec):
    """None, or what is wrong with a metablock's record by rules that hold whatever the splitter decided."""
    syms = symbols(case, cmds, mb)
    nc = rec["which"]
    if nc not in (1, 2, 3, 13):
        return "%d literal contexts" % nc
    for cat, A in enumerate((256, 704, 64)):
        name, mn = sc.CATS[cat], sc.MIN_BLOCK[cat]
        t, ln, s = rec["types"][cat].astype(np.int64), rec["lengths"][cat].astype(np.int64), syms[cat]
        nt, ctx = rec["num_types"][cat], (nc if cat == 0 else 1)
        if not len(t) or t[0] != 0 or nt != t.max() + 1:
            return "%s: types %s, %d types" % (name, t[:8], nt)
        if nt > 256 // ctx:
            return "%s: %d types over the cap %d" % (name, nt, 256 // ctx)
        seen = 1
        for k in range(1, len(t)):
            if t[k] == t[k - 1]:
                return "%s: blocks %d and %d have the same type" % (name, k - 1, k)
            if t[k] == seen:
                seen += 1
            elif k < 2 or t[k] != t[k - 2]:
                return "%s: block %d has type %d, neither new (%d) nor the type before last" % (name, k, t[k], seen)
        if (ln[:-1] < mn).any():
            return "%s: a block before the last is shorter than %d" % (name, mn)
        tot = int(ln.sum())
        if not (tot == mn if len(s) == 0 else len(s) <= tot <= len(s) + mn and tot >= mn):
            return "%s: lengths sum to %d for %d symbols" % (name, tot, len(s))
        H = rec["H"][cat].reshape(nt, ctx, A).sum(1)
        want = np.zeros((nt, A), np.int64)
        bt = np.repeat(t, ln)[:len(s)]
        np.add.at(want, (bt, s), 1)
        if not np.array_equal(H, want):
            r, x = np.argwhere(H != want)[0]
            return "%s: type %d symbol %d counted %d, recounted %d" % (name, r, x, H[r, x], want[r, x])
    return None


def families():
    text = open(os.path.join(ROOT, "tests", "golden", "fixtures", "alice29.txt"), "rb").read()
    return {
        "ties": sc.ties(),
        "block counts": sc.block_counts(),
        "type caps": sc.type_caps(),
        "contexts": sc.contexts(text),
        "E2 lengths": sc.e2_lengths(text),
        "random": sc.random_streams(40, 77),
    }


FAMILIES = sorted(families())


@pytest.fixture(scope="module")
def cases():
    return families()


@pytest.mark.parametrize("fam", FAMILIES)
def test_sim_equals_oracle(sim, oracle, cases, fam):
    for case in cases[fam]:
        compare(run(sim.sim_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case), case.label, "sim")


@pytest.mark.parametrize("fam", FAMILIES)
def test_oracle_independent_checks(oracle, cases, fam):
    for case in cases[fam]:
        recs = run(oracle.lib.oracle_split, oracle, case)
        comp = [mb for mb in case.mbs if mb[5]]
        for m, (mb, rec) in enumerate(zip(comp, recs)):
            err = check_record(case, case.cmds, mb, rec)
            assert err is None, "%s, metablock %d: %s" % (case.label, m, err)


def test_independent_checks_catch_a_wrong_split(oracle):
    """The checks reject a histogram count moved, a type sequence broken and a short block."""
    case = sc.tie_back(0, 2, 5)[0]
    rec = run(oracle.lib.oracle_split, oracle, case)[0]
    mb = case.mbs[0]
    assert check_record(case, case.cmds, mb, rec) is None
    bad = dict(rec, H=[h.copy() for h in rec["H"]])
    r, s = np.argwhere(bad["H"][0] > 0)[0]
    bad["H"][0][r, s] -= 1
    bad["H"][0][r, (s + 1) % 256] += 1
    assert check_record(case, case.cmds, mb, bad) is not None
    bad = dict(rec, types=[t.copy() for t in rec["types"]])
    bad["types"][0][2] = 1
    assert check_record(case, case.cmds, mb, bad) is not None
    bad = dict(rec, lengths=[x.copy() for x in rec["lengths"]])
    bad["lengths"][0][0] -= 1
    bad["lengths"][0][-1] += 1
    assert check_record(case, case.cmds, mb, bad) is not None


@pytest.mark.parametrize("fam", FAMILIES)
def test_cases_reach_their_branch(oracle, cases, fam):
    for case in cases[fam]:
        if not case.expect:
            continue
        oracle.edge_stats_reset()
        run(oracle.lib.oracle_split, oracle, case)
        st = oracle.edge_stats()
        for k, v in case.expect.items():
            assert st[k] >= v, "%s: edge counter %s is %d" % (case.label, k, st[k])


def test_exact_ties_decide_as_built(oracle):
    """Exactly at the threshold the block merges; 2 bits above it splits; exactly 20 bits apart the third block merges;
    22 apart it goes back to the first type.  In every category."""
    for cat in range(3):
        mn = sc.MIN_BLOCK[cat]
        for extra, want in ((0, [0]), (2, [0, 1])):
            case = sc.tie_split(cat, extra, 10 + cat)[0]
            rec = run(oracle.lib.oracle_split, oracle, case)[0]
            assert list(rec["types"][cat]) == want, (case.label, rec["types"][cat])
        for extra, want, lens in ((0, [0, 1], [mn]), (2, [0, 1, 0], [mn, mn])):
            case = sc.tie_back(cat, extra, 20 + cat)[0]
            rec = run(oracle.lib.oracle_split, oracle, case)[0]
            assert list(rec["types"][cat]) == want and list(rec["lengths"][cat])[:len(lens)] == lens, (case.label, rec["types"][cat], rec["lengths"][cat])
        case = sc.clamp(cat, 30 + cat)
        assert list(run(oracle.lib.oracle_split, oracle, case)[0]["types"][cat]) == [0], case.label


def test_float_rounded_log2_decides(oracle):
    """The exact ties moved off the tie by float-rounded log2 entries below 256: the literal split tie splits, the
    literal go-back tie goes back; in exact arithmetic both would merge."""
    (cat, small), (cat2, xa) = sc.ROUNDING
    rec = run(oracle.lib.oracle_split, oracle, sc.tie_split(cat, 0, 14, small)[0])[0]
    assert list(rec["types"][cat]) == [0, 1], rec["types"][cat]
    rec = run(oracle.lib.oracle_split, oracle, sc.tie_back(cat2, 0, 24, xa)[0])[0]
    assert list(rec["types"][cat2]) == [0, 1, 0], rec["types"][cat2]


def test_context_counts_by_quality(oracle, cases):
    """The two-byte UTF-8 data takes 3 literal contexts from quality 7 on and fewer below."""
    got = {}
    for case in cases["E2 lengths"]:
        if "UTF-8" in case.label:
            got[case.quality] = run(oracle.lib.oracle_split, oracle, case)[0]["which"]
    assert all(got[q] != 3 for q in (5, 6)) and all(got[q] == 3 for q in (7, 8, 9)), got


def test_stride_count_boundary(oracle, cases):
    """A metablock of 4 159 bytes samples one 64-byte stride for the context decision, one of 4 160 bytes two."""
    got = {}
    for case in cases["E2 lengths"]:
        if "stride boundary" in case.label:
            side = 13 if "13-context" in case.label else 0
            got[(side, case.quality, len(case.data))] = run(oracle.lib.oracle_split, oracle, case)[0]["which"]
    for q in range(5, 10):
        assert got[(0, q, 4159)] == 1 and got[(0, q, 4160)] == got[(0, q, 4161)] != 1 and (q < 7 or got[(0, q, 4160)] == 3), got
        assert got[(13, q, 4159)] == 1 and got[(13, q, 4160)] == got[(13, q, 4161)] == 13, got


def test_context_counts_reached(oracle, cases):
    """The context and E2 families reach 1, 2 or 3 and 13 literal contexts (the 13-context map only with a size hint of
    1 MiB or more)."""
    seen = {}
    for case in cases["contexts"] + cases["E2 lengths"]:
        for rec in run(oracle.lib.oracle_split, oracle, case):
            seen.setdefault(rec["which"], set()).add(case.size_hint >= 1 << 20)
    assert 1 in seen and 13 in seen and seen[13] == {True} and (2 in seen or 3 in seen), seen


# ---- the oracle's splitter against the reference's BrotliBuildMetaBlockGreedy (oracle/split_ref.c)
def _ref_input(oracle, case, mb, nctx):
    """The harness's input for one metablock, with the context count and static map the oracle chose."""
    import struct
    start, end, c0, nc, _, _, base = mb
    p1 = case.data[start - 1] if start >= base + 1 else 0
    p2 = case.data[start - 2] if start >= base + 2 else 0
    smap = np.zeros(64, np.uint32)
    if nctx > 1:
        assert oracle.lib.oracle_static_context_map(nctx, smap.ctypes.data) == 1
    return (struct.pack("<5I", nctx, p1, p2, end - start, nc) + smap.tobytes() + bytes(case.data[start:end]) +
            case.cmds[c0:c0 + nc].tobytes())


def _split_line(rec):
    """A record's splits and histograms as the harness prints them."""
    out = []
    for cat in range(3):
        out += [rec["num_types"][cat], rec["num_blocks"][cat]] + list(rec["types"][cat]) + list(rec["lengths"][cat])
    w = [str(int(x)) for x in out] + [str(int(x)) for h in rec["H"] for x in h.ravel()]
    return " " + " ".join(w)


def _sha(b):
    import hashlib
    return hashlib.sha256(b).hexdigest()[:32]


class RecordedSplitRef:
    """The reference's splits, as digests of the harness's output keyed by the digest of its input: recorded in
    tests/golden/split_reference.json when BROTLI_SPLIT_REF_RECORD is set (and oracle/_ref/split_ref is built), read
    from it otherwise.  An input that was never recorded fails."""

    def __init__(self):
        import json
        self.record = bool(os.environ.get("BROTLI_SPLIT_REF_RECORD"))
        self.calls = json.load(open(SPLIT_REF_CALLS)) if os.path.exists(SPLIT_REF_CALLS) else {}

    def digests(self, inputs):
        if self.record:
            import json
            import subprocess
            assert os.path.exists(SPLIT_REF), "oracle/_ref/split_ref is not built"
            res = subprocess.run([SPLIT_REF], input=b"".join(inputs) + b"\0\0\0\0", stdout=subprocess.PIPE, check=True)
            lines = res.stdout.decode().split("\n")[:len(inputs)]
            for i, line in zip(inputs, lines):
                self.calls[_sha(i)] = _sha(line.encode())
            with open(SPLIT_REF_CALLS, "w") as f:
                json.dump(dict(sorted(self.calls.items())), f, indent=0)
        missing = [k for k in map(_sha, inputs) if k not in self.calls]
        assert not missing, "%d metablocks have no recorded reference split (BROTLI_SPLIT_REF_RECORD=1 records them)" % len(missing)
        return [self.calls[_sha(i)] for i in inputs]


E3_FAMILIES = [f for f in FAMILIES if f != "E2 lengths"]


@pytest.mark.parametrize("fam", E3_FAMILIES)
def test_oracle_equals_reference(oracle, cases, fam):
    """Every compressed metablock of every E3 case: the oracle's splits and histograms equal the reference's."""
    ref = RecordedSplitRef()
    inputs, lines, where = [], [], []
    for case in cases[fam]:
        _cmds(oracle, case)
        comp = [mb for mb in case.mbs if mb[5]]
        for m, (mb, rec) in enumerate(zip(comp, run(oracle.lib.oracle_split, oracle, case))):
            inputs.append(_ref_input(oracle, case, mb, rec["which"]))
            lines.append(_split_line(rec))
            where.append("%s, metablock %d" % (case.label, m))
    for w, line, d in zip(where, lines, ref.digests(inputs)):
        assert _sha(line.encode()) == d, "%s: the oracle's splits or histograms differ from the reference's" % w


def test_e2_one_shot_equals_reference(oracle, cases):
    """E2 through whole streams: every E2 case whose size hint is below 1 MiB, compressed in one shot (its own length is
    then the size hint), equals the reference's bytes, and its metablock takes the context count the oracle's counters
    show, the one oracle_split chose."""
    from brotli_libs import RecordedRef
    ref = RecordedRef()
    for case in cases["E2 lengths"]:
        if case.size_hint >= 1 << 20:
            continue
        data = bytes(case.data)
        oracle.edge_stats_reset()
        got = oracle.compress(data, case.quality, 22)
        st = oracle.edge_stats()
        assert got == ref.compress(data, case.quality, 22), case.label
        which = run(oracle.lib.oracle_split, oracle, case)[0]["which"]
        assert st["ctx_nc%d" % which] == 1 and sum(st["ctx_nc%d" % k] for k in (1, 2, 3, 13)) == 1, (case.label, which)


@pytest.fixture(scope="module")
def e2_near(oracle):
    """The seeded search's cases closest below and above each threshold of the context decision."""
    import functools
    blob = open(TABLES, "rb").read()
    off = 8 + 32 + 128 + 122784 + 65536 + 32768 + 1024      # oracle_init's layout: the UTF-8 context lookup
    ctx_lut = list(blob[off:off + 512])
    map13 = np.zeros(64, np.uint32)
    oracle.lib.oracle_static_context_map(13, map13.ctypes.data)
    log2 = functools.lru_cache(None)(lambda v: oracle.lib.oracle_fast_log2(v) if v else 0.0)
    return sc.e2_search(log2, ctx_lut, [int(x) for x in map13])


def test_e2_near_thresholds(sim, oracle, e2_near):
    """Just below and just above each threshold (0.2 twice and 0.02 at quality 9; 3.0 and 0.2 on the 13-context side):
    the sim equals the oracle, and the oracle's choice follows the margins."""
    for k, pair in e2_near.items():
        assert all(pair), "%s: no case on one side" % k
        for margin, data in pair:
            print("%s: margin %+.3g" % (k, margin))
            side13 = k.startswith("13")
            case = sc.Case("E2 %s %+.3g" % (k, margin), quality=9, size_hint=(1 << 20) if side13 else (1 << 20) - 1,
                           disable_ctx=0).mb([(data, 0, 0)]).done()
            got, want = run(sim.sim_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case)
            compare(got, want, case.label, "sim")
            q = sc.e2_quantities(data, lambda v: oracle.lib.oracle_fast_log2(v) if v else 0.0, *_e2_tables(oracle))
            if side13:
                assert (want[0]["which"] == 13) == (not (q["13: e2 (3.0)"] > 3.0 or q["13: e1-e2 (0.2)"] < 0.2)), (k, q)
            else:
                one = q["e1-e2 (0.2)"] < 0.2 and q["e1-e3 (0.2)"] < 0.2
                assert (want[0]["which"] == 1) == one, (k, q, want[0]["which"])
                if not one:
                    assert want[0]["which"] == (2 if q["e2-e3 (0.02)"] < 0.02 else 3), (k, q)


def _e2_tables(oracle):
    blob = open(TABLES, "rb").read()
    off = 8 + 32 + 128 + 122784 + 65536 + 32768 + 1024
    map13 = np.zeros(64, np.uint32)
    oracle.lib.oracle_static_context_map(13, map13.ctypes.data)
    return list(blob[off:off + 512]), [int(x) for x in map13]


@pytest.mark.gpu
def test_gpu_e2_near_thresholds(gpu, oracle, e2_near):
    for k, pair in e2_near.items():
        for margin, data in pair:
            case = sc.Case("E2 %s %+.3g" % (k, margin), quality=9, size_hint=(1 << 20) if k.startswith("13") else (1 << 20) - 1,
                           disable_ctx=0).mb([(data, 0, 0)]).done()
            compare(run(gpu.br_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case), case.label, "device")


def test_sim_16mib_metablock(sim, oracle):
    case = sc.large()
    compare(run(sim.sim_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case), case.label, "sim")


# ---- GPU
@pytest.fixture(scope="module")
def gpu(oracle):
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    L = brotli_b200.lib()
    L.br_debug_split.argtypes = _ARGS
    L.br_debug_split.restype = C.c_long
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
def test_gpu_equals_oracle_and_sim(gpu, sim, oracle, cases, fam):
    for case in cases[fam]:
        got = run(gpu.br_debug_split, oracle, case)
        compare(got, run(oracle.lib.oracle_split, oracle, case), case.label, "device")
        compare(got, run(sim.sim_debug_split, oracle, case), case.label, "device vs sim")


@pytest.mark.gpu
def test_gpu_16mib_metablock(gpu, oracle):
    case = sc.large()
    compare(run(gpu.br_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case), case.label, "device")


def _concat(cases, label):
    """The cases laid end to end as one job, each a stream of its own (its metablocks' base is its first byte)."""
    out = sc.Case(label, quality=9, size_hint=1 << 20, disable_ctx=0)
    cm = []
    for case in cases:
        off, coff = len(out.data), sum(len(x) for x in cm)
        out.data += case.data
        cm.append(case.cmds)
        for mb in case.mbs:
            out.mbs.append([mb[0] + off, mb[1] + off, mb[2] + coff, mb[3], 0, mb[5], mb[6] + off])
    out.cmds = np.concatenate(cm)
    return out.done()


@pytest.mark.gpu
def test_gpu_mixed_job(gpu, oracle, cases):
    """Every family but the E2 one (its quality and size hint are its point) in one job of a few thousand metablocks,
    raw ones among them."""
    pool = [c for f in FAMILIES if f != "E2 lengths" for c in cases[f]]
    for c in pool:
        _cmds(oracle, c)
    job = []
    while sum(len(c.mbs) for c in job) < 2000:
        job += pool
    job = job[:max(k for k in range(len(job) + 1) if sum(len(c.mbs) for c in job[:k]) <= 2500)]
    big = _concat(job, "mixed job")
    for mb in big.mbs[::7]:
        mb[5] = 0
    big.mbs[0][5] = 1
    print("mixed job: %d metablocks, %d bytes" % (len(big.mbs), len(big.data)))
    compare(run(gpu.br_debug_split, oracle, big), run(oracle.lib.oracle_split, oracle, big), big.label, "device")


def _corpus_case(oracle, data, q):
    """The oracle's own parse of data at quality q: every metablock's commands as its compressor hands them over."""
    case = sc.Case("corpus q%d" % q, quality=q, size_hint=len(data), disable_ctx=0)
    got = []
    HOOK = C.CFUNCTYPE(None, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t)

    def hook(p, n, pos, nbytes):
        if n and nbytes:
            got.append((np.frombuffer(C.string_at(p, 16 * n), CMD_DT).copy(), pos, nbytes))
    cb = HOOK(hook)
    L = oracle.lib
    L.oracle_brotli_compress_hook.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, HOOK]
    cap = len(data) * 2 + 4096
    out = C.create_string_buffer(cap)
    n = C.c_size_t(cap)
    assert L.oracle_brotli_compress_hook(q, 22, len(data), data, C.byref(n), out, cb) == 1
    case.data = bytearray(data)
    cm, c0 = [], 0
    for cmds, pos, nbytes in got:
        case.mbs.append([pos, pos + nbytes, c0, len(cmds), 0, 1, 0])
        cm.append(cmds)
        c0 += len(cmds)
    case.cmds = np.concatenate(cm)
    return case.done()


@pytest.mark.gpu
@pytest.mark.parametrize("q", [5, 6, 7, 8, 9])
def test_gpu_corpus(gpu, oracle, q):
    from corpus import synth_binary, synth_text, synth_web
    data = synth_text(1_500_000, 31) + synth_web(1_000_000, 32) + synth_binary(500_000, 33)
    case = _corpus_case(oracle, data, q)
    compare(run(gpu.br_debug_split, oracle, case), run(oracle.lib.oracle_split, oracle, case), case.label, "device")
