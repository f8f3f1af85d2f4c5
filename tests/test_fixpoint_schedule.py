"""The LZ77 fixpoint under every schedule (DESIGN.md section 3).

Qualities 2..9 walk chunks speculatively, commit their stored-bits, and repeat until nothing is dirty.  The schedule decides
which chunks a launch walks, in what order their walks and commits land (on the GPU they run concurrently), when sweeps
start (sweep_epoch), when the full-sweep and forced safety nets take over (full sweeps from sweep_epoch + 9, the forced
walker from force_epoch), where the dependency marking falls back to the block rule (step_cap), which buckets take the
counter-wrap path (heavy_min), whether the first launch is a pilot and how many input blocks a sweep may cross
(sweep_blocks).  The bytes must not depend on any of it: every legal schedule ends on the sequential parse.

The default schedule settles every input of the suite within a dozen launches, so the safety nets never run there.  These
tests set the knobs through the sim's explicit schedule entry (tests/sim/br_sim.cc sim_compress_sched), run walks and
commits in list order, reversed and shuffled, and check for every run that
  - the bytes equal the oracle's (or, for FLUSH-cut streams, the reference's recorded stream);
  - the fixpoint is self-consistent: re-walking every chunk from its final in-state gives the same bits and commands;
  - no launch appended more chunk walks than the product's ran_list holds.
The sim is built here with BR_SIM_DEBUG, whose counters show which paths a run reached; the path tests assert that
a full sweep, a forced walker, a step-cap hit and an accepted and a refused block-boundary prediction all happened."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from brotli_libs import ROOT, TABLES, Oracle
from fuzz_cases import REGRESSIONS, cases, dict_cases

KEEP = 0xFFFFFFFF
SCHEDULED, REVERSED, SHUFFLED = 0, 1, 2
# stats words (tests/sim/br_sim.cc SIM_ST_*)
LAUNCHES, WALKS, CHUNKS, FULL_SWEEP, FORCED, STEP_CAP, PREDICT_OK, PREDICT_NO, MAX_WALKS, RAN_CAP, VERIFY_DIFF = \
    0, 1, 2, 5, 6, 7, 8, 9, 10, 11, 12
ERR_CAPACITY = -5


class Sched(C.Structure):
    _fields_ = [(f, C.c_uint32) for f in ("sweep_epoch", "force_epoch", "step_cap", "heavy_min", "pilot", "sweep_blocks",
                                          "batch_chunk_bits", "walk_order", "commit_order", "walk_seed", "commit_seed",
                                          "verify")]


def sched(**kw):
    s = Sched(*[KEEP] * 7, SCHEDULED, SCHEDULED, 0, 0, 1)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sched") / "libbrsim_sched.so")
    subprocess.check_call(["g++", "-O2", "-DBR_SIM_ENTROPY", "-DBR_SIM_DEBUG", "-fPIC", "-shared", "-std=c++17",
                           "-ffp-contract=off", "-Wno-unused-function", "-I", os.path.join(ROOT, "include"), "-o", so,
                           os.path.join(ROOT, "tests", "sim", "br_sim.cc")])
    L = C.CDLL(so)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    L.sim_compress_sched.restype = C.c_long
    L.sim_compress_sched.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                     C.c_uint32, C.POINTER(Sched), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def ora():
    return Oracle()


def run(sim, d, q, w, s, cuts=(), kinds=(), hint=0, nstreams=1):
    """the sim under schedule s: (return code, output, stats)"""
    cap = len(d) + len(d) // 2 + 4096 + 64 * nstreams
    out = C.create_string_buffer(cap)
    st = np.zeros(16, np.uint32)
    cp = np.array(cuts, np.uint32) if cuts else None
    ck = np.array(kinds, np.uint32) if cuts else None
    ends = np.zeros(nstreams + 1, np.uint64)
    r = sim.sim_compress_sched(q, w, d, len(d), cp.ctypes.data if cuts else None, ck.ctypes.data if cuts else None,
                               len(cuts), hint or len(d), C.byref(s), ends.ctypes.data, out, cap, st.ctypes.data)
    if r >= 0 and nstreams > 1:
        res, a = [], 0
        for k in range(nstreams):
            res.append(out.raw[a:int(ends[k])])
            a = int(ends[k])
        return r, res, st
    return r, (out.raw[:r] if r >= 0 else None), st


def check(sim, d, q, w, s, want, what, **kw):
    r, got, st = run(sim, d, q, w, s, **kw)
    assert r >= 0, ("sim failed", r, what)
    assert st[MAX_WALKS] <= st[RAN_CAP], ("more walks in one launch than ran_list holds", what)
    assert got == want, ("bytes differ from the oracle", what, len(got) if got else got, len(want))
    assert st[VERIFY_DIFF] == 0, ("fixpoint not self-consistent", int(st[VERIFY_DIFF]), what)
    return st


# ---------------------------------------------------------------------------------------------------------------- inputs
def _fuzz(seed, idx):
    for i, d, q, w in cases(seed, idx + 1):
        if i == idx:
            return d, q, w


def _noise(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _int32_walk(count, seed):
    rng = np.random.default_rng(seed)
    return np.cumsum(rng.integers(-3, 4, count)).astype(np.int32).tobytes()


def _short_period(n, seed):
    """a few short periods, each with sparse point mutations: buckets whose positions are mostly unstored (long copies),
    stored-bit flips that ripple from chunk to chunk (the shape of fuzz case (35, 22))"""
    rng = np.random.default_rng(seed)
    out = bytearray()
    while len(out) < n:
        per = bytes(rng.integers(0, 4, int(rng.integers(1, 7)), dtype=np.uint8))
        seg = bytearray(per * int(rng.integers(200, 4000)))
        for p in rng.integers(0, len(seg), max(1, len(seg) // 700)):
            seg[p] ^= 1
        out += seg
    return bytes(out[:n])


def _slice_inputs():
    """the regressions, a seeded slice of the fuzz generators, noise, an int32 random walk and short-period data"""
    ins = [("regression-%d-%d" % (s, i),) + _fuzz(s, i) for s, i in REGRESSIONS]
    for i, d, q, w in cases(2, 51):
        if i == 50:
            ins.append(("cases-2-50", d, q, w))
    for i, d, q, w in cases(20260101, 40):
        if q >= 5 and 2000 <= len(d) <= 80000:
            ins.append(("cases-20260101-%d" % i, d, q, w))
    for i, d, q, w in dict_cases(20260102, 6, TABLES):
        ins.append(("dict-%d" % i, d, q, w))
    ins.append(("noise", _noise(70000, 3), 5, 22))
    ins.append(("int32-walk", _int32_walk(20000, 4), 6, 22))
    ins.append(("short-period", _short_period(90000, 6), 5, 20))
    return ins


INPUTS = _slice_inputs()
QUALITIES = (5, 6, 7, 9)


def _want(ora, d, q, w, memo={}):
    k = (hash(d), len(d), q, w)
    if k not in memo:
        memo[k] = ora.compress(d, q, w)
    return memo[k]


# ------------------------------------------------------------------------------------------------------- the two findings
def test_forced_walker_within_ran_list(sim, ora):
    """The forced walker runs to its block's end through chunks other walkers of the same launch also walk; each such walk
    took another ran_list slot, past the product's nblocks + 16 (found with force_epoch 1 on 256 KiB of noise).  A chunk is
    now walked at most once per launch."""
    d = _noise(262144, 5)
    r, got, st = run(sim, d, 5, 22, sched(force_epoch=1))
    assert r != ERR_CAPACITY, "a launch appended more chunk walks than ran_list holds"
    assert r >= 0 and got == ora.compress(d, 5, 22)
    assert st[FORCED] > 0 and st[VERIFY_DIFF] == 0
    assert st[MAX_WALKS] <= st[CHUNKS], "a chunk was walked twice in one launch"


@pytest.mark.parametrize("sweep_epoch", [0, 1])
def test_forced_walker_shares_no_bitmap(sim, ora, sweep_epoch):
    """cases(2, 51)[50] at quality 5, lgwin 24, force_epoch 2: the forced walker and the scheduled walker of a later chunk
    of its block, heads of equal parity, walked that chunk in one launch into one bits_cur bitmap.  Each read the other's
    fresh bits as its own, the commit stored their union, and the fixpoint settled after 3 launches on bits no walk had
    produced (37191 bytes instead of 37121; chunks 2..8 not self-consistent)."""
    d, q, w = _fuzz(2, 50)
    assert (len(d), q, w) == (68742, 5, 24)
    st = check(sim, d, 5, 24, sched(sweep_epoch=sweep_epoch, force_epoch=2), _want(ora, d, 5, 24), "cases(2, 51)[50]")
    assert st[FORCED] > 0


@pytest.mark.parametrize("sweep_epoch", [KEEP, 0], ids=["default", "sweep0"])
def test_marking_gap_without_heavy_buckets(sim, ora, sweep_epoch):
    """fuzz case (35, 22) with the counter-wrap path of heavy buckets switched off (heavy_min beyond any bucket): that path
    re-walks chunks whenever heavy buckets flip and so hides a marking rule that ignores the runs' own fresh bits
    (br_commit_bits: a shield must be stored before the launch and in the covering run, prev && (!cov || cur))"""
    d, q, w = _fuzz(35, 22)
    check(sim, d, q, w, sched(heavy_min=0xFFFFFFFE, sweep_epoch=sweep_epoch), _want(ora, d, q, w), "(35, 22) heavy off")


# ------------------------------------------------------------------------------------------------------------ the matrix
SCHEDULES = [("default", {})] + \
    [("force%d-sweep%d" % (f, s), dict(force_epoch=f, sweep_epoch=s)) for f in (0, 1, 2, 3) for s in (0, 1, 3)] + \
    [("stepcap%d" % c, dict(step_cap=c)) for c in (0, 1, 16)] + \
    [("heavy%d" % h, dict(heavy_min=h)) for h in (2, 16)] + \
    [("sweepblocks%d" % b, dict(sweep_blocks=b)) for b in (1, 32)]


# the regressions of 200 KB and more take seconds each in the sim: they run under these schedules only
LARGE_SCHEDULES = ("default", "force1-sweep0", "force2-sweep0", "force2-sweep1")


@pytest.mark.parametrize("name,knobs", SCHEDULES, ids=[s[0] for s in SCHEDULES])
def test_schedule_matrix(sim, ora, name, knobs):
    """every input of the slice at its own quality, and the generic inputs at every quality of the marking path"""
    for label, d, q, w in INPUTS:
        if len(d) > 200000 and name not in LARGE_SCHEDULES:
            continue
        qs = QUALITIES if label in ("noise", "int32-walk", "short-period") else (q,)
        for qq in qs:
            check(sim, d, qq, w, sched(**knobs), _want(ora, d, qq, w), (name, label, qq, w))


def test_sweep_blocks_not_a_power_of_two(sim):
    """sweep_blocks must be a power of two (BrParams::sweep_blocks): the sim refuses any other value, as the product's
    br_debug_compress_sched does"""
    d = _noise(20000, 11)
    for b in (0, 3, 24):
        r, _, _ = run(sim, d, 5, 22, sched(sweep_blocks=b))
        assert r < 0, b


def test_jacobi_only(sim, ora):
    """sweep_epoch beyond any launch: no sweep ever, every dirty chunk walked on its own until the fixpoint (the forced
    walker still ends it)"""
    for label, d, q, w in INPUTS:
        if len(d) <= 70000:
            check(sim, d, q, w, sched(sweep_epoch=1 << 20), _want(ora, d, q, w), ("jacobi", label))


ORDERS = [("reversed", REVERSED, 0)] + [("shuffle%d" % k, SHUFFLED, 1000 + k) for k in range(3)]


@pytest.mark.parametrize("force", [KEEP, 1], ids=["default", "force1"])
@pytest.mark.parametrize("oname,order,seed", ORDERS, ids=[o[0] for o in ORDERS])
def test_walk_and_commit_orders(sim, ora, oname, order, seed, force):
    """a launch's walks and commits in another order (on the GPU they are concurrent), at qualities 2..9"""
    ins = [x for x in INPUTS if x[0] in ("regression-7-249", "regression-5-297", "cases-2-50", "dict-3", "noise", "short-period")]
    for label, d, q, w in ins:
        for qq in ((q,) if label.startswith(("regression", "cases")) else (2, 3, 4, 5, 7)):
            for walk_order, commit_order in ((order, SCHEDULED), (SCHEDULED, order), (order, order)):
                s = sched(force_epoch=force, walk_order=walk_order, commit_order=commit_order, walk_seed=seed,
                          commit_seed=seed + 7)
                check(sim, d, qq, w, s, _want(ora, d, qq, w), (oname, force, label, qq, walk_order, commit_order))


@pytest.mark.parametrize("q", [2, 3, 4])
def test_quick_qualities_forced(sim, ora, q):
    """qualities 2..4 check every run against the committed bits (br_verify_run) instead of marking: the forced walker and
    early sweeps must not change that"""
    for label, d, _, w in [x for x in INPUTS if x[0] in ("regression-7-13", "cases-2-50", "noise", "short-period")]:
        for f, s in ((0, 0), (1, 1), (2, 0), (KEEP, KEEP)):
            check(sim, d, q, w, sched(force_epoch=f, sweep_epoch=s), _want(ora, d, q, w), (label, q, f, s))


def test_pilot_forced_on_at_quality_5(sim, ora):
    for label, d, q, w in [x for x in INPUTS if x[0] in ("cases-2-50", "noise", "short-period", "regression-6-104")]:
        for knobs in (dict(pilot=1), dict(pilot=1, force_epoch=1)):
            check(sim, d, 5, w, sched(**knobs), _want(ora, d, 5, w), (label, knobs))


def test_pilot_on_a_large_stream(sim, ora):
    """the pilot launch of a 1 MiB+ stream at quality 7..9 (its default there), on and off, with early safety nets"""
    from corpus import synth_web
    d = synth_web(1_150_000, 31)
    for q in (7, 9):
        want = _want(ora, d, q, 22)
        for knobs in (dict(), dict(pilot=0), dict(pilot=1, force_epoch=1, sweep_epoch=0)):
            check(sim, d, q, 22, sched(**knobs), want, (q, knobs))


def test_flush_cut_stream(sim):
    """a FLUSH one or two bytes behind a block boundary (a block too short to stitch), against the reference's recorded
    stream, under the safety nets and reordered commits"""
    from brotli_libs import RecordedRef, ref_stream_ops
    from corpus import synth_text
    ref = RecordedRef()
    d = synth_text(200000, 77)
    n = len(d)
    for q, w in ((5, 22), (7, 17), (3, 12)):
        bs = 1 << (14 if q < 4 else 16)
        for extra in (1, 2):
            c = 2 * bs + extra
            want = ref_stream_ops(ref, d, q, w, [c, n - c], [1, 2])
            for knobs in (dict(), dict(force_epoch=1, sweep_epoch=0), dict(force_epoch=2, commit_order=REVERSED),
                          dict(step_cap=0, walk_order=SHUFFLED, walk_seed=5)):
                r, got, st = run(sim, d, q, w, sched(**knobs), cuts=[c], kinds=[1], hint=c)
                assert r >= 0 and got == want, (q, w, extra, knobs)
                assert st[VERIFY_DIFF] == 0 and st[MAX_WALKS] <= st[RAN_CAP]


@pytest.mark.parametrize("chunk_bits", [9, 11])
def test_batch_of_three_streams(sim, ora, chunk_bits):
    """a three-stream batch (cuts of kind 3) at both chunk sizes, every stream as the oracle compresses it alone"""
    d0, _, _ = _fuzz(2, 50)
    streams = [d0[:60000], _noise(30000, 9), _short_period(50000, 10)]
    d = b"".join(streams)
    bounds = list(np.cumsum([len(x) for x in streams])[:-1])
    for q, w in ((5, 22), (9, 18), (3, 20)):
        want = [ora.compress(x, q, w) for x in streams]
        for knobs in (dict(), dict(force_epoch=1), dict(force_epoch=2, sweep_epoch=0, commit_order=SHUFFLED, commit_seed=3),
                      dict(step_cap=1, walk_order=REVERSED)):
            r, got, st = run(sim, d, q, w, sched(batch_chunk_bits=chunk_bits, **knobs), cuts=bounds, kinds=[3, 3],
                             hint=max(len(x) for x in streams), nstreams=3)
            assert r >= 0 and got == want, (q, w, chunk_bits, knobs)
            assert st[VERIFY_DIFF] == 0 and st[MAX_WALKS] <= st[RAN_CAP]


# ------------------------------------------------------------------------------------------------------ paths reached
def test_paths_reached(sim, ora):
    """each safety net and each branch of the block-boundary prediction runs in some case of this file"""
    tot = np.zeros(16, np.int64)
    runs = [
        ("short-period", dict(step_cap=0, sweep_epoch=0)),
        ("noise", dict(force_epoch=1)),
        ("int32-walk", dict(step_cap=1)),
        ("regression-5-297", dict(sweep_epoch=0)),
        ("dict-3", dict()),   # (17 launches under the default schedule: full sweeps at launches 12 and 15)
        # sweeps from the first launch, walked last chunk first: a block's last chunk reaches the boundary while the chunks
        # in front of it have no records yet, which the prediction refuses
        ("noise", dict(sweep_epoch=0, walk_order=REVERSED)),
        ("cases-2-50", dict(sweep_epoch=0, walk_order=REVERSED)),
    ]
    by = {x[0]: x for x in INPUTS}
    for label, knobs in runs:
        _, d, q, w = by[label]
        tot += check(sim, d, q, w, sched(**knobs), _want(ora, d, q, w), (label, knobs)).astype(np.int64)
    assert tot[FULL_SWEEP] > 0, "no full-sweep launch"
    assert tot[FORCED] > 0, "no forced launch"
    assert tot[STEP_CAP] > 0, "no step-cap hit"
    assert tot[PREDICT_OK] > 0, "no sweep crossed a block boundary"
    assert tot[PREDICT_NO] > 0, "no block-boundary prediction refused"
