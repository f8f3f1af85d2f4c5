"""The entropy stage at its limits (tests/entropy_cases.py: prefix-code depth limits, the block-type cap, simple prefix
codes, count smoothing and code-length runs, the longest insert / block-length / distance codes), and the fuzz corpora
the GPU tests compare against the oracle.

CPU: every case reaches the branch it was built for (the oracle's edge counters); the oracle equals the reference
(recorded results, brotli_libs.RecordedRef) and the reference decoder round-trips it; the device code run on the CPU
(tests/sim) equals the oracle, one stream at a time and as batch jobs.  The oracle equals the reference on the fuzz
inputs of tests/test_gpu_parity.py and tests/test_zz_gpu_q234.py at the qualities and windows used there, so what those
tests trust is pinned to the reference.
GPU (-m gpu): every case through BrotliEncoderCompress, through the batch call below and above the 8 MiB point where
the batch chunk size changes, and the block-type-cap and Fibonacci cases through BrotliB200CompressDevice."""
import collections
import ctypes as C
import os

import numpy as np
import pytest

import entropy_cases
from brotli_libs import ROOT, TABLES, Oracle, RecordedRef

CASES = entropy_cases.cases()
IDS = [c[0] for c in CASES]
SIM_SO = os.path.join(ROOT, "tests", "sim", "libbrsim.so")
BATCH_LIMIT = 1 << 20            # streams below 1 MiB take the batch path (br_driver.h)


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


@pytest.fixture(scope="module")
def ref():
    return RecordedRef()


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_case_reaches_its_branch(oracle, case):
    label, d, q, w = case
    oracle.edge_stats_reset()
    oracle.compress(d, q, w)
    st = oracle.edge_stats()
    for k, least in entropy_cases.expect(label).items():
        assert st[k] >= least, (label, k, st[k], least)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_against_reference(oracle, ref, case):
    label, d, q, w = case
    want = ref.compress(d, q, w)
    assert oracle.compress(d, q, w) == want, label
    assert ref.decompress(want, len(d)) == d, label


@pytest.fixture(scope="module")
def sim():
    if not os.path.exists(SIM_SO):
        import __graft_entry__
        __graft_entry__.build_checkers()
    L = C.CDLL(SIM_SO)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    L.sim_compress.restype = C.c_long
    L.sim_compress.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
    L.sim_compress_multi.restype = C.c_long
    L.sim_compress_multi.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                     C.c_size_t, C.c_void_p]
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    return L


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_sim_against_oracle(sim, oracle, case):
    label, d, q, w = case
    cap = 2 * len(d) + 100000
    out = C.create_string_buffer(cap)
    st = np.zeros(8, np.uint32)
    r = sim.sim_compress(q, w, d, len(d), out, cap, st.ctypes.data)
    assert r >= 0 and out.raw[:r] == oracle.compress(d, q, w), label


def _groups():
    """The cases below 1 MiB by (quality, lgwin)."""
    g = collections.defaultdict(list)
    for label, d, q, w in CASES:
        if len(d) < BATCH_LIMIT:
            g[(q, w)].append((label, d))
    return sorted(g.items())


def test_sim_batch_against_oracle(sim, oracle):
    """The cases below 1 MiB of one (quality, lgwin) as one batch job (cuts of kind 3), both chunk sizes."""
    for (q, w), items in _groups():
        if len(items) < 2:           # (one stream is not a batch job)
            continue
        d = b"".join(x for _, x in items)
        bounds = np.cumsum([len(x) for _, x in items]).astype(np.uint32)
        for bits in ("9", "11"):
            os.environ["BR_SIM_BATCH_CHUNK_BITS"] = bits
            try:
                ends = np.zeros(len(items) + 1, np.uint64)
                cap = 2 * len(d) + 4096 + 64 * len(items)
                out = C.create_string_buffer(cap)
                st = np.zeros(8, np.uint32)
                r = sim.sim_compress_multi(q, w, d, len(d), bounds.ctypes.data, len(items), ends.ctypes.data, out, cap,
                                           st.ctypes.data)
            finally:
                os.environ.pop("BR_SIM_BATCH_CHUNK_BITS", None)
            assert r >= 0 and int(ends[len(items) - 1]) == r
            a = 0
            for k, (label, x) in enumerate(items):
                assert out.raw[a:int(ends[k])] == oracle.compress(x, q, w), (label, bits)
                a = int(ends[k])


def _fuzz_calls():
    """(name, data, quality, lgwin) of every oracle comparison the GPU fuzz tests make (test_gpu_parity.py::test_fuzz_gpu,
    test_zz_gpu_q234.py::test_q234_fuzz_gpu, one-shot and batch)."""
    from fuzz_cases import REGRESSIONS, cases, dict_cases
    calls = []
    by_seed = collections.defaultdict(set)
    for seed, idx in REGRESSIONS:
        by_seed[seed].add(idx)
    for seed, idxs in sorted(by_seed.items()):
        calls += [("regression %d/%d" % (seed, i), d, q, w) for i, d, q, w in cases(seed, max(idxs) + 1) if i in idxs]
    calls += [("31337/%d" % i, d, q, w) for i, d, q, w in cases(31337, 250)]
    todo = [(i, d) for i, d, q, w in cases(31339, 200) if d] + [(1000 + i, d) for i, d, q, w in dict_cases(31340, 40, TABLES) if d]
    calls += [("q234 %d" % i, d, 2 + i % 3, 10 + (i * 7) % 15) for i, d in todo]
    small = [d for i, d in todo if len(d) < BATCH_LIMIT]
    for a in range(0, len(small), 12):
        q, w = 2 + (a // 12) % 3, 10 + (a // 12 * 5) % 15
        calls += [("q234 batch %d+%d" % (a, k), x, q, w) for k, x in enumerate(small[a:a + 12])]
    return calls


def test_oracle_against_reference_on_fuzz_corpora(oracle, ref):
    """The fuzz inputs the GPU tests check against the oracle, oracle against the reference at the same settings."""
    seen = set()
    for name, d, q, w in _fuzz_calls():
        if not d or (q, w, d) in seen:
            continue
        seen.add((q, w, d))
        assert oracle.compress(d, q, w) == ref.compress(d, q, w), (name, len(d), q, w)


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def b200():
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    return brotli_b200


@pytest.mark.gpu
def test_gpu_oneshot_against_reference(b200, ref):
    bad = [label for label, d, q, w in CASES if b200.compress_oneshot(d, q, w) != ref.compress(d, q, w)]
    assert not bad, bad


@pytest.mark.gpu
def test_gpu_batch_against_reference(b200, ref):
    """All cases below 1 MiB of one (quality, lgwin) through one batch call: as they are (less than 8 MiB in all, 512-byte
    chunks) and repeated past 8 MiB (2 KiB chunks, br_params.h br_batch_chunk_bits) where that takes at most 2048
    streams (each has its own entropy scratch on the device)."""
    above = 0
    for (q, w), items in _groups():
        want = [ref.compress(x, q, w) for _, x in items]
        total = sum(len(x) for _, x in items)
        assert total < (8 << 20)
        reps = (8 << 20) // total + 1
        above += reps * len(items) <= 2048
        for r in (1, reps) if reps * len(items) <= 2048 else (1,):
            got = b200.compress_batch([x for _, x in items] * r, q, w, threads=4)
            bad = [(items[k % len(items)][0], k) for k, g in enumerate(got) if g != want[k % len(items)]]
            assert not bad, (q, w, r, bad)
    assert above >= 15


@pytest.mark.gpu
def test_gpu_device_api_against_reference(b200, ref):
    import torch
    L = b200.lib()
    for label, d, q, w in CASES:
        if not label.startswith(("many_dialects", "fib_")):
            continue
        t = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
        out = torch.empty(len(d) + (len(d) >> 3) + 4096, dtype=torch.uint8, device="cuda")
        sz = C.c_size_t(out.numel())
        assert L.BrotliB200CompressDevice(q, w, len(d), t.data_ptr(), C.byref(sz), out.data_ptr()), label
        assert bytes(out[:sz.value].cpu().numpy().tobytes()) == ref.compress(d, q, w), label
