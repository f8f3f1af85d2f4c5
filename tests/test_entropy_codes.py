"""The prefix codes of a job (E4 in br_entropy2.h): built and stored by one warp per code when the job has at most
BR_CODE_WARP_MAX (8 192) of them, else by one thread per code, with the metablock headers written in between.

CPU: the device code run on the CPU (tests/sim, which takes the warp workers' functions) equals the oracle for inputs in
which stored-raw metablocks lie between compressed ones (they have no codes).
GPU (-m gpu): the same inputs through BrotliEncoderCompress, and batch jobs of thousands of tiny streams through
BrotliB200CompressBatch, whose codes outnumber what the warps take, so the thread workers build and store them.  The late
uncompressed fallback (encode.c:604), which runs the entropy stage a second time on the same job, is covered by
test_zz_gpu_q234.py at quality 4 and by the batch tests of test_gpu_parity.py."""
import ctypes as C
import os

import numpy as np
import pytest

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
    """8 192 tiny streams, one device job (br_api.cc kBatchGroupStreams): over 24 000 codes for the thread workers."""
    items = _tiny_streams(8192, 920 + q)
    got = b200.compress_batch(items, q, 22, threads=4)
    for k, x in enumerate(items):
        assert got[k] == oracle.compress(x, q, 22), k
