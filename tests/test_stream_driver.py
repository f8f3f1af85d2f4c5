"""CPU suite: the C API's host driver (brotli_b200/csrc/br_driver.h) -- parameters, the one-shot wrapper's rules, the
grouping of batches and the streaming state machine -- run by tests/sim/br_sim.cc over the device code compiled for the
host, against the reference's CompressStream for the same calls (recorded results) and the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from brotli_libs import ROOT, TABLES, Oracle, RecordedRef, ref_stream_ops

SIM_SO = os.path.join(ROOT, "tests", "sim", "libbrsim.so")
FINISH = 2                      # BrotliEncoderOperation


@pytest.fixture(scope="module")
def sim():
    if not os.path.exists(SIM_SO):
        import __graft_entry__
        __graft_entry__.build_checkers()
    L = C.CDLL(SIM_SO)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    L.sim_stream_ops.restype = C.c_long
    L.sim_stream_ops.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_void_p, C.c_void_p,
                                 C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t]
    L.sim_compress_oneshot.restype = C.c_int
    L.sim_compress_oneshot.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
    L.sim_plan_groups.restype = C.c_size_t
    L.sim_plan_groups.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    L.sim_compress.restype = C.c_long
    L.sim_compress.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
    L.sim_q1_compress.restype = C.c_long
    L.sim_q1_compress.argtypes = [C.c_int, C.c_char_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    return L


def stream_ops(sim, d, q, w, sizes, ops, params=None, q1_segment_bytes=0):
    """The (size, op) calls of brotli_libs.ref_stream_ops through the driver's CompressStream; returns the stream."""
    prm = sorted((params or {}).items())
    ids = (C.c_uint32 * max(1, len(prm)))(*[k for k, v in prm])
    vals = (C.c_uint32 * max(1, len(prm)))(*[v for k, v in prm])
    sz = (C.c_size_t * len(sizes))(*sizes)
    op = (C.c_int * len(ops))(*ops)
    cap = 2 * len(d) + 100000
    out = C.create_string_buffer(cap)
    r = sim.sim_stream_ops(q, w, ids, vals, len(prm), d, sz, op, len(ops), q1_segment_bytes, out, cap)
    assert r >= 0, (q, w, sizes, ops, r)
    return out.raw[:r]


def test_driver_flush_cuts_and_parameters(sim):
    """The input cut by FLUSH operations (encode.c:1356, :1700), the size hint frozen at the first EncodeData (encode.c:1619),
    FINISH arriving without input behind a full block (encode.c:520), and BROTLI_PARAM_LGBLOCK /
    DISABLE_LITERAL_CONTEXT_MODELING, against the reference's CompressStream driven with the same calls."""
    from corpus import synth_binary, synth_text, synth_web
    ref = RecordedRef()
    for d in (synth_text(400000, 3), synth_binary(600000, 5)):
        n = len(d)
        for q, w in ((5, 22), (9, 24), (7, 19)):
            bs = 1 << (18 if (q >= 9 and w >= 18) else 16)
            for sizes, ops in (([100000, 50000, n - 150000], [0, 1, 2]), ([bs, 0, n - bs, 0], [0, 1, 1, 2]), ([100, n - 100, 0], [1, 0, 2])):
                assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, sizes, ops)
    # quality 7..9 above 1 MiB: the pilot launch (BrParams::pilot) with the input cut by FLUSH, incl. a first block of 2 bytes
    d = synth_web(1_400_000, 3)
    for q, w in ((9, 24), (7, 18)):
        for sizes, ops in (([500000, 0, 900000, 0], [1, 1, 0, 2]), ([2, 700000, 699998], [1, 1, 2])):
            assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, sizes)
    d = synth_web(2 * 262144, 9)
    for q, w in ((5, 22), (9, 24)):
        sizes, ops = [len(d), 0], [0, 2]                                  # FINISH without input behind full blocks
        assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w)
        for lgb, dis in ((0, 1), (17, 0), (20, 1), (24, 0)):
            prm = {}
            if lgb:
                prm[3] = lgb
            if dis:
                prm[4] = 1
            want = ref_stream_ops(ref, d, q, w, [len(d)], [2], params=prm)
            assert stream_ops(sim, d, q, w, [len(d)], [2], params=prm) == want, (q, w, lgb, dis)


def test_driver_q234_flush_cuts(sim):
    """Qualities 2..4 with the input cut by FLUSH operations: input blocks of 1 << 14 bytes below quality 4 (quality.h:81),
    the MAX_NUM_DELAYED_SYMBOLS flush rule (encode.c:1152), FINISH without input behind a full block."""
    from corpus import synth_binary, synth_text
    ref = RecordedRef()
    for d in (synth_text(300000, 3), synth_binary(400000, 5)):
        n = len(d)
        for q, w in ((2, 22), (3, 18), (4, 22), (4, 12)):
            bs = 1 << (14 if q < 4 else 16)
            for sizes, ops in (([100000, 50000, n - 150000], [0, 1, 2]), ([bs, 0, n - bs, 0], [0, 1, 1, 2]), ([100, n - 100, 0], [1, 0, 2])):
                assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, sizes, ops)
    d = synth_text(4 * 65536, 9)
    for q, w in ((2, 22), (3, 22), (4, 22)):
        sizes, ops = [len(d), 0], [0, 2]                                  # FINISH without input behind full blocks
        assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w)
    # an empty stream, and a FLUSH and metadata before any input: the driver writes the window bits, of the window
    # sanitised to 10 when lgwin is below (quality.h:60)
    d = synth_text(20000, 9)
    for q, w in ((2, 9), (3, 5), (4, 10)):
        for sizes, ops in (([0], [2]), ([0, 4, len(d) - 4], [1, 3, 2])):
            assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, sizes, ops)


def test_driver_flush_just_behind_a_block_boundary(sim):
    """A FLUSH one or two bytes (up to HashTypeLength - 2) behind a block boundary leaves an input block too short to stitch
    (hash_longest_match_quickly_inc.h:119 / hash_longest_match64_inc.h:127: num_bytes >= HashTypeLength - 1); the block behind
    it stitches instead, and its three positions reach back across the short block into the block in front.  Their owner must
    still commit them (br_commit_bits; found by a randomized FLUSH campaign: q3, lgwin 12, flush at 14 * 16384 + 2)."""
    from corpus import synth_text
    ref = RecordedRef()
    d = synth_text(200000, 77)
    n = len(d)
    for q, w in ((3, 12), (2, 22), (4, 16), (5, 22), (7, 17)):
        bs = 1 << (14 if q < 4 else 16)
        for extra in (1, 2, 3, 5, 6):
            c = 2 * bs + extra
            sizes, ops = [c, n - c], [1, 2]
            assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, extra)
        c1, c2 = bs + 1, bs + 2                                    # two short blocks in a row
        sizes, ops = [c1, 1, n - c2], [1, 1, 2]
        assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w)


def test_driver_stream_offset(sim):
    """BROTLI_PARAM_STREAM_OFFSET (encode.h:231, the sanctioned way to stitch shards into one stream, SURVEY.md 8e): no
    window bits, poisoned distance cache (encode.c:656), dictionary distances counted from the virtual start
    (backward_references_inc.h:94), and the first two bytes flushed on their own (encode.c:1704) -- against the reference."""
    from corpus import synth_text, synth_web
    ref = RecordedRef()
    for d in (synth_text(300000, 4), synth_web(500000, 10)):
        for q, w in ((5, 22), (9, 24), (6, 18)):
            for off in (1, 1000, 1 << 20, 1 << 30):
                want = ref_stream_ops(ref, d, q, w, [len(d)], [2], params={9: off})
                got = stream_ops(sim, d, q, w, [len(d)], [2], params={9: off})
                assert got == want, (q, w, off, len(got), len(want))


def test_driver_flush_and_metadata(sim):
    """EMIT_METADATA (encode.c:1549) and FLUSH at quality 5..9: a flush / metadata before any input, metadata between data,
    empty metadata, repeated operations at one position, FINISH without input behind a full block -- the call sequences of
    test_gpu_parity.py::test_streaming_flush_and_metadata, against the reference.  The output is drained by calling again
    with the same operation, so a metadata block must stay open until its bytes are out."""
    from corpus import synth_binary, synth_text
    ref = RecordedRef()
    for d, q, w in ((synth_text(700000, 61), 5, 22), (synth_binary(900000, 62), 5, 22), (synth_text(700000, 61), 9, 24),
                    (synth_binary(900000, 62), 6, 18)):
        n = len(d)
        bs = 1 << (18 if q >= 9 else 16)
        seqs = [
            ([100000, 50000, 250000, n - 400000], [0, 1, 1, 2]),
            ([0, 300000, 0, n - 300000, 0], [1, 1, 1, 1, 2]),
            ([bs, 0, n - bs], [0, 1, 2]),
            ([2 * bs, 0], [0, 2]),
            ([7, 200000, 5, n - 200012, 0], [3, 0, 3, 1, 2]),          # metadata first (payload = the input bytes), between data
            ([0, 100, 0, 0, 11, n - 111], [3, 1, 3, 1, 3, 2]),        # empty metadata, repeated operations at one position
        ]
        for sizes, ops in seqs:
            assert stream_ops(sim, d, q, w, sizes, ops) == ref_stream_ops(ref, d, q, w, sizes, ops), (q, w, sizes, ops)


def test_driver_q1_flush_segments(sim):
    """FLUSH at quality 1: the stream is a chain of byte-aligned segments (window bits only in the first, byte padding behind
    every flushed one) == the oracle for the whole op sequence."""
    from corpus import synth_web
    d = synth_web(500000, 42)
    ora = Oracle()
    cases = [([0, 500000], [1, 2]), ([100000, 0, 400000, 0], [1, 1, 1, 2]), ([1, 2, 3, 499994], [1, 1, 0, 2]),
             ([200000, 150000, 150000], [0, 1, 2]), ([250000, 250000, 0], [1, 1, 2])]
    for sizes, ops in cases:
        for w in (16, 22):
            assert stream_ops(sim, d, 1, w, sizes, ops) == ora.compress_q1_stream(d, w, sizes, ops), (sizes, ops, w)


def test_driver_q1_small_segments(sim):
    """Quality 1 with segments of one fragment (1 << lgwin bytes): every PROCESS call of more than half a segment runs
    segments, a call is split inside at fragment multiples, and most segments end mid-byte with the next one starting
    behind their pending bits (br_driver.h q1_run / q1_segment) == the oracle for the op sequence.  A smaller segment
    cannot hold a fragment and fails."""
    from corpus import synth_web
    d = synth_web(400000, 7) + bytes(np.random.default_rng(5).integers(0, 256, 70000, dtype=np.uint8))
    ora = Oracle()
    cases = [([100000, 200000, 170000], [0, 0, 2]), ([1, 65536, 70000, 334463], [0, 0, 1, 2]),
             ([300000, 100000, 70000, 0], [0, 0, 0, 2]), ([131072, 131072, 207856], [0, 1, 2]), ([470000], [2]),
             ([100000, 0, 370000, 0], [1, 1, 1, 2])]
    for sizes, ops in cases:
        for w in (16, 18):
            want = ora.compress_q1_stream(d, w, sizes, ops)
            assert stream_ops(sim, d, 1, w, sizes, ops, q1_segment_bytes=1 << w) == want, (sizes, ops, w)
    sz = (C.c_size_t * 1)(len(d))
    op = (C.c_int * 1)(FINISH)
    out = C.create_string_buffer(2 * len(d))
    assert sim.sim_stream_ops(1, 18, None, None, 0, d, sz, op, 1, (1 << 18) - 1, out, len(out)) == -1


def test_driver_batch_groups(sim):
    """plan_groups at its limits: at most 8 192 streams and 128 MiB per group, in order; empty streams and streams of 1 MiB
    or more go one by one."""
    def plan(sizes):
        arr = np.array(sizes, np.uint64)
        group_of = np.zeros(len(sizes), np.int64)
        ng = sim.sim_plan_groups(arr.ctypes.data, len(sizes), group_of.ctypes.data)
        return ng, group_of.tolist()

    assert plan([1] * 8192) == (1, [0] * 8192)
    assert plan([1] * 8193) == (2, [0] * 8192 + [1])
    mib = 1 << 20
    # 128 streams just below 1 MiB fill 128 MiB - 128 bytes; the next one opens a new group, and 128 bytes more still fit
    ng, g = plan([mib - 1] * 128 + [mib - 1, 128])
    assert ng == 2 and g == [0] * 128 + [1, 1]
    ng, g = plan([mib - 1] * 128 + [128, mib - 1])
    assert ng == 2 and g == [0] * 129 + [1]
    # empty and long streams go one by one; the group continues across them
    ng, g = plan([5, 0, mib, 7, mib - 1, 3 * mib, 0])
    assert ng == 1 and g == [0, -1, -1, 0, 0, -1, -1]
    assert plan([]) == (0, [])


def test_driver_oneshot_wrapper_rules(sim):
    """BrotliEncoderCompress's rules around the encoder (encode.c:1296-1353): a stream longer than
    BrotliEncoderMaxCompressedSize is replaced by the raw stream, a buffer below that bound then fails with size 0, and
    empty input is the one-byte empty stream."""
    ora = Oracle()
    noise = np.random.RandomState(67).randint(0, 256, 300000, dtype=np.uint8).tobytes()
    bound = len(noise) + 4 * (len(noise) >> 14) + 6
    cap = 2 * len(noise) + 100000
    out = C.create_string_buffer(cap)
    assert sim.sim_q1_compress(10, noise, len(noise), None, 0, out, cap) > bound     # a metablock header per 1 KiB fragment

    def oneshot(d, q, w, cap):
        buf = C.create_string_buffer(max(1, cap))
        n = C.c_size_t(cap)
        ok = sim.sim_compress_oneshot(q, w, d, len(d), C.byref(n), buf)
        return ok, buf.raw[:n.value]

    ok, got = oneshot(noise, 1, 10, cap)
    assert ok == 1 and got[:2] == b"\x21\x03" and len(got) == len(noise) + 6 and got == ora.compress(noise, 1, 10)
    assert oneshot(noise, 1, 10, bound) == (1, got)
    assert oneshot(noise, 1, 10, bound - 1) == (0, b"")
    d = noise[:1000] * 200
    ok, got = oneshot(d, 5, 22, cap)
    assert ok == 1 and got == ora.compress(d, 5, 22)
    assert oneshot(d, 5, 22, len(got) - 1) == (0, b"")                  # compressed, but the buffer is too small
    assert oneshot(b"", 5, 22, 1) == (1, b"\x06")
    assert oneshot(d, 1, 27, cap) == (1, ora.compress(d, 1, 24))        # quality 1: lgwin above 24 is sanitised to 24
    assert oneshot(d, 5, 25, cap) == (0, b"")                           # quality 5: it asks for the large window
