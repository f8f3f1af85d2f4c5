"""The position index and the stored-bit snapshot.

GPU (-m gpu): br_debug_index builds the index with the pipeline's own host function (br_build_index) and returns S, rank,
seg and the sorted keys; they must equal a numpy stable sort of the keys.  The sizes straddle the radix tile (8192) and the
switch from the 4-byte to the 8-byte hash at 1 MiB; all-zero input puts every position into one bucket, so one digit fills
every tile.

CPU: the sim's LZ77 fixpoint (tests/sim/snapshot_check.cc) runs br_snapshot_update after every launch's commits, as the
pipeline does, and compares the snapshot it keeps with one gathered from scratch (sim_build_storedS) before every launch."""
import ctypes as C
import os

import numpy as np
import pytest

from brotli_libs import ROOT, TABLES
from corpus import synth_binary, synth_text, synth_web

TILE = 8192
SIZES = [1, 7, TILE - 1, TILE, TILE + 1, 3 * TILE + 1234, (1 << 20) - 1, 1 << 20]


def _input(kind, n):
    if kind == "text":
        return synth_text(n, seed=11)
    if kind == "web":
        return synth_web(n, seed=12)
    if kind == "binary":
        return synth_binary(n, seed=13)
    if kind == "noise":
        return np.random.RandomState(14).randint(0, 256, n, dtype=np.uint8).tobytes()
    return bytes(n)


def _bucket_keys(d, q, w):
    """the bucket key of every position at qualities 5..9 (br_lz77.h br_hash_key; as tools/gpu_check.py computes it)"""
    n = len(d)
    a = np.frombuffer(d + bytes(16), np.uint8)
    with np.errstate(over="ignore"):
        if n >= (1 << 20) and w >= 19:
            v = np.zeros(n, np.uint64)
            for i in range(8):
                v |= a[i:i + n].astype(np.uint64) << np.uint64(8 * i)
            mul = np.uint64((0x1FE35A7BD3579BD3 << 24) & 0xFFFFFFFFFFFFFFFF)
            key = ((v * mul) >> np.uint64(49)).astype(np.uint32)
            htl, nb = 8, 1 << 15
        else:
            v = np.zeros(n, np.uint32)
            for i in range(4):
                v |= a[i:i + n].astype(np.uint32) << np.uint32(8 * i)
            bb = 14 if q < 7 else 15
            key = ((v * np.uint32(0x1E35A7BD)) >> np.uint32(32 - bb)).astype(np.uint32)
            htl, nb = 4, 1 << bb
    key[max(0, n - htl + 1):] = nb
    return key, nb


def _gpu_index(L, d, q, w, nb):
    n = len(d)
    S = np.zeros(n, np.uint32); rank = np.zeros(n, np.uint32); keys = np.zeros(n, np.uint32)
    seg = np.zeros(nb + 2, np.uint32)
    assert L.br_debug_index(q, w, d, n, S.ctypes.data, seg.ctypes.data, rank.ctypes.data, keys.ctypes.data), (q, n)
    return S, seg, rank, keys


def _check(S, seg, rank, keys, want_S, want_seg, want_keys, ctx):
    n = len(want_S)
    assert np.array_equal(S, want_S), (ctx, int(np.argmax(S != want_S)))
    assert np.array_equal(seg, want_seg), ctx
    assert np.array_equal(keys, want_keys), ctx
    want_rank = np.empty(n, np.uint32); want_rank[want_S] = np.arange(n, dtype=np.uint32)
    assert np.array_equal(rank, want_rank), (ctx, int(np.argmax(rank != want_rank)))


@pytest.fixture(scope="module")
def lib():
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    L = brotli_b200.lib()
    L.br_debug_index.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32] + [C.c_void_p] * 4
    return L


def _check_q5_9(L, kind, n, q, w=22):
    d = _input(kind, n)
    key, nb = _bucket_keys(d, q, w)
    want_S = np.argsort(key, kind="stable").astype(np.uint32)
    want_seg = np.searchsorted(key[want_S], np.arange(nb + 2), side="left").astype(np.uint32)
    _check(*_gpu_index(L, d, q, w, nb), want_S, want_seg, key[want_S], (kind, n, q))


@pytest.mark.gpu
@pytest.mark.parametrize("q", [5, 6, 7, 9])
@pytest.mark.parametrize("kind", ["text", "web", "binary", "noise", "zeros"])
def test_index_matches_stable_sort(lib, kind, q):
    for n in SIZES:
        _check_q5_9(lib, kind, n, q)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["text", "web", "binary", "noise", "zeros"])
def test_index_large(lib, kind):
    """48 MiB + 5: thousands of tiles, and the 8-byte hash every quality 5..9 uses at this size"""
    _check_q5_9(lib, kind, (48 << 20) + 5, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [2, 3, 4])
@pytest.mark.parametrize("kind", ["text", "web", "binary", "noise", "zeros"])
def test_index_q234_three_passes(lib, kind, q):
    """the slot-sorted index of qualities 2..4: 32-bit keys, three passes, rank = r3[r2[inv1]]"""
    from slot_index import slot_index
    for n in SIZES + [(48 << 20) + 5] * (kind in ("text", "zeros") and q == 4):
        d = _input(kind, n)
        want_S, want_seg, bits = slot_index(d, q)
        want_keys = np.repeat(np.arange((1 << bits) + 1, dtype=np.uint32), np.diff(want_seg.astype(np.int64)))
        _check(*_gpu_index(lib, d, q, 22, 1 << bits), want_S, want_seg, want_keys, (kind, n, q))


# ---------------------------------------------------------------------------- CPU: the kept snapshot in the sim
@pytest.fixture(scope="module")
def snap(tmp_path_factory):
    """tests/sim/snapshot_check.cc (the sim's LZ77 fixpoint with the kept snapshot), compiled into a temporary directory"""
    import subprocess
    so = str(tmp_path_factory.mktemp("snap") / "libsnapcheck.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-Wno-unused-function",
                           "-o", so, os.path.join(ROOT, "tests", "sim", "snapshot_check.cc")])
    L = C.CDLL(so)
    L.sim_init.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32]
    blob = open(TABLES, "rb").read()
    L.sim_init(blob, len(blob), (1 << 22) + 2)
    L.snap_check_lz77.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                  C.c_void_p]
    return L


def _snap_check(L, d, q, cuts=(), kinds=(), hint=None):
    st = np.zeros(3, np.uint64)
    cp = np.array(list(cuts) or [0], np.uint32); ck = np.array(list(kinds) or [0], np.uint32)
    assert L.snap_check_lz77(q, 22, d, len(d), hint or len(d), cp.ctypes.data, ck.ctypes.data, len(cuts), st.ctypes.data)
    checked, bad, flipped = (int(x) for x in st)
    assert checked >= 1 and bad == 0, (checked, bad, flipped)
    return flipped


@pytest.mark.parametrize("q", [5, 9])
@pytest.mark.parametrize("kind", ["text", "web", "binary", "noise"])
def test_sim_snapshot_kept_across_launches(snap, kind, q):
    flipped = _snap_check(snap, _input(kind, 1 << 19), q)
    if kind == "noise" and q == 5:
        assert flipped > 0   # the sparse search of quality 5 leaves noise unstored: the updates have work to do


def test_sim_snapshot_batch_and_flush(snap):
    t = synth_text(300000, seed=15)
    parts = [t[:70000], _input("noise", 50000), t[100000:160000]]
    bounds = np.cumsum([len(x) for x in parts]).tolist()
    _snap_check(snap, b"".join(parts), 5, bounds[:-1], [3, 3], hint=max(len(x) for x in parts))   # a batch of three streams
    _snap_check(snap, t, 5, [65536 + 3, 200001], [1, 1])                                          # two FLUSH cuts
