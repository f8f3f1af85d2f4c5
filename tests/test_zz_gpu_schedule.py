"""GPU suite (-m gpu): the LZ77 fixpoint's schedule knobs on the CUDA kernels (tests/test_fixpoint_schedule.py runs the
whole matrix in the sim).

br_debug_compress_sched runs br_job_compress_device with sweep_epoch, force_epoch, step_cap, heavy_min, pilot and
sweep_blocks set on the host; the release build has no switch for them.  On the GPU a launch's walks and commits are
concurrent, so every case here also runs them in whatever order the hardware picks.  Every case must give the oracle's
bytes, and no launch may walk more chunks than ran_list holds: every chunk at most once."""
import ctypes as C

import numpy as np
import pytest

from brotli_libs import Oracle
from fuzz_cases import cases

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

KEEP = 0xFFFFFFFF
LAUNCHES, WALKS, CHUNKS, FORCED, MAX_WALKS, RAN_CAP = 0, 1, 2, 3, 4, 5


class Knobs(C.Structure):
    _fields_ = [(f, C.c_uint32) for f in ("sweep_epoch", "force_epoch", "step_cap", "heavy_min", "pilot", "sweep_blocks")]


@pytest.fixture(scope="module")
def lib():
    import brotli_b200
    assert brotli_b200.available(), "no CUDA device"
    L = brotli_b200.lib()
    L.br_debug_compress_sched.restype = C.c_long
    L.br_debug_compress_sched.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.POINTER(Knobs), C.c_void_p,
                                          C.c_size_t, C.c_void_p]
    return L


def run(L, d, q, w, **kw):
    k = Knobs(*[KEEP] * 6)
    for f, v in kw.items():
        setattr(k, f, v)
    cap = len(d) + len(d) // 2 + 4096
    out = C.create_string_buffer(cap)
    st = np.zeros(8, np.uint32)
    r = L.br_debug_compress_sched(q, w, d, len(d), C.byref(k), out, cap, st.ctypes.data)
    assert r > 0, ("the job failed", q, w, kw)
    return out.raw[:r], st


def check(L, d, q, w, want, **kw):
    got, st = run(L, d, q, w, **kw)
    assert st[MAX_WALKS] <= st[CHUNKS] <= st[RAN_CAP], ("a chunk was walked twice in one launch", q, w, kw, st)
    assert got == want, ("bytes differ from the oracle", q, w, kw, len(got), len(want))
    return st


def _case_2_50():
    for i, d, q, w in cases(2, 51):
        if i == 50:
            return d


def test_regressions(lib):
    """the two schedules the sim found wrong: force_epoch 1 on 256 KiB of noise (more walks than ran_list held) and
    cases(2, 51)[50] with force_epoch 2 (the forced walker and a scheduled walker shared a chunk and its bitmap)"""
    ora = Oracle()
    d = np.random.default_rng(5).integers(0, 256, 262144, dtype=np.uint8).tobytes()
    st = check(lib, d, 5, 22, ora.compress(d, 5, 22), force_epoch=1)
    assert st[FORCED] > 0
    d = _case_2_50()
    want = ora.compress(d, 5, 24)
    for s in (0, 1):
        assert check(lib, d, 5, 24, want, sweep_epoch=s, force_epoch=2)[FORCED] > 0


@pytest.mark.parametrize("q", [5, 7, 9])
def test_schedules(lib, q):
    """force_epoch 0/1/2 crossed with sweep_epoch 0/1/3, step_cap 0 and the pilot launch on"""
    from corpus import synth_web
    ora = Oracle()
    ins = [_case_2_50(), synth_web(300000, 41)]
    for d in ins:
        want = ora.compress(d, q, 22)
        for f in (0, 1, 2):
            for s in (0, 1, 3):
                check(lib, d, q, 22, want, force_epoch=f, sweep_epoch=s)
        check(lib, d, q, 22, want, step_cap=0)
        check(lib, d, q, 22, want, pilot=1)
        check(lib, d, q, 22, want, pilot=1, force_epoch=1, sweep_epoch=0)


def test_large_binary_forced(lib):
    """8 MiB of binary input with force_epoch 1: every launch from the first has a forced walker that runs through a
    whole input block whose other chunks are scheduled too"""
    from corpus import synth_binary
    d = synth_binary(8 << 20, 17)
    st = check(lib, d, 5, 22, Oracle().compress(d, 5, 22), force_epoch=1)
    assert st[FORCED] > 0 and st[LAUNCHES] > 1
