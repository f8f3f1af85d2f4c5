"""brotli_b200 -- Python face of libbrotlienc_b200.so (GPU-native Brotli encoder hot path for the H100).

Mirrors the encoder half of the reference's Python module (python/brotli.py:24-49,
python/_brotli.c:403-458): ``compress()`` and ``Compressor.process/flush/finish`` with the same
argument names.  Everything goes through the C ABI declared in include/brotli_b200.h; there is
no Python or CPU implementation behind it -- if the CUDA library is missing or no GPU is
present the calls raise ``brotli_b200.error``.
"""
import ctypes as C
import os

MODE_GENERIC, MODE_TEXT, MODE_FONT = 0, 1, 2
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbrotlienc_b200.so")


class error(Exception):
    pass


_lib = None


def lib():
    """The loaded C-ABI library (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise error("libbrotlienc_b200.so is not built (run python __graft_entry__.py); "
                        "there is no fallback implementation")
        L = C.CDLL(LIB_PATH, mode=os.RTLD_LOCAL)
        L.BrotliEncoderCompress.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_void_p,
                                            C.POINTER(C.c_size_t), C.c_void_p]
        L.BrotliEncoderCompress.restype = C.c_int
        L.BrotliEncoderMaxCompressedSize.argtypes = [C.c_size_t]
        L.BrotliEncoderMaxCompressedSize.restype = C.c_size_t
        L.BrotliEncoderCreateInstance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.BrotliEncoderCreateInstance.restype = C.c_void_p
        L.BrotliEncoderDestroyInstance.argtypes = [C.c_void_p]
        L.BrotliEncoderSetParameter.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
        L.BrotliEncoderSetParameter.restype = C.c_int
        L.BrotliEncoderCompressStream.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t),
                                                  C.POINTER(C.c_void_p), C.POINTER(C.c_size_t),
                                                  C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.BrotliEncoderCompressStream.restype = C.c_int
        L.BrotliEncoderIsFinished.argtypes = [C.c_void_p]
        L.BrotliEncoderHasMoreOutput.argtypes = [C.c_void_p]
        L.BrotliEncoderTakeOutput.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        L.BrotliEncoderTakeOutput.restype = C.c_void_p
        L.BrotliEncoderVersion.restype = C.c_uint32
        L.BrotliB200CompressDevice.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p,
                                               C.POINTER(C.c_size_t), C.c_void_p]
        L.BrotliB200CompressDevice.restype = C.c_int
        L.BrotliB200CompressBatch.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int]
        L.BrotliB200CompressBatch.restype = C.c_size_t
        L.BrotliB200CompressBatchDevice.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.BrotliB200CompressBatchDevice.restype = C.c_size_t
        L.BrotliB200LastStats.argtypes = [C.POINTER(C.c_double)]
        L.BrotliB200LastStatsQ1.argtypes = [C.POINTER(C.c_double)]
        L.BrotliB200Available.restype = C.c_int
        _lib = L
    return _lib


def available():
    return bool(lib().BrotliB200Available())


def last_stats():
    """Timings of the calling thread's last compress call (ms) and pipeline counters."""
    a = (C.c_double * 16)()
    lib().BrotliB200LastStats(a)
    keys = ["ms_total", "ms_index", "ms_lz77", "ms_entropy", "ms_assemble", "lz77_iterations",
            "block_runs", "blocks", "metablocks", "launches", "ms_walk", "ms_encode", "walk_launches",
            "encode_launches", "walk_bytes", "total_cmds"]
    return dict(zip(keys, list(a)))


def last_stats_q1():
    """Timings (ms) and counters of the calling thread's last quality-1 batch."""
    a = (C.c_double * 12)()
    lib().BrotliB200LastStatsQ1(a)
    keys = ["ms_total", "ms_h2d", "ms_parse", "ms_code", "ms_pack", "ms_d2h", "streams", "fragments", "blocks",
            "in_bytes", "out_bytes", "launches"]
    return dict(zip(keys, list(a)))


def compress_batch(streams, quality, lgwin, threads=8):
    """Many independent one-shot streams in one call (BrotliB200CompressBatch); returns a list of bytes."""
    L = lib()
    n = len(streams)
    bufs = [C.create_string_buffer(bytes(s), max(1, len(s))) for s in streams]
    sizes = (C.c_size_t * n)(*[len(s) for s in streams])
    caps = [L.BrotliEncoderMaxCompressedSize(len(s)) + 16 for s in streams]
    outs = [C.create_string_buffer(c) for c in caps]
    in_ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    out_ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in outs])
    out_sizes = (C.c_size_t * n)(*caps)
    good = L.BrotliB200CompressBatch(quality, lgwin, n, in_ptrs, sizes, out_ptrs, out_sizes, threads)
    if good != n:
        raise error("BrotliB200CompressBatch: %d of %d streams failed" % (n - good, n))
    return [outs[i].raw[:out_sizes[i]] for i in range(n)]


def compress(string, mode=MODE_GENERIC, quality=11, lgwin=22, lgblock=0):
    """One-shot compression: python/brotli.py:24 ``compress`` (Compressor.process + finish)."""
    c = Compressor(mode=mode, quality=quality, lgwin=lgwin, lgblock=lgblock)
    return c.process(string) + c.finish()


def compress_oneshot(data, quality, lgwin, mode=MODE_GENERIC):
    """BrotliEncoderCompress (encode.h:405) on host buffers."""
    L = lib()
    n = len(data)
    cap = L.BrotliEncoderMaxCompressedSize(n) + 16
    out = C.create_string_buffer(cap)
    out_n = C.c_size_t(cap)
    if not L.BrotliEncoderCompress(quality, lgwin, mode, n, bytes(data), C.byref(out_n), out):
        raise error("BrotliEncoderCompress failed (unsupported parameters or no CUDA device)")
    return out.raw[:out_n.value]


class Compressor(object):
    """python/_brotli.c:403 Compressor: streaming interface over BrotliEncoderCompressStream."""
    _PROCESS, _FLUSH, _FINISH = 0, 1, 2

    def __init__(self, mode=MODE_GENERIC, quality=11, lgwin=22, lgblock=0):
        L = lib()
        self._s = L.BrotliEncoderCreateInstance(None, None, None)
        if not self._s:
            raise error("BrotliEncoderCreateInstance failed")
        for param, val in ((0, mode), (1, quality), (2, lgwin), (3, lgblock)):
            if not L.BrotliEncoderSetParameter(self._s, param, val):   # python/_brotli.c:432 raises as well
                raise error("BrotliEncoderSetParameter(%d, %d) failed" % (param, val))

    def __del__(self):
        if getattr(self, "_s", None):
            lib().BrotliEncoderDestroyInstance(self._s)
            self._s = None

    def _stream(self, data, op):
        L = lib()
        buf = C.create_string_buffer(bytes(data), len(data)) if len(data) else None
        avail_in = C.c_size_t(len(data))
        next_in = C.c_void_p(C.addressof(buf) if buf is not None else None)
        out = []
        while True:
            avail_out = C.c_size_t(0)
            next_out = C.c_void_p(None)
            ok = L.BrotliEncoderCompressStream(self._s, op, C.byref(avail_in), C.byref(next_in),
                                               C.byref(avail_out), C.byref(next_out), None)
            if not ok:
                raise error("BrotliEncoderCompressStream failed")
            while L.BrotliEncoderHasMoreOutput(self._s):
                sz = C.c_size_t(0)
                p = L.BrotliEncoderTakeOutput(self._s, C.byref(sz))
                out.append(C.string_at(p, sz.value))
            if avail_in.value == 0:
                break
        return b"".join(out)

    def emit_metadata(self, payload):
        """BROTLI_OPERATION_EMIT_METADATA (encode.h:127): a metadata block with `payload` (<= 16 MiB) at the current position."""
        return self._stream(payload, 3)

    def process(self, string):
        return self._stream(string, self._PROCESS)

    def flush(self):
        return self._stream(b"", self._FLUSH)

    def finish(self):
        return self._stream(b"", self._FINISH)
