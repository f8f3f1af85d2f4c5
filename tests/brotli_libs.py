"""ctypes loaders for the checker libraries (oracle/ and oracle/_ref) and the product
C-ABI (brotli_b200/libbrotlienc_b200.so).  Test infrastructure only."""
import ctypes as C
import hashlib
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libbrotli_ref.so")
PROBE_SO = os.path.join(ROOT, "oracle", "_ref", "libbrotli_probe.so")
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
TABLES = os.path.join(ROOT, "brotli_b200", "data", "brotli_tables.bin")
PRODUCT_SO = os.path.join(ROOT, "brotli_b200", "libbrotlienc_b200.so")
REF_CALLS = os.path.join(ROOT, "tests", "golden", "reference_calls.json")

_u8p = C.POINTER(C.c_uint8)


def _buf(b):
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(b if len(b) else b"\0")


def zeroed_malloc():
    """The reference reads ring-buffer bytes it never wrote in some call sequences (c/enc/ringbuffer.h:104-116: the first write
    of less than a block skips the tail copy, and the buffer is grown by a plain malloc, :70-78; a later block that runs across
    the ring's end then compares against tail bytes nobody filled), so its output depends on what malloc hands out: identical
    in a fresh process (zero pages), different on a dirty heap (found by tools/sim_campaign.py: quality 4, lgwin 10, three
    FLUSHes; MALLOC_PERTURB_ flips it).  This makes malloc hand out zeroed memory in the calling process -- what a fresh
    process gets and what the oracle models (stale_byte) -- so that comparisons do not flake.  Called by tests/conftest.py and
    the campaign tools only: bench.py must time the reference with the allocator as it is."""
    try:
        C.CDLL(None).mallopt(-6, 255)      # M_PERTURB: allocations are filled with ~255 = 0
    except Exception:
        pass


class Ref:
    """The unmodified reference encoder, live (oracle/_ref, built by oracle/Makefile from a google/brotli tree)."""

    def __init__(self, path=REF_SO):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        L = self.lib
        L.BrotliEncoderCompress.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_void_p,
                                            C.POINTER(C.c_size_t), C.c_void_p]
        L.BrotliEncoderCompress.restype = C.c_int
        L.BrotliEncoderMaxCompressedSize.argtypes = [C.c_size_t]
        L.BrotliEncoderMaxCompressedSize.restype = C.c_size_t
        L.BrotliDecoderDecompress.argtypes = [C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p]
        L.BrotliDecoderDecompress.restype = C.c_int

    def compress(self, data, quality, lgwin, mode=0):
        n = len(data)
        cap = self.lib.BrotliEncoderMaxCompressedSize(n) + 16
        out = C.create_string_buffer(cap)
        out_n = C.c_size_t(cap)
        ok = self.lib.BrotliEncoderCompress(quality, lgwin, mode, n, data, C.byref(out_n), out)
        assert ok == 1
        return out.raw[:out_n.value]

    def decompress(self, comp, max_out):
        out = C.create_string_buffer(max(1, max_out))
        out_n = C.c_size_t(max_out)
        ok = self.lib.BrotliDecoderDecompress(len(comp), comp, C.byref(out_n), out)
        assert ok == 1, "decoder rejected the stream"
        return out.raw[:out_n.value]


class Oracle:
    """Our CPU restatement (oracle/brotli_oracle.c)."""

    def __init__(self, path=ORACLE_SO):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        L = self.lib
        L.oracle_init.argtypes = [C.c_void_p, C.c_size_t]
        L.oracle_init.restype = C.c_int
        L.oracle_brotli_compress.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_void_p,
                                             C.POINTER(C.c_size_t), C.c_void_p]
        L.oracle_brotli_compress.restype = C.c_int
        L.oracle_fast_log2.argtypes = [C.c_size_t]
        L.oracle_fast_log2.restype = C.c_double
        blob = open(TABLES, "rb").read()
        assert L.oracle_init(blob, len(blob)) == 1

    def compress_q1_stream(self, data, lgwin, calls=None, ops=None):
        """The quality-1 stream for a sequence of CompressStream calls (sizes, and optionally their
        operations: 0 PROCESS, 1 FLUSH, 2 FINISH); None = one FINISH call."""
        L = self.lib
        L.oracle_brotli_compress_q1_ops.argtypes = [C.c_int, C.c_size_t, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                    C.POINTER(C.c_size_t), C.c_void_p]
        cap = 2 * len(data) + 100000
        out = C.create_string_buffer(cap)
        n = C.c_size_t(cap)
        arr = (C.c_size_t * len(calls))(*calls) if calls is not None else None
        oarr = (C.c_int * len(ops))(*ops) if ops is not None else None
        assert L.oracle_brotli_compress_q1_ops(lgwin, len(data), data, len(calls) if calls is not None else 0, arr, oarr,
                                               C.byref(n), out) == 1
        return out.raw[:n.value]

    def edge_stats_reset(self):
        self.lib.oracle_edge_stats_reset()

    def edge_stats(self):
        """The entropy-stage edge counters since the last reset (oracle/brotli_oracle.c EDGE_FIELDS) as a dict."""
        L = self.lib
        L.oracle_edge_stats.restype = C.c_size_t
        L.oracle_edge_stats.argtypes = [C.c_void_p, C.c_size_t]
        L.oracle_edge_stats_names.restype = C.c_char_p
        n = L.oracle_edge_stats(None, 0)
        vals = (C.c_uint64 * n)()
        L.oracle_edge_stats(vals, n)
        names = L.oracle_edge_stats_names().decode().rstrip(",").split(",")
        assert len(names) == n
        return dict(zip(names, vals))

    def stored_codes(self):
        """The literal, command and distance prefix codes stored by compressed metablocks since the last edge_stats_reset()."""
        return self.edge_stats()["codes"]

    def build_code(self, histo):
        """One prefix code as a metablock of quality 4+ builds and stores it (oracle_build_code): the smoothed counts, the
        depths, the code words, the stored bits (bytes, LSB first) and their number.  histo: 256, 704 or 64 counts."""
        import numpy as np
        L = self.lib
        L.oracle_build_code.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.POINTER(C.c_size_t)]
        L.oracle_build_code.restype = C.c_int
        h = np.ascontiguousarray(histo, np.uint32)
        n = len(h)
        H, depth, bits = np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.uint16)
        stored = C.create_string_buffer(2 * n + 256)
        nbits = C.c_size_t(0)
        assert L.oracle_build_code(h.ctypes.data, n, H.ctypes.data, depth.ctypes.data, bits.ctypes.data, stored, len(stored),
                                   C.byref(nbits)) == 1, n
        return H, depth, bits, stored.raw[:(nbits.value + 7) // 8], nbits.value

    def compress(self, data, quality, lgwin):
        n = len(data)
        cap = n + (n >> 1) + 4096
        out = C.create_string_buffer(cap)
        out_n = C.c_size_t(cap)
        ok = self.lib.oracle_brotli_compress(quality, lgwin, n, data, C.byref(out_n), out)
        assert ok == 1
        return out.raw[:out_n.value]


def ref_compress_stream(ref, data, quality, lgwin, chunk, out_buf=1 << 19):
    """Drives the reference's streaming API the way c/tools/brotli.c:1357 does: PROCESS calls of
    `chunk` bytes, FINISH once the input is exhausted (an extra empty call when the size is a
    multiple of `chunk`, like feof() after a full read)."""
    if isinstance(ref, RecordedRef):
        return ref.compress_stream(data, quality, lgwin, chunk, out_buf)
    L = ref.lib
    L.BrotliEncoderCreateInstance.restype = C.c_void_p
    L.BrotliEncoderCreateInstance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.BrotliEncoderSetParameter.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.BrotliEncoderDestroyInstance.argtypes = [C.c_void_p]
    L.BrotliEncoderIsFinished.argtypes = [C.c_void_p]
    L.BrotliEncoderCompressStream.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_size_t), C.POINTER(C.c_void_p), C.c_void_p]
    s = L.BrotliEncoderCreateInstance(None, None, None)
    L.BrotliEncoderSetParameter(s, 1, quality)
    L.BrotliEncoderSetParameter(s, 2, lgwin)
    src = C.create_string_buffer(data, max(1, len(data)))
    dst = C.create_string_buffer(out_buf)
    out = bytearray()
    pos, eof = 0, False
    avail_in = C.c_size_t(0); next_in = C.c_void_p(C.addressof(src))
    avail_out = C.c_size_t(out_buf); next_out = C.c_void_p(C.addressof(dst))
    while True:
        if avail_in.value == 0 and not eof:
            n = min(chunk, len(data) - pos)
            next_in = C.c_void_p(C.addressof(src) + pos); avail_in = C.c_size_t(n)
            pos += n
            eof = n < chunk          # fread() came back short
        ok = L.BrotliEncoderCompressStream(s, 2 if eof else 0, C.byref(avail_in), C.byref(next_in),
                                           C.byref(avail_out), C.byref(next_out), None)
        assert ok == 1
        if avail_out.value == 0:
            out += dst.raw[:out_buf]
            avail_out = C.c_size_t(out_buf); next_out = C.c_void_p(C.addressof(dst))
        if L.BrotliEncoderIsFinished(s):
            out += dst.raw[:out_buf - avail_out.value]
            break
    L.BrotliEncoderDestroyInstance(s)
    return bytes(out)


def ref_stream_ops(ref, data, quality, lgwin, sizes, ops, out_buf=1 << 16, params=None):
    """Drives the reference's CompressStream with an explicit list of (size, op) calls, draining the
    output after each call the way encode.h:473 asks (repeat until no input and no more output)."""
    if isinstance(ref, RecordedRef):
        return ref.stream_ops(data, quality, lgwin, sizes, ops, out_buf, params)
    L = ref.lib
    L.BrotliEncoderCreateInstance.restype = C.c_void_p
    L.BrotliEncoderCreateInstance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.BrotliEncoderSetParameter.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.BrotliEncoderDestroyInstance.argtypes = [C.c_void_p]
    L.BrotliEncoderHasMoreOutput.argtypes = [C.c_void_p]
    L.BrotliEncoderCompressStream.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_size_t), C.POINTER(C.c_void_p), C.c_void_p]
    s = L.BrotliEncoderCreateInstance(None, None, None)
    L.BrotliEncoderSetParameter(s, 1, quality)
    L.BrotliEncoderSetParameter(s, 2, lgwin)
    for k, v in (params or {}).items():        # further BrotliEncoderParameter ids (3 LGBLOCK, 4 DISABLE_LITERAL_CONTEXT_MODELING ...)
        assert L.BrotliEncoderSetParameter(s, k, v) == 1
    src = C.create_string_buffer(data, max(1, len(data)))
    dst = C.create_string_buffer(out_buf)
    out = bytearray()
    pos = 0
    for size, op in zip(sizes, ops):
        avail_in = C.c_size_t(size); next_in = C.c_void_p(C.addressof(src) + pos)
        pos += size
        while True:
            avail_out = C.c_size_t(out_buf); next_out = C.c_void_p(C.addressof(dst))
            assert L.BrotliEncoderCompressStream(s, op, C.byref(avail_in), C.byref(next_in), C.byref(avail_out),
                                                 C.byref(next_out), None) == 1
            out += dst.raw[:out_buf - avail_out.value]
            if avail_in.value == 0 and not L.BrotliEncoderHasMoreOutput(s):
                break
    L.BrotliEncoderDestroyInstance(s)
    return bytes(out)


class Digest(object):
    """A byte string of the reference kept as its length and the first 128 bits of its SHA-256; compares equal to the
    bytes it was made from."""

    def __init__(self, n, sha):
        self.n, self.sha = n, sha

    def __eq__(self, other):
        if isinstance(other, Digest):
            return (self.n, self.sha) == (other.n, other.sha)
        if isinstance(other, (bytes, bytearray)):
            return len(other) == self.n and hashlib.sha256(other).hexdigest()[:32] == self.sha
        return NotImplemented

    def __ne__(self, other):
        r = self.__eq__(other)
        return r if r is NotImplemented else not r

    __hash__ = None

    def __len__(self):
        return self.n

    def __repr__(self):
        return "Digest(%d bytes, sha256 %s)" % (self.n, self.sha[:16])


def _digest(b):
    return [len(b), hashlib.sha256(b).hexdigest()[:32]]


def _tag(b):
    return "%d:%s" % (len(b), (b.sha if isinstance(b, Digest) else hashlib.sha256(b).hexdigest())[:24])


_CALLS = None


class RecordedRef(object):
    """The unmodified reference encoder and decoder as the tests compare against them: every result the tests ask for was
    computed once by the compiled reference (oracle/_ref) and is replayed from tests/golden/reference_calls.json as a
    Digest, so the comparisons run where the reference is not available.  A call that was not recorded -- above all a
    decompress() of bytes the reference did not produce -- fails.  With BROTLI_REF_RECORD=<file> (and oracle/_ref
    built) every call runs the live reference instead and appends its result to <file> as a JSON line;
    tests/golden/merge_reference_calls.py folds such files into reference_calls.json."""

    def __init__(self):
        global _CALLS
        self.record = os.environ.get("BROTLI_REF_RECORD")
        self.live = Ref() if self.record else None
        if _CALLS is None:
            _CALLS = json.load(open(REF_CALLS)) if os.path.exists(REF_CALLS) else {}

    def _call(self, key, run):
        if self.live is not None:
            v = run(self.live)
            val = v if isinstance(v, int) else _digest(v)
            with open(self.record, "a") as f:
                f.write(json.dumps({"key": key, "value": val}) + "\n")
            return v
        if key not in _CALLS:
            raise AssertionError("no recorded reference result for %r: the reference was never asked this (for decompress: "
                                 "the bytes are not what the reference encoder produced)" % key)
        val = _CALLS[key]
        return val if isinstance(val, int) else Digest(*val)

    def compress(self, data, quality, lgwin, mode=0):
        return self._call("compress q%d w%d m%d %s" % (quality, lgwin, mode, _tag(data)),
                          lambda r: r.compress(data, quality, lgwin, mode))

    def decompress(self, comp, max_out):
        return self._call("decompress %d %s" % (max_out, _tag(comp)), lambda r: r.decompress(comp, max_out))

    def max_compressed_size(self, n):
        return self._call("max_compressed_size %d" % n, lambda r: int(r.lib.BrotliEncoderMaxCompressedSize(n)))

    def compress_stream(self, data, quality, lgwin, chunk, out_buf):
        return self._call("compress_stream q%d w%d chunk%d %s" % (quality, lgwin, chunk, _tag(data)),
                          lambda r: ref_compress_stream(r, data, quality, lgwin, chunk, out_buf))

    def stream_ops(self, data, quality, lgwin, sizes, ops, out_buf, params):
        prm = sorted((params or {}).items())
        return self._call("stream_ops q%d w%d sizes%s ops%s params%s %s" % (quality, lgwin, list(sizes), list(ops), prm, _tag(data)),
                          lambda r: ref_stream_ops(r, data, quality, lgwin, sizes, ops, out_buf, params))
