"""CPU suite, part 3: the C-ABI library loads, exports every symbol include/brotli_b200.h
declares, and fails loudly (never falls back) when no CUDA device is present."""
import ctypes as C
import os
import re

import pytest

from brotli_libs import ROOT

SO = os.path.join(ROOT, "brotli_b200", "libbrotlienc_b200.so")
HEADER = os.path.join(ROOT, "include", "brotli_b200.h")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO):
        import __graft_entry__
        __graft_entry__.build_product()
    return C.CDLL(SO, mode=os.RTLD_LOCAL)


ENCODE_H = os.path.join(ROOT, "include", "brotli", "encode.h")


def declared_symbols():
    """Every function the public headers declare: the reference API (include/brotli/encode.h) and the device-resident extensions."""
    names = set()
    for path, macro in ((HEADER, "BROTLI_B200_API"), (ENCODE_H, "BROTLI_ENC_API")):
        names |= set(re.findall(macro + r"[^;(]*?\b(Brotli\w+)\s*\(", open(path).read()))
    return sorted(names)


def test_header_declares_reference_api():
    names = declared_symbols()
    for n in ["BrotliEncoderSetParameter", "BrotliEncoderCreateInstance", "BrotliEncoderDestroyInstance",
              "BrotliEncoderPrepareDictionary", "BrotliEncoderDestroyPreparedDictionary",
              "BrotliEncoderAttachPreparedDictionary", "BrotliEncoderMaxCompressedSize", "BrotliEncoderCompress",
              "BrotliEncoderCompressStream", "BrotliEncoderIsFinished", "BrotliEncoderHasMoreOutput",
              "BrotliEncoderTakeOutput", "BrotliEncoderVersion"]:
        assert n in names      # the 13 BROTLI_ENC_API functions of c/include/brotli/encode.h


def test_library_exports_every_declared_symbol(lib):
    for n in declared_symbols():
        assert hasattr(lib, n), n


def test_host_only_entry_points(lib):
    lib.BrotliEncoderMaxCompressedSize.restype = C.c_size_t
    lib.BrotliEncoderMaxCompressedSize.argtypes = [C.c_size_t]
    assert lib.BrotliEncoderMaxCompressedSize(0) == 2
    assert lib.BrotliEncoderMaxCompressedSize(1 << 20) == (1 << 20) + 2 + 4 * 64 + 3 + 1   # encode.c:1251
    lib.BrotliEncoderVersion.restype = C.c_uint32
    assert lib.BrotliEncoderVersion() == 0x1002000
    # empty input never needs the GPU: single byte 0x06 (encode.c:1310)
    out = C.create_string_buffer(8)
    n = C.c_size_t(8)
    lib.BrotliEncoderCompress.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p]
    assert lib.BrotliEncoderCompress(5, 22, 0, 0, None, C.byref(n), out) == 1 and out.raw[:n.value] == b"\x06"


def test_state_api_and_loud_failure(lib):
    lib.BrotliEncoderCreateInstance.restype = C.c_void_p
    lib.BrotliEncoderCreateInstance.argtypes = [C.c_void_p] * 3
    lib.BrotliEncoderSetParameter.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    lib.BrotliEncoderDestroyInstance.argtypes = [C.c_void_p]
    s = lib.BrotliEncoderCreateInstance(None, None, None)
    assert s
    assert lib.BrotliEncoderSetParameter(s, 1, 5) == 1      # QUALITY
    assert lib.BrotliEncoderSetParameter(s, 2, 22) == 1     # LGWIN
    assert lib.BrotliEncoderSetParameter(s, 99, 0) == 0     # unknown parameter
    lib.BrotliEncoderDestroyInstance(s)
    import brotli_b200
    if not brotli_b200.available():
        with pytest.raises(brotli_b200.error):
            brotli_b200.compress_oneshot(b"no gpu here " * 100, 5, 22)
        with pytest.raises(brotli_b200.error):           # the quality-1 batch path has no CPU fallback either
            brotli_b200.compress_oneshot(b"no gpu here " * 100, 1, 22)
        with pytest.raises(brotli_b200.error):
            brotli_b200.compress_batch([b"a" * 100, b"b" * 100], 1, 22)
    # parameters outside the implemented path are refused instead of silently changed
    out = C.create_string_buffer(4096)
    n = C.c_size_t(4096)
    assert lib.BrotliEncoderCompress(11, 22, 0, 100, b"x" * 100, C.byref(n), out) == 0
    n = C.c_size_t(4096)
    assert lib.BrotliEncoderCompress(5, 12, 0, 100, b"x" * 100, C.byref(n), out) == 0
    for q in (0, 10):                                     # qualities without a GPU path: refused, never other bytes
        n = C.c_size_t(4096)
        assert lib.BrotliEncoderCompress(q, 22, 0, 100, b"x" * 100, C.byref(n), out) == 0
    if not brotli_b200.available():                       # qualities 2..4 have a GPU path and, like the others, no CPU fallback
        for q in (2, 3, 4):
            n = C.c_size_t(4096)
            assert lib.BrotliEncoderCompress(q, 22, 0, 100, b"x" * 100, C.byref(n), out) == 0


def test_pkgconfig_dropin_layout(tmp_path):
    """packaging/install_dropin.sh lays the library out under the reference's names (libbrotlienc.so.1, libbrotlienc.pc,
    brotli/encode.h): a C99 program built the way go/cbrotli/cgo.go:10 or a USE_SYSTEM_BROTLI python build would (pkg-config
    libbrotlienc) links against it and runs the host-only entry points."""
    import shutil
    import subprocess
    if not (shutil.which("pkg-config") and shutil.which("gcc")):
        pytest.skip("pkg-config / gcc not available")
    if not os.path.exists(SO):
        import __graft_entry__
        __graft_entry__.build_product()
    prefix = tmp_path / "prefix"
    subprocess.check_call([os.path.join(ROOT, "packaging", "install_dropin.sh"), str(prefix)])
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <brotli/encode.h>\n#include <brotli_b200.h>\n'
                   'int main(void) { BrotliEncoderState* s = BrotliEncoderCreateInstance(0, 0, 0);\n'
                   '  int ok = s && BrotliEncoderSetParameter(s, BROTLI_PARAM_QUALITY, 5); BrotliEncoderDestroyInstance(s);\n'
                   '  printf("%u %zu %d\\n", BrotliEncoderVersion(), BrotliEncoderMaxCompressedSize(1 << 20), ok); return 0; }\n')
    env = dict(os.environ, PKG_CONFIG_PATH=str(prefix / "lib" / "pkgconfig"))
    flags = subprocess.check_output(["pkg-config", "--cflags", "--libs", "libbrotlienc"], env=env, text=True).split()
    exe = tmp_path / "t"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-o", str(exe), str(src)] + flags)
    out = subprocess.check_output([str(exe)], env=dict(os.environ, LD_LIBRARY_PATH=str(prefix / "lib")), text=True)
    assert out.split() == ["16785408", str((1 << 20) + 2 + 4 * 64 + 3 + 1), "1"]
    needed = subprocess.check_output(["readelf", "-d", str(exe)], text=True)
    assert "libbrotlienc.so.1" in needed
