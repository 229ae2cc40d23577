"""ctypes binding of the CPU restatement of BZip2.compress (oracle/bzip2_compress.c -> oracle/libswco_bzip2c.so).
TEST INFRASTRUCTURE ONLY: the same rules as swco.py, whose libswco.so it does not touch.

bzip2_compress returns (status, output_bytes, None) where status is an include/swc_status.h code."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = ["bzip2_compress.c", "checksums.c"]
_LIB = None


class _Buf(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_size_t), ("cap", C.c_size_t)]


def build(force=False):
    so = os.path.join(_HERE, "libswco_bzip2c.so")
    deps = [os.path.join(_HERE, f) for f in _SRCS + ["swco.h"]] + [os.path.join(_HERE, "..", "include", "swc_status.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-g", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-shared",
                               "-o", so] + [os.path.join(_HERE, f) for f in _SRCS] + ["-lpthread"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _ptr(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(bytes(b) + (b"\0" if not b else b""))


def bzip2_compress(data, block_size=1):
    """BZip2.compress(data:blockSize:) of BZip2+Compress.swift:44-74; block_size is BlockSize.rawValue (1-9)"""
    buf = _Buf()
    st = lib().swco_bzip2_compress(_ptr(data), C.c_size_t(len(data)), C.c_int(block_size), C.byref(buf))
    out = C.string_at(buf.data, buf.len) if buf.len else b""
    C.CDLL(None).free(C.c_void_p(buf.data))
    return st, out, None


def suffix_array(seq, alphabet=256):
    """SuffixArray.make(from:with:) as written: len(seq) + 1 entries, entry 0 is the empty suffix"""
    import numpy as np
    b = np.asarray(list(seq) + [0], dtype=np.int32)
    sa = np.zeros(len(seq) + 1, dtype=np.int64)
    st = lib().swco_bzip2c_suffix_array(b.ctypes.data_as(C.c_void_p), C.c_int64(len(seq)), C.c_int32(alphabet),
                                        sa.ctypes.data_as(C.c_void_p))
    assert st == 0
    return [int(x) for x in sa]


def lengths(stats):
    """BZip2.lengths(from:) of BZip2+Lengths.swift: the code length of symbols 0, 1, 2, ..."""
    import numpy as np
    s = np.asarray(list(stats) + [0], dtype=np.int64)
    out = np.zeros(len(stats) + 1, dtype=np.int32)
    st = lib().swco_bzip2c_lengths(s.ctypes.data_as(C.c_void_p), C.c_int64(len(stats)), out.ctypes.data_as(C.c_void_p))
    assert st == 0
    return [int(x) for x in out[: len(stats)]]


def batch_mt(units, total, threads, block_size=1):
    """Compress `total` units (wrapping over `units`) on `threads` pthreads inside C: no interpreter in the timed loop.
    -> (seconds, compressed bytes, failures)."""
    import numpy as np
    lens = np.fromiter((len(u) for u in units), dtype=np.uint64, count=len(units))
    offs = np.zeros(len(units), dtype=np.uint64)
    if len(units) > 1:
        offs[1:] = np.cumsum(lens[:-1])
    blob = np.frombuffer(b"".join(units) + b"\0" * 16, dtype=np.uint8)
    sec, nbytes, fails = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    rc = lib().swco_bzip2c_batch_mt(blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p),
                                    lens.ctypes.data_as(C.c_void_p), C.c_uint64(len(units)), C.c_uint64(total),
                                    C.c_int(block_size), C.c_int(threads), C.byref(sec), C.byref(nbytes), C.byref(fails))
    if rc != 0:
        raise RuntimeError("swco_bzip2c_batch_mt could not start its threads")
    return sec.value, nbytes.value, fails.value
