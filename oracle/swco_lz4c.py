"""ctypes binding of the CPU restatement of LZ4.compress (oracle/lz4_compress.c -> oracle/libswco_lz4c.so).  TEST
INFRASTRUCTURE ONLY: the same rules as swco.py, whose libswco.so it does not touch.

Every function returns (status, output_bytes, extra) where status is an include/swc_status.h code."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = ["lz4_compress.c", "checksums.c"]
_LIB = None


class _Buf(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_size_t), ("cap", C.c_size_t)]


def build(force=False):
    so = os.path.join(_HERE, "libswco_lz4c.so")
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


def _take(buf):
    out = C.string_at(buf.data, buf.len) if buf.len else b""
    C.CDLL(None).free(C.c_void_p(buf.data))
    return out


def _ptr(b):
    return (C.c_uint8 * max(len(b), 1)).from_buffer_copy(bytes(b) + (b"\0" if not b else b""))


def lz4_block_compress(data, dictionary=None):
    """compress(block:_:) of LZ4+Compress.swift:156-277: the raw block, even when it is longer than `data`"""
    buf = _Buf()
    d = dictionary or b""
    st = lib().swco_lz4_block_compress(_ptr(data), C.c_size_t(len(data)), _ptr(d), C.c_size_t(len(d)), C.byref(buf))
    return st, _take(buf), None


def lz4_compress(data, independentBlocks=True, blockChecksums=False, contentChecksum=True, contentSize=False,
                 blockSize=4 << 20, dictionary=None, dictionaryID=None):
    """LZ4.compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:dictionary:dictionaryID:)"""
    buf = _Buf()
    dp, dl = (None, 0) if dictionary is None else (_ptr(dictionary), len(dictionary))
    st = lib().swco_lz4_compress(_ptr(data), C.c_size_t(len(data)), C.c_int(int(bool(independentBlocks))),
                                 C.c_int(int(bool(blockChecksums))), C.c_int(int(bool(contentChecksum))),
                                 C.c_int(int(bool(contentSize))), C.c_int64(blockSize), dp, C.c_size_t(dl),
                                 C.c_int(0 if dictionaryID is None else 1), C.c_uint32(dictionaryID or 0), C.byref(buf))
    return st, _take(buf), None


def batch_mt(units, total, threads):
    """Compress `total` raw blocks (wrapping over `units`, no dictionary) on `threads` pthreads inside C: no interpreter in
    the timed loop.  -> (seconds, compressed bytes, failures)."""
    import numpy as np
    lens = np.fromiter((len(u) for u in units), dtype=np.uint64, count=len(units))
    offs = np.zeros(len(units), dtype=np.uint64)
    if len(units) > 1:
        offs[1:] = np.cumsum(lens[:-1])
    blob = np.frombuffer(b"".join(units) + b"\0" * 16, dtype=np.uint8)
    sec, nbytes, fails = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    rc = lib().swco_lz4c_batch_mt(blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p),
                                  lens.ctypes.data_as(C.c_void_p), C.c_uint64(len(units)), C.c_uint64(total),
                                  C.c_int(threads), C.byref(sec), C.byref(nbytes), C.byref(fails))
    if rc != 0:
        raise RuntimeError("swco_lz4c_batch_mt could not start its threads")
    return sec.value, nbytes.value, fails.value
