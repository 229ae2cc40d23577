"""ctypes binding of the CPU restatement of Deflate.compress, GzipArchive.archive and ZlibArchive.archive
(oracle/deflate_compress.c -> oracle/libswco_deflatec.so).  TEST INFRASTRUCTURE ONLY: the same rules as swco.py, whose
libswco.so it does not touch.

Every function returns (status, output_bytes, extra) where status is an include/swc_status.h code."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = ["deflate_compress.c", "checksums.c"]
_LIB = None


class _Buf(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_size_t), ("cap", C.c_size_t)]


def build(force=False):
    so = os.path.join(_HERE, "libswco_deflatec.so")
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


def deflate_compress(data):
    """Deflate.compress(data:) of Deflate+Compress.swift:22-42"""
    buf = _Buf()
    st = lib().swco_deflate_compress(_ptr(data), C.c_size_t(len(data)), C.byref(buf))
    return st, _take(buf), None


def zlib_archive(data):
    """ZlibArchive.archive(data:) of ZlibArchive.swift:54-70"""
    buf = _Buf()
    st = lib().swco_zlib_archive(_ptr(data), C.c_size_t(len(data)), C.byref(buf))
    return st, _take(buf), None


def gzip_archive(data, comment=None, fileName=None, writeHeaderCRC=False, isTextFile=False, osByte=255,
                 modificationTime=None, extraFields=()):
    """GzipArchive.archive of GzipArchive.swift:126-241.  comment / fileName are ISO-Latin-1 bytes or None; osByte is
    osTypeByte; modificationTime is Int(timeIntervalSince1970) or None; extraFields are (si1, si2, bytes) triples."""
    import numpy as np
    buf = _Buf()
    c = b"" if comment is None else bytes(comment)
    f = b"" if fileName is None else bytes(fileName)
    ids = bytes(b for e in extraFields for b in (e[0], e[1]))
    lens = np.array([len(e[2]) for e in extraFields] + [0], dtype=np.uint64)
    blob = b"".join(bytes(e[2]) for e in extraFields)
    st = lib().swco_gzip_archive(_ptr(data), C.c_size_t(len(data)), _ptr(c), C.c_size_t(len(c)), C.c_int(comment is not None),
                                 _ptr(f), C.c_size_t(len(f)), C.c_int(fileName is not None), C.c_int(int(bool(writeHeaderCRC))),
                                 C.c_int(int(bool(isTextFile))), C.c_uint8(osByte), C.c_int(modificationTime is not None),
                                 C.c_int64(modificationTime or 0), C.c_size_t(len(extraFields)), _ptr(ids),
                                 lens.ctypes.data_as(C.c_void_p), _ptr(blob), C.byref(buf))
    return st, _take(buf), None


def batch_mt(units, total, threads):
    """Compress `total` units (wrapping over `units`) on `threads` pthreads inside C: no interpreter in the timed loop.
    -> (seconds, compressed bytes, failures)."""
    import numpy as np
    lens = np.fromiter((len(u) for u in units), dtype=np.uint64, count=len(units))
    offs = np.zeros(len(units), dtype=np.uint64)
    if len(units) > 1:
        offs[1:] = np.cumsum(lens[:-1])
    blob = np.frombuffer(b"".join(units) + b"\0" * 16, dtype=np.uint8)
    sec, nbytes, fails = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    rc = lib().swco_deflatec_batch_mt(blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p),
                                      lens.ctypes.data_as(C.c_void_p), C.c_uint64(len(units)), C.c_uint64(total),
                                      C.c_int(threads), C.byref(sec), C.byref(nbytes), C.byref(fails))
    if rc != 0:
        raise RuntimeError("swco_deflatec_batch_mt could not start its threads")
    return sec.value, nbytes.value, fails.value
