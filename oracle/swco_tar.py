"""ctypes binding of the CPU restatement of TarContainer.open / info / formatOf (oracle/tar.c -> oracle/libswco_tar.so).
TEST INFRASTRUCTURE ONLY: the same rules as swco.py, whose libswco.so it does not touch.

walk(data) returns what one unit of swc_tar_walk_batch reports: (n_entries, info_status, open_status, format,
format_status, records), with records as dicts of the swc_tar_entry fields (include/swcgpu.h)."""
import ctypes as C
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = ["tar.c"]
_LIB = None

# the record layout is swc_tar_entry (include/swcgpu.h), the same struct the library fills: one ctypes definition for both
sys.path.insert(0, os.path.dirname(_HERE))
from swcompression_b200._lib import TarEntry, tar_record as record  # noqa: E402


def build(force=False):
    so = os.path.join(_HERE, "libswco_tar.so")
    deps = [os.path.join(_HERE, f) for f in _SRCS] + [os.path.join(_HERE, "..", "include", n) for n in ("swc_status.h", "swcgpu.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-g", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-shared",
                               "-o", so] + [os.path.join(_HERE, f) for f in _SRCS])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def walk(data, cap=None):
    """-> (n_entries, info_status, open_status, format, format_status, [record dict]); `cap` is the entry table size
    (default len // 512 + 1, grown to the reported count when the walk has more)."""
    data = bytes(data)
    buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
    first = cap is None
    cap = len(data) // 512 + 1 if cap is None else cap
    while True:
        tab = (TarEntry * max(cap, 1))()
        n, ist, ost, fmt, fst = C.c_uint64(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        lib().swco_tar_walk(buf, C.c_uint64(len(data)), tab, C.c_uint64(cap), C.byref(n), C.byref(ist), C.byref(ost),
                            C.byref(fmt), C.byref(fst))
        if first and n.value > cap:
            cap, first = n.value, False
            continue
        return n.value, ist.value, ost.value, fmt.value, fst.value, [record(tab[i]) for i in range(min(n.value, cap))]


def walk_seconds(units, threads):
    """Wall time of swco_tar_walk alone over `units` on `threads` threads (ctypes releases the GIL during each call): the
    input buffers and in_len // 512 + 1 record tables are prepared before the clock starts, and no record is converted."""
    import time
    from concurrent.futures import ThreadPoolExecutor
    jobs = []
    for u in units:
        cap = len(u) // 512 + 1
        jobs.append(((C.c_uint8 * max(len(u), 1)).from_buffer_copy(bytes(u) or b"\0"), len(u), (TarEntry * cap)(), cap))
    fn = lib().swco_tar_walk

    def run(j):
        outs = [C.c_uint64(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()]
        fn(j[0], C.c_uint64(j[1]), j[2], C.c_uint64(j[3]), *[C.byref(o) for o in outs])
        return outs[0].value

    with ThreadPoolExecutor(threads) as ex:
        t0 = time.perf_counter()
        list(ex.map(run, jobs))
        return time.perf_counter() - t0
