#!/usr/bin/env python3
"""What gzip / zlib framing adds to the batched Deflate decode: BASELINE config 2 (4 096 distinct 64 KiB units from bench.py's
make_corpus, tiled on the device to 262 144) as raw Deflate streams, as gzip members (10-byte header, CRC-32, ISIZE) and as
zlib streams (78 9c, big-endian Adler-32).  In one process, alternating, CUDA events time swc_deflate_decompress_batch,
swc_gzip_unarchive_batch and swc_zlib_unarchive_batch on the same device-resident Deflate bytes; swc_timing_enable /
swc_timing_collect give the per-stage intervals.  Every unit's status, length, consumed count and CRC-32 is checked.

    python tools/bench_unarchive_batch.py [--steps 5] [--warmup 2] [--units 262144] [--distinct 4096]

Prints one JSON line with the GPU's name and power limit beside the numbers."""
import argparse
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UNIT = 65536
GZIP_HEAD = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03"
ZLIB_HEAD = b"\x78\x9c"
# interval names in launch order (marks: swc_*_unarchive_batch around its stages, inflate::launch around its kernels)
DEFLATE_STAGES = ["inflate_kernel (K1)", "inflate_slow_kernel", "lz_resolve_kernel (K2)"]
UNARCHIVE_STAGES = ["header", "ticket reset"] + DEFLATE_STAGES + ["checksum", "trailer"]


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=262144)
    ap.add_argument("--distinct", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from bench import make_corpus
    units, crcs = make_corpus(args.distinct, seed0=2)             # the generator pool forks before CUDA is initialised
    adlers = [zlib.adler32(zlib.decompress(u, -15)) for u in units]
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import pack_units
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    tile = args.units // args.distinct
    n = tile * args.distinct

    def tiled(blobs):
        """the distinct blobs packed 16-byte aligned, repeated `tile` times on the device -> (device buffer, offsets, lengths)"""
        buf, offs, lens = pack_units(blobs)
        stride = len(buf) - 64
        d = torch.cat([torch.from_numpy(buf[:stride]).to(dev).repeat(tile), torch.zeros(64, dtype=torch.uint8, device=dev)])
        all_off = (offs[None, :] + (np.arange(tile, dtype=np.uint64) * np.uint64(stride))[:, None]).reshape(-1)
        return d, all_off, np.tile(lens, tile)

    d_gz, gz_off, gz_len = tiled([GZIP_HEAD + u + struct.pack("<II", c, UNIT) for u, c in zip(units, crcs)])
    d_zl, zl_off, zl_len = tiled([ZLIB_HEAD + u + struct.pack(">I", a) for u, a in zip(units, adlers)])
    raw_off, raw_len = gz_off + np.uint64(len(GZIP_HEAD)), gz_len - np.uint64(len(GZIP_HEAD) + 8)   # the same Deflate bytes
    total_in = int(raw_len.sum())
    del units
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).to(dev)
    cols = {"deflate": (d_gz, t(raw_off), t(raw_len)), "gzip": (d_gz, t(gz_off), t(gz_len)), "zlib": (d_zl, t(zl_off), t(zl_len))}
    out_total = n * UNIT
    d_out = torch.empty(out_total + 64, dtype=torch.uint8, device=dev)
    d_ooff = t(np.arange(n, dtype=np.uint64) * np.uint64(UNIT))
    d_ocap = t(np.full(n, UNIT, dtype=np.uint64))
    d_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_used = torch.zeros(n, dtype=torch.int64, device=dev)
    d_st = torch.zeros(n, dtype=torch.int32, device=dev)
    d_crc = torch.zeros(n, dtype=torch.int32, device=dev)
    scratch_bytes = L.swc_unarchive_batch_scratch_bytes(n, out_total)
    assert scratch_bytes >= L.swc_deflate_batch_scratch_bytes(n, out_total)
    d_scr = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def call(fmt):
        d_in, d_off, d_ln = cols[fmt]
        common = (p(d_out), p(d_ooff), p(d_ocap), out_total, p(d_len), p(d_used), p(d_st))
        if fmt == "deflate":
            rc = L.swc_deflate_decompress_batch(p(d_in), p(d_off), p(d_ln), None, *common, n, p(d_scr), scratch_bytes, stream())
        elif fmt == "gzip":
            rc = L.swc_gzip_unarchive_batch(p(d_in), p(d_off), p(d_ln), *common, None, n, p(d_scr), scratch_bytes, stream())
        else:
            rc = L.swc_zlib_unarchive_batch(p(d_in), p(d_off), p(d_ln), *common, n, p(d_scr), scratch_bytes, stream())
        assert rc == 0, _lib.status_name(rc)

    crc_want = torch.tensor(crcs, dtype=torch.int64, device=dev)[torch.arange(n, device=dev) % args.distinct]

    def check(fmt):
        d_st.fill_(-1); d_len.zero_(); d_used.zero_(); d_crc.zero_()
        call(fmt)
        assert L.swc_crc32_batch(p(d_out), p(d_ooff), p(d_len), p(d_st), p(d_crc), n, stream()) == 0
        torch.cuda.synchronize(dev)
        assert bool((d_st == 0).all()) and bool((d_len == UNIT).all()), f"{fmt}: a unit failed"
        assert torch.equal(d_crc.to(torch.int64) & 0xFFFFFFFF, crc_want), f"{fmt}: a decoded unit has the wrong CRC-32"
        if fmt != "deflate":
            assert torch.equal(d_used, cols[fmt][2]), f"{fmt}: consumed bytes differ from the archive lengths"
        else:
            assert bool(((d_used + 7) // 8 == cols[fmt][2]).all()), "deflate: consumed bits do not end in the last byte"

    fmts = ["deflate", "gzip", "zlib"]
    for fmt in fmts:
        for _ in range(args.warmup):
            call(fmt)
        check(fmt)
    torch.cuda.synchronize(dev)
    ms = {f: [] for f in fmts}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.steps):                                   # alternating: deflate, gzip, zlib, deflate, ...
        for fmt in fmts:
            e0.record()
            call(fmt)
            e1.record()
            torch.cuda.synchronize(dev)
            ms[fmt].append(e0.elapsed_time(e1))
    stages = {}
    buf = (C.c_float * 16)()
    for fmt in fmts:                                              # per-stage intervals, in runs of their own
        names = DEFLATE_STAGES if fmt == "deflate" else UNARCHIVE_STAGES
        acc = np.zeros(len(names))
        for _ in range(args.steps):
            L.swc_timing_enable(1)
            call(fmt)
            torch.cuda.synchronize(dev)
            k = L.swc_timing_collect(buf, len(buf))
            L.swc_timing_enable(0)
            assert k == len(names), (fmt, k)
            acc += np.array(list(buf)[:k])
        stages[fmt] = dict(zip(names, (acc / args.steps).round(3).tolist()))
    for fmt in fmts:
        check(fmt)                                                # the timed calls left the right answers behind too
    med = {f: float(np.median(v)) for f, v in ms.items()}
    framing = {f: stages[f]["header"] + stages[f]["checksum"] + stages[f]["trailer"] for f in ("gzip", "zlib")}
    deflate_ms = sum(stages["deflate"].values())
    print(json.dumps({
        "gpu": gpu_identity(), "torch_device": torch.cuda.get_device_name(dev),
        "workload": f"{n} units x 64 KiB ({args.distinct} distinct tiled x{tile}); {total_in} Deflate bytes, {out_total} decoded bytes",
        "ms_median": med, "ms_all": ms, "decoded_GB_per_s": {f: out_total / (v * 1e-3) / 1e9 for f, v in med.items()},
        "stage_ms": stages, "framing_ms": framing, "framing_share_of_deflate": {f: v / deflate_ms for f, v in framing.items()},
        "steps": args.steps, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
