#!/usr/bin/env python3
"""What XZ framing and the per-block check add to the batched LZMA2 decode: BASELINE config 5 (1 184 independent 1 MiB text
streams, preset 6, 1 MiB dictionary, 32 distinct inputs as in tools/bench_codecs.py --workload xz) as raw LZMA2 block
payloads and as whole .xz files with no check, CRC-32, CRC-64 and SHA-256.  In one process, alternating, CUDA events time
swc_lzma2_decompress_batch on the payloads and swc_xz_unarchive_batch on the archives.  Every unit's status and length is
checked; the raw batch's output is compared with the source text (the distinct units on the host, every tiled copy against
its distinct unit on the device), and every variant's whole output with the raw batch's.

    python tools/bench_xz_batch.py [--steps 5] [--warmup 1] [--units 1184] [--distinct 32]

Prints one JSON line with the GPU's name and power limit and the resident warps per SM of lzma_kernel and xz_kernel."""
import argparse
import ctypes as C
import json
import lzma
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

UNIT = 1 << 20
CHECKS = {"none": lzma.CHECK_NONE, "crc32": lzma.CHECK_CRC32, "crc64": lzma.CHECK_CRC64, "sha256": lzma.CHECK_SHA256}
FILTERS = [{"id": lzma.FILTER_LZMA2, "preset": 6, "dict_size": 1 << 20}]


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def block_payload(arc):
    """(LZMA2 payload, dictionary byte) of the single block of an archive from Python's lzma"""
    hsz = (arc[12] + 1) * 4
    hdr = arc[12:12 + hsz]
    k = hdr.index(b"\x21\x01", 2)
    return arc[12 + hsz:], hdr[k + 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=1184)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import helpers as H
    raws = [H.textlike(UNIT, 5 + k) for k in range(args.distinct)]
    archives = {c: [lzma.compress(r, format=lzma.FORMAT_XZ, check=v, filters=FILTERS) for r in raws] for c, v in CHECKS.items()}
    payloads = [block_payload(a) for a in archives["crc64"]]
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import pack_units
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    n = args.units
    pick = [i % args.distinct for i in range(n)]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)

    def columns(blobs):
        buf, offs, lens = pack_units([blobs[i] for i in pick])
        return t(buf), t(offs), t(lens), int(lens.sum())

    cols = {"lzma2": columns([p for p, _ in payloads])}
    for c in CHECKS:
        cols[c] = columns(archives[c])
    d_dict = t(np.array([payloads[i][1] for i in pick], dtype=np.uint8))
    d_out = torch.empty(n * UNIT + 64, dtype=torch.uint8, device=dev)
    d_ooff = t(np.arange(n, dtype=np.uint64) * np.uint64(UNIT))
    d_ocap = t(np.full(n, UNIT, dtype=np.uint64))
    d_len = torch.zeros(n, dtype=torch.int64, device=dev)
    d_used = torch.zeros(n, dtype=torch.int64, device=dev)
    d_st = torch.zeros(n, dtype=torch.int32, device=dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(v):
        d_in, d_off, d_ilen, _ = cols[v]
        if v == "lzma2":
            rc = L.swc_lzma2_decompress_batch(p(d_in), p(d_off), p(d_ilen), p(d_dict), p(d_out), p(d_ooff), p(d_ocap), p(d_len),
                                              p(d_used), p(d_st), n, stream())
        else:
            rc = L.swc_xz_unarchive_batch(p(d_in), p(d_off), p(d_ilen), p(d_out), p(d_ooff), p(d_ocap), p(d_len), p(d_st), n,
                                          stream())
        assert rc == 0, (v, rc)

    variants = ["lzma2"] + list(CHECKS)
    reference = None
    for v in variants:                                                # correctness and warm-up of every variant
        d_st.fill_(-1)
        run(v)
        torch.cuda.synchronize()
        assert (d_st == 0).all().item() and (d_len == UNIT).all().item(), v
        if reference is None:                                         # the raw batch: every unit against its source text
            reference = d_out[: n * UNIT].clone()
            host = reference.view(n, UNIT)[: args.distinct].cpu().numpy()
            assert all(host[i].tobytes() == raws[i] for i in range(args.distinct))
            assert torch.equal(reference.view(n, UNIT), reference.view(n, UNIT)[torch.tensor(pick, device=dev)])
        assert torch.equal(d_out[: n * UNIT], reference), v            # every variant: all n units, byte for byte
    for _ in range(args.warmup - 1):
        for v in variants:
            run(v)
    torch.cuda.synchronize()
    times = {v: [] for v in variants}
    for _ in range(args.steps):
        for v in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(v)
            e1.record()
            e1.synchronize()
            times[v].append(e0.elapsed_time(e1))
    lw, xw = C.c_int32(), C.c_int32()
    assert L.swc_xz_occupancy(C.byref(lw), C.byref(xw)) == 0
    med = {v: float(np.median(times[v])) for v in variants}
    print(json.dumps({
        "workload": "config 5: %d x 1 MiB text, preset 6, 1 MiB dictionary (%d distinct)" % (n, args.distinct),
        "gpu": gpu_identity(),
        "warps_per_sm": {"lzma_kernel": lw.value, "xz_kernel": xw.value},
        "median_ms": {v: round(med[v], 2) for v in variants},
        "all_ms": {v: [round(x, 2) for x in times[v]] for v in variants},
        "vs_lzma2_pct": {v: round(100 * (med[v] / med["lzma2"] - 1), 2) for v in CHECKS},
        "input_bytes": {v: cols[v][3] for v in variants},
        "output_GBps": {v: round(n * UNIT / med[v] / 1e6, 3) for v in variants},
    }))


if __name__ == "__main__":
    main()
