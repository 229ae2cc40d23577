#!/usr/bin/env python3
"""What the gzip / zlib framing costs on the compress side: the same 64 KiB units as raw Deflate streams through
swc_deflate_compress_batch, as gzip members through swc_gzip_archive_batch and as zlib streams through
swc_zlib_archive_batch (caller scratch, max_in_bytes = the batch's input), and the gzip batch replayed from a CUDA graph.
In one process, alternating, CUDA events around whole calls.  The input is 64 distinct 64 KiB units (80 % text-like, 10 %
zeros, 10 % random), tiled on the device; every tile must equal the first on the device, and the first 64 units equal the
CPU restatement of GzipArchive.archive / ZlibArchive.archive (oracle/swco_deflatec.py).

    python tools/bench_archive_batch.py [--units 65536] [--steps 3] [--warmup 1] [--other-lib PATH]

--other-lib loads a second build of libswcgpu.so (for example the previous commit's) and adds its raw batch on the same
data as shape "raw_other", alternating with this build's: a regression check of the raw batch in one session.  Prints one
JSON line with the GPU's name and power limit, per shape the median call time and GB/s of input, and the stage intervals
of one call with swc_timing_enable."""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

UNIT = 64 << 10
ARCHIVE_STAGES = ["place", "checksum", "link", "parse", "emit", "seam", "finish"]
RAW_STAGES = ["link", "parse", "emit", "seam"]


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--other-lib", default=None)
    args = ap.parse_args()
    T = args.units
    assert T % 64 == 0
    import helpers as H
    import swco_deflatec
    import torch
    from swcompression_b200 import GzipArchive, ZlibArchive, _lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    O = None
    if args.other_lib:
        O = C.CDLL(os.path.abspath(args.other_lib))
        O.swc_deflate_compress_batch.argtypes = L.swc_deflate_compress_batch.argtypes
    rng = random.Random(4)
    distinct = [bytes(UNIT) if i % 10 == 8 else H.random_bytes(rng, UNIT) if i % 10 == 9 else H.textlike(UNIT, 500 + i)
                for i in range(64)]
    tile, total = T // 64, T * UNIT
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)
    d_in = torch.cat([t(np.frombuffer(b"".join(distinct), dtype=np.uint8)).repeat(tile), torch.zeros(64, dtype=torch.uint8, device=dev)])
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    in_off, in_len = t(np.arange(T, dtype=np.uint64) * np.uint64(UNIT)), t(np.full(T, UNIT, dtype=np.uint64))
    opts = dict(fileName="member.bin", modificationTime=1700000000)
    hdr = GzipArchive.archive_header(**opts)
    d_hdr = t(np.frombuffer(hdr, dtype=np.uint8).copy())
    h_off, h_len = t(np.zeros(T, dtype=np.uint64)), t(np.full(T, len(hdr), dtype=np.uint64))
    caps = {"raw": (9 * UNIT + 17) // 8, "gzip": GzipArchive.max_archive_size(UNIT, **opts), "zlib": ZlibArchive.max_archive_size(UNIT)}
    # one output buffer at the largest stride; every shape writes unit i at i x its own 16-byte-rounded capacity
    cols = {}
    for k, cap in caps.items():
        stride = (cap + 15) // 16 * 16
        cols[k] = dict(cap=cap, stride=stride, ooff=t(np.arange(T, dtype=np.uint64) * np.uint64(stride)),
                       ocap=t(np.full(T, cap, dtype=np.uint64)), ln=torch.zeros(T, dtype=torch.int64, device=dev),
                       st=torch.zeros(T, dtype=torch.int32, device=dev))
    d_out = torch.empty(max(c["stride"] for c in cols.values()) * T + 64, dtype=torch.uint8, device=dev)
    nbytes = max(L.swc_archive_compress_batch_scratch_bytes(T, total), L.swc_deflate_compress_batch_scratch_bytes(T, total))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)       # the calls follow each other on one stream and share it

    def run(name):
        c = cols["raw" if name.startswith("raw") else name]
        if name.startswith("raw"):
            lib = O if name == "raw_other" else L
            rc = lib.swc_deflate_compress_batch(p(d_in), p(in_off), p(in_len), p(d_out), p(c["ooff"]), p(c["ocap"]), p(c["ln"]),
                                                p(c["st"]), T, p(scratch), scratch.numel(), stream())
        elif name == "gzip":
            rc = L.swc_gzip_archive_batch(p(d_in), p(in_off), p(in_len), p(d_hdr), p(h_off), p(h_len), p(d_out), p(c["ooff"]),
                                          p(c["ocap"]), p(c["ln"]), p(c["st"]), T, total, p(scratch), scratch.numel(), stream())
        else:
            rc = L.swc_zlib_archive_batch(p(d_in), p(in_off), p(in_len), p(d_out), p(c["ooff"]), p(c["ocap"]), p(c["ln"]),
                                          p(c["st"]), T, total, p(scratch), scratch.numel(), stream())
        assert rc == 0, (name, rc)

    def check(name):
        c = cols["raw" if name.startswith("raw") else name]
        assert (c["st"] == 0).all().item(), name
        ln = c["ln"].cpu().numpy()
        assert (ln.reshape(tile, 64) == ln[:64][None, :]).all(), name
        if name.startswith("raw"):
            exp = [swco_deflatec.deflate_compress(u)[1] for u in distinct]
        elif name == "gzip":
            exp = [swco_deflatec.gzip_archive(u, fileName=b"member.bin", modificationTime=1700000000)[1] for u in distinct]
        else:
            exp = [swco_deflatec.zlib_archive(u)[1] for u in distinct]
        out = d_out[: T * c["stride"]].view(tile, 64, c["stride"])
        assert all(bool((out[:, j, :int(ln[j])] == out[0:1, j, :int(ln[j])]).all()) for j in range(64)), name
        host = out[0].cpu().numpy()
        for j, e in enumerate(exp):
            assert int(ln[j]) == len(e) and bytes(host[j, :len(e)]) == e, (name, j)
        del out

    shapes = ["raw"] + (["raw_other"] if O else []) + ["gzip", "zlib"]
    stages = {}
    for name in shapes:                                               # correctness, warm-up and stage intervals
        L.swc_timing_enable(1)
        run(name)
        torch.cuda.synchronize()
        tb = (C.c_float * 256)()
        k = L.swc_timing_collect(tb, 256)
        L.swc_timing_enable(0)
        check(name)
        if name == "raw_other":
            continue
        names = RAW_STAGES if name == "raw" else ARCHIVE_STAGES
        stages[name] = {names[i] if k == len(names) else str(i): round(tb[i], 3) for i in range(k)}
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            run("gzip")
    torch.cuda.synchronize()
    shapes.append("gzip_graph_replay")

    def timed(name):
        if name == "gzip_graph_replay":
            g.replay()
        else:
            run(name)

    for _ in range(args.warmup):
        for name in shapes:
            timed(name)
    torch.cuda.synchronize()
    times = {name: [] for name in shapes}
    for _ in range(args.steps):
        for name in shapes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            timed(name)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    check("gzip")
    med = {name: float(np.median(times[name])) for name in shapes}
    print(json.dumps({
        "workload": "%d units of 64 KiB (64 distinct: 80%% text-like, 10%% zeros, 10%% random), %.1f GiB of input per call"
                    % (T, total / 2 ** 30),
        "gpu": gpu_identity(),
        "median_ms": {k: round(v, 3) for k, v in med.items()},
        "all_ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "input_GBps": {k: round(total / v / 1e6, 3) for k, v in med.items()},
        "vs_raw_pct": {k: round(100 * (v / med["raw"] - 1), 2) for k, v in med.items()},
        "output_bytes": {k: int(cols[k]["ln"].sum().item()) for k in ("raw", "gzip", "zlib")},
        "stage_ms": stages,
    }))


if __name__ == "__main__":
    main()
