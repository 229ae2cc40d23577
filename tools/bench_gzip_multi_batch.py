#!/usr/bin/env python3
"""The member-parallel gzip batch (swc_gzip_multi_unarchive_batch, Batch codec 'gzip_multi') on config 2's bytes as bgzip
stores them: the bytes cut into bgzip's 65 280-byte blocks (Deflate level 6, each a BGZF member) and written as 16 BGZF files
with the 28-byte EOF member.  The blocks are `--distinct` textlike blocks compressed once and tiled, so the CPU side takes
seconds.  In one process:

  (a) 'gzip_multi' over the 16 files against the 'gzip' batch over the same members as separate units (the upper bound:
      no scan, no spans, no validation), alternated step by step;
  (b) GzipArchive.multiUnarchive per file (host memory in and out, one file per call), once;
  (c) (a)'s batch captured into a CUDA graph with a caller scratch and max_members set, then replayed;
  (d) one plain-concatenation shape: the same members without the BC subfield (`cat a.gz b.gz ...`), 'gzip_multi'.

Calls are timed with CUDA events; every unit's status, out_len and parallel_members is checked and the outputs are
compared with the source blocks on the device.  One more call of (a) with swc_timing_enable gives the stage intervals.

    python tools/bench_gzip_multi_batch.py [--steps 5] [--warmup 1] [--gib 4] [--distinct 64]

Prints one JSON line with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

FILES = 16


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--distinct", type=int, default=64)
    args = ap.parse_args()
    import torch
    import gzip_member_cases as G
    import helpers as H
    import unarchive_cases as U
    from swcompression_b200.api import GzipArchive
    from swcompression_b200.batch import Batch
    log = lambda *m: print(*m, file=sys.stderr, flush=True)
    total = int(args.gib * (1 << 30))
    nblk = total // G.BGZF_BLOCK
    per = nblk // FILES
    raws = [H.textlike(G.BGZF_BLOCK, 4000 + i) for i in range(args.distinct)]
    bgzf_blobs = [G.bgzf_member(r) for r in raws]
    plain_blobs = [U.gzip_member(r) for r in raws]
    t0 = time.perf_counter()
    files = [b"".join(bgzf_blobs[(f * per + k) % args.distinct] for k in range(per)) + G.BGZF_EOF for f in range(FILES)]
    plain = [b"".join(plain_blobs[(f * per + k) % args.distinct] for k in range(per)) for f in range(FILES)]
    members = [bgzf_blobs[(f * per + k) % args.distinct] for f in range(FILES) for k in range(per)]
    log(f"built {FILES} files of {per} members ({sum(map(len, files)) / 1e9:.2f} GB) in {time.perf_counter() - t0:.1f} s")
    size = per * G.BGZF_BLOCK
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(b):
        a, z = ev(), ev()
        a.record(); b.run(); z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z)

    multi = Batch.from_units("gzip_multi", files, size)
    single = Batch.from_units("gzip", members, G.BGZF_BLOCK)
    ref = torch.from_numpy(np.frombuffer(b"".join(raws), dtype=np.uint8).copy()).cuda().view(args.distinct, G.BGZF_BLOCK)

    def check_multi(b, want_par):
        st, ln, used = b.results()
        assert (st == 0).all() and (ln == size).all(), (st, ln)
        assert (b.parallel_members() == want_par).all(), b.parallel_members()
        for f in range(FILES):
            o = int(b.h_out_off[f])
            got = b.d_out[o:o + size].view(per, G.BGZF_BLOCK)
            idx = torch.arange(f * per, (f + 1) * per, device="cuda") % args.distinct
            assert bool((got == ref[idx]).all()), f

    ms = {"gzip_multi": [], "gzip": []}
    for step in range(args.warmup + args.steps):
        for name, b in (("gzip_multi", multi), ("gzip", single)):
            t = timed(b)
            if step >= args.warmup:
                ms[name].append(t)
    check_multi(multi, per + 1)
    # the stage intervals of one more call: scan+place+fill, sort, span, the decode stage (unarchive_batch_impl), validate+fallback
    from swcompression_b200 import _lib
    import ctypes as C
    L = _lib.lib()
    torch.cuda.synchronize()
    L.swc_timing_enable(1)
    multi.run()
    torch.cuda.synchronize()
    iv = (C.c_float * 64)()
    k = L.swc_timing_collect(iv, 64)
    L.swc_timing_enable(0)
    iv = [iv[i] for i in range(k)]
    stages = ({"scan_place_fill_ms": iv[0], "sort_ms": iv[1], "span_ms": iv[2], "decode_ms": sum(iv[3:-1]),
               "validate_fallback_ms": iv[-1]} if k >= 5 else {})
    log("stages", stages)
    st, ln, _ = single.results()
    assert (st == 0).all() and (ln == G.BGZF_BLOCK).all()
    log("batches", {k: min(v) for k, v in ms.items()})
    # (b) the host API per file
    t = time.perf_counter()
    for f in files:
        parts = GzipArchive.multiUnarchive(f)
        assert len(parts) == per + 1
    host_ms = (time.perf_counter() - t) * 1e3
    log("host", host_ms)
    # (c) graph replay
    del single
    torch.cuda.empty_cache()
    gb = Batch.from_units("gzip_multi", files, size, max_members=FILES * (per + 1) + 64)
    gb.run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            gb.run()
    torch.cuda.synchronize()
    graph_ms = []
    for step in range(args.warmup + args.steps):
        gb.d_status.fill_(-1)
        a, z = ev(), ev()
        a.record(); g.replay(); z.record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            graph_ms.append(a.elapsed_time(z))
    check_multi(gb, per + 1)
    del gb, g, multi
    torch.cuda.empty_cache()
    # (d) plain concatenation
    pb = Batch.from_units("gzip_multi", plain, size)
    plain_ms = []
    for step in range(args.warmup + args.steps):
        t = timed(pb)
        if step >= args.warmup:
            plain_ms.append(t)
    check_multi(pb, per)
    out_bytes = FILES * size
    best = {k: min(v) for k, v in ms.items()}
    print(json.dumps({
        "gpu": gpu_identity(), "files": FILES, "members_per_file": per + 1, "decompressed_bytes": out_bytes,
        "compressed_bytes": sum(map(len, files)),
        "gzip_multi_ms": best["gzip_multi"], "gzip_members_as_units_ms": best["gzip"],
        "gzip_multi_GBps": out_bytes / best["gzip_multi"] / 1e6, "gzip_members_as_units_GBps": out_bytes / best["gzip"] / 1e6,
        "gzip_multi_over_gzip": best["gzip_multi"] / best["gzip"],
        "host_multiUnarchive_per_file_total_ms": host_ms, "graph_replay_ms": min(graph_ms),
        "plain_concatenation_ms": min(plain_ms), "stages": stages, "steps": args.steps, "all_ms": ms}))


if __name__ == "__main__":
    main()
