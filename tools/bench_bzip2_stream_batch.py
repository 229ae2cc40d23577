#!/usr/bin/env python3
"""What block-parallel BZip2 decoding buys: swc_bzip2_stream_decompress_batch (blocks of all streams side by side, caller
scratch and an exact max_blocks: the form a CUDA graph can hold) against swc_bzip2_decompress_batch (one warp per stream),
alternating in one process, CUDA events around whole calls.  The streams are bz2.compress(x, 9) of text-like data.  Every
unit's status and length is checked, and each shape's whole output of the new batch is compared with the old batch's.

    python tools/bench_bzip2_stream_batch.py [--steps 3] [--warmup 1] [--old-steps-b 1]

Shapes: (a) 2 048 streams of 900 000 B (BASELINE §4.1 config 4: 64 distinct, tiled; libbzip2's level-9 block holds
899 981 bytes, so each stream is one full block and one of 19 bytes); (b) 32 streams of 16 MiB (19 blocks each; 4 distinct,
tiled); (c) shape (b) replayed from a CUDA graph.  The new batch's scratch (one slot per block) and the old batch's pool do
not fit an 80 GB card together for shape (a), so each is allocated before its call and freed after it, outside the timed
window.  Also a sweep of the old batch over 16 .. 24 config-4 streams per SM, where the call time steps up once the warps no longer fit on the card at once
(the resident warps per SM of bzip2_kernel).  Prints one JSON line with the GPU's name, power limit and maximum SM clock, per shape the median
call time and GB/s of decoded bytes, and the stage intervals of one new call with swc_timing_enable."""
import argparse
import bz2
import ctypes as C
import json
import os
import subprocess
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PIECE = 900000
STAGES = ["scan+place+fill", "blocks+layout+copy", "resolve", "fallback"]


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def _piece(seed):
    import helpers as H
    return H.textlike(PIECE, seed)


def _compress(raw):
    return bz2.compress(raw, 9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--old-steps-b", type=int, default=1)
    args = ap.parse_args()
    import torch
    from swcompression_b200 import _lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    with Pool(min(32, os.cpu_count() or 1)) as pool:
        pieces = pool.map(_piece, range(4, 4 + 64))                       # config 4's seeds
        big_raw = [b"".join(pieces[(7 * s + k) % 64] for k in range(19))[:16 << 20] for s in range(4)]
        small = pool.map(_compress, pieces)
        big = pool.map(_compress, big_raw)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def tiled(blobs, n, size):
        """n units, unit u = blobs[u % len(blobs)] 16-byte aligned, regions of `size` bytes -> the device columns"""
        k = len(blobs)
        stride = [(len(b) + 15) // 16 * 16 for b in blobs]
        one = np.zeros(sum(stride), dtype=np.uint8)
        starts = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint64)
        for b, s in zip(blobs, starts):
            one[int(s):int(s) + len(b)] = np.frombuffer(b, dtype=np.uint8)
        d_buf = torch.cat([t(one).repeat(n // k), torch.zeros(64, dtype=torch.uint8, device=dev)])
        u = np.arange(n, dtype=np.uint64)
        offs = (u // np.uint64(k)) * np.uint64(len(one)) + starts[(u % np.uint64(k)).astype(np.int64)]
        lens = np.array([len(b) for b in blobs], dtype=np.uint64)[(u % np.uint64(k)).astype(np.int64)]
        return dict(n=n, size=size, d_in=d_buf, off=t(offs), len=t(lens), ooff=t(u * np.uint64(size)),
                    ocap=t(np.full(n, size, dtype=np.uint64)), ln=torch.zeros(n, dtype=torch.int64, device=dev),
                    used=torch.zeros(n, dtype=torch.int64, device=dev), st=torch.zeros(n, dtype=torch.int32, device=dev),
                    out=torch.empty(n * size + 64, dtype=torch.uint8, device=dev))

    def blocks_of(stream_bytes):
        bits = bin(int.from_bytes(b"\x01" + stream_bytes, "big"))[3:]
        return bits.count(format(0x314159265359, "048b"))

    def old(s):
        assert L.swc_bzip2_decompress_batch(p(s["d_in"]), p(s["off"]), p(s["len"]), p(s["out"]), p(s["ooff"]), p(s["ocap"]),
                                            p(s["ln"]), p(s["used"]), p(s["st"]), s["n"], stream()) == 0

    def new(s):
        assert L.swc_bzip2_stream_decompress_batch(p(s["d_in"]), p(s["off"]), p(s["len"]), p(s["out"]), p(s["ooff"]),
                                                   p(s["ocap"]), p(s["ln"]), p(s["used"]), p(s["st"]), s["n"], s["mb"],
                                                   p(s["scratch"]), s["scratch"].numel(), stream()) == 0

    def timed(fn, s, steps):
        ms = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(s)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms

    def check(s, raws):
        assert (s["st"] == 0).all().item() and (s["ln"] == s["size"]).all().item()
        host = s["out"][:len(raws) * s["size"]].cpu().numpy()
        assert all(host[i * s["size"]:(i + 1) * s["size"]].tobytes() == r for i, r in enumerate(raws))

    out = {"gpu": gpu_identity(), "gpu_fields": "name, power limit, maximum SM clock (clocks.max.sm)", "sms": sms}
    results, stages = {}, {}
    L.swc_release_scratch.restype = C.c_int32
    for name, blobs, raws, n, size in (("a", small, pieces, 2048, PIECE), ("b", big, big_raw, 32, 16 << 20)):
        s = tiled(blobs, n, size)
        s["mb"] = sum(blocks_of(b) for b in blobs) * (n // len(blobs))
        scratch_bytes = L.swc_bzip2_stream_batch_scratch_bytes(n, s["mb"], n * size)

        def with_scratch(fn):
            """the new batch with its whole scratch, which is freed again: with the old batch's pool beside it, shape (a)'s
            scratch (one slot per block) would not fit an 80 GB card"""
            s["scratch"] = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
            r = fn()
            del s["scratch"]
            torch.cuda.empty_cache()
            return r

        def with_pool(fn):
            """the old batch, its pool grown by an untimed call first and released after"""
            old(s)
            torch.cuda.synchronize()
            r = fn()
            L.swc_release_scratch()
            return r

        def first_new():
            L.swc_timing_enable(1)
            new(s)
            torch.cuda.synchronize()
            tb = (C.c_float * 16)()
            k = L.swc_timing_collect(tb, 16)
            L.swc_timing_enable(0)
            return {STAGES[i] if k == len(STAGES) else str(i): round(tb[i], 3) for i in range(k)}

        stages[name] = with_scratch(first_new)
        check(s, raws)
        reference = s["out"][:n * size].cpu()
        s["out"].zero_()
        with_pool(lambda: None)
        check(s, raws)
        assert torch.equal(s["out"][:n * size].cpu(), reference), name
        ms_new, ms_old = [], []
        old_steps = args.steps if name == "a" else args.old_steps_b
        for i in range(args.steps):                                        # alternating
            ms_new += with_scratch(lambda: [timed(new, s, 1 + args.warmup)[-1]])
            if i < old_steps:
                ms_old += with_pool(lambda: timed(old, s, 1))
        results[name] = dict(new_ms=[round(x, 1) for x in ms_new], old_ms=[round(x, 1) for x in ms_old], blocks=s["mb"],
                             scratch_GB=round(scratch_bytes / 1e9, 2))
        if name == "b":                                                    # (c): the same call replayed from a CUDA graph
            s["scratch"] = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
            new(s)
            s["st"].fill_(-1); s["out"].zero_()
            torch.cuda.synchronize()
            cs = torch.cuda.Stream()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(cs):
                with torch.cuda.graph(g, stream=cs):
                    new(s)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(s["out"][:n * size].cpu(), reference)
            ms_graph = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                ms_graph.append(e0.elapsed_time(e1))
            results["c"] = dict(graph_ms=[round(x, 1) for x in ms_graph])
            del g, s["scratch"]
        del s, reference
        torch.cuda.empty_cache()
    # the old batch's call time over 16 .. 24 single-block streams per SM
    sweep = {}
    for per_sm in (16, 18, 20, 21, 22, 24):
        s = tiled(small, 64 * ((per_sm * sms + 63) // 64), PIECE)
        old(s)
        torch.cuda.synchronize()
        sweep[per_sm] = round(float(np.median(timed(old, s, 2))), 1)
        del s
    out["old_sweep_ms_by_streams_per_sm"] = sweep
    L.swc_release_scratch()

    summary = {}
    for name in ("a", "b"):
        r = results[name]
        mn, mo = float(np.median(r["new_ms"])), float(np.median(r["old_ms"]))
        total = (2048 * PIECE) if name == "a" else 32 * (16 << 20)
        summary[name] = dict(new_median_ms=round(mn, 1), old_median_ms=round(mo, 1), speedup=round(mo / mn, 2),
                             new_GBps=round(total / mn / 1e6, 2), old_GBps=round(total / mo / 1e6, 2))
    summary["c"] = dict(graph_median_ms=round(float(np.median(results["c"]["graph_ms"])), 1))
    out.update(summary=summary, runs=results, stage_ms=stages)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
