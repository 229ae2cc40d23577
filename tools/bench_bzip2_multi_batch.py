#!/usr/bin/env python3
"""What the block-parallel multi-stream batch costs and buys: swc_bzip2_multi_decompress_batch (every stream of every file,
blocks side by side, caller scratch and an exact max_blocks: the form a CUDA graph can hold) against the same streams as
separate units of swc_bzip2_stream_decompress_batch and swc_bzip2_decompress_batch, alternated in one process, CUDA
events around whole calls.  Streams are bz2.compress(x, 9) of seeded text from tests/helpers.textlike, compressed in a
process pool; every file's status, size, stream count, parallel_streams and bytes are checked.

    python tools/bench_bzip2_multi_batch.py [--steps 3] [--warmup 1]

Shapes: (a) 16 files of 74 streams of 900 000 B (pbzip2's layout, about 64 MiB each; 64 distinct pieces, tiled);
(b) 4 files of 2 000 streams of 64-256 KiB (the multistream-dump shape; 256 distinct streams, tiled); (c) 16 files of four
16 MiB multi-block streams; (d) shape (a) replayed from a CUDA graph.  Each shape's caller scratch holds one block slot per
block up to 40 GiB (shape (b)'s 8 000 blocks then run in slices), shared with the separate-unit batches.  Shape (a) is also timed through
BZip2.multiDecompress file by file (the single call, host in the loop).  Prints one JSON line with the GPU's name, power
limit and maximum SM clock, per shape the median call times and GB/s of decoded bytes, and the stage intervals of one
call of each shape with swc_timing_enable."""
import argparse
import bz2
import ctypes as C
import json
import os
import subprocess
import sys
import time
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PIECE = 900000
STAGES = ["scan+place+fill", "blocks+layout+copy", "resolve", "fallback"]
SCRATCH_CAP = 40 << 30


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def _raw(arg):
    import helpers as H
    n, seed = arg
    return H.textlike(n, seed)


def _compress(raw):
    return bz2.compress(raw, 9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    from swcompression_b200 import BZip2, _lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    rng = np.random.default_rng(5)
    small_sizes = [int(x) for x in rng.integers(64 << 10, 256 << 10, 256)]
    with Pool(min(32, os.cpu_count() or 1)) as pool:
        pieces = pool.map(_raw, [(PIECE, s) for s in range(4, 4 + 64)])
        smalls = pool.map(_raw, [(n, 1000 + i) for i, n in enumerate(small_sizes)])
        bigs = [b"".join(pieces[(7 * s + k) % 64] for k in range(19))[:16 << 20] for s in range(4)]
        c_pieces, c_smalls, c_bigs = pool.map(_compress, pieces), pool.map(_compress, smalls), pool.map(_compress, bigs)
    # each shape: files as lists of stream indices into (compressed, raw)
    shapes = {
        "a": (c_pieces, pieces, [[(f * 74 + k) % 64 for k in range(74)] for f in range(16)]),
        "b": (c_smalls, smalls, [[(f * 2000 + k * 7) % 256 for k in range(2000)] for f in range(4)]),
        "c": (c_bigs, bigs, [[(f + k) % 4 for k in range(4)] for f in range(16)]),
    }
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    magic = format(0x314159265359, "048b")
    blocks_of = lambda b: bin(int.from_bytes(b"\x01" + b, "big"))[3:].count(magic)

    def columns(units, sizes):
        """units packed 16-byte aligned, output regions of `sizes` bytes -> the device columns"""
        lens = np.array([len(u) for u in units], dtype=np.uint64)
        offs = np.concatenate([[0], np.cumsum((lens + np.uint64(15)) // np.uint64(16) * np.uint64(16))[:-1]]).astype(np.uint64)
        buf = np.zeros(int(offs[-1] + lens[-1]) + 64, dtype=np.uint8)
        for u, o in zip(units, offs):
            buf[int(o):int(o) + len(u)] = np.frombuffer(u, dtype=np.uint8)
        caps = np.array(sizes, dtype=np.uint64)
        ooff = np.concatenate([[0], np.cumsum((caps + np.uint64(15)) // np.uint64(16) * np.uint64(16))[:-1]]).astype(np.uint64)
        n = len(units)
        return dict(n=n, d_in=t(buf), off=t(offs), len=t(lens), ooff=t(ooff), ocap=t(caps), h_ooff=ooff, h_cap=caps,
                    ln=torch.zeros(n, dtype=torch.int64, device=dev), used=torch.zeros(n, dtype=torch.int64, device=dev),
                    st=torch.zeros(n, dtype=torch.int32, device=dev),
                    out=torch.empty(int(ooff[-1] + caps[-1]) + 64, dtype=torch.uint8, device=dev),
                    total=int(caps.sum()))

    def multi(s):
        assert L.swc_bzip2_multi_decompress_batch(p(s["d_in"]), p(s["off"]), p(s["len"]), p(s["out"]), p(s["ooff"]),
                                                  p(s["ocap"]), p(s["ln"]), p(s["st"]), p(s["ns"]), p(s["soff"]), p(s["scap"]),
                                                  p(s["send"]), p(s["sin"]), p(s["par"]), s["n"], s["mb"], p(s["scratch"]),
                                                  s["scratch"].numel(), stream()) == 0

    def stream_batch(s):
        assert L.swc_bzip2_stream_decompress_batch(p(s["d_in"]), p(s["off"]), p(s["len"]), p(s["out"]), p(s["ooff"]),
                                                   p(s["ocap"]), p(s["ln"]), p(s["used"]), p(s["st"]), s["n"], s["mb"],
                                                   p(s["scratch"]), s["scratch"].numel(), stream()) == 0

    def warp_batch(s):
        assert L.swc_bzip2_decompress_batch(p(s["d_in"]), p(s["off"]), p(s["len"]), p(s["out"]), p(s["ooff"]), p(s["ocap"]),
                                            p(s["ln"]), p(s["used"]), p(s["st"]), s["n"], stream()) == 0

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

    def stage_ms(fn, s):
        L.swc_timing_enable(1)
        fn(s)
        torch.cuda.synchronize()
        tb = (C.c_float * 16)()
        k = L.swc_timing_collect(tb, 16)
        L.swc_timing_enable(0)
        return {STAGES[i] if k == len(STAGES) else str(i): round(tb[i], 3) for i in range(k)}

    out = {"gpu": gpu_identity(), "gpu_fields": "name, power limit, maximum SM clock (clocks.max.sm)",
           "sms": torch.cuda.get_device_properties(dev).multi_processor_count}
    summary, runs, stages = {}, {}, {}
    for name, (comp, raws, files) in shapes.items():
        units = [b"".join(comp[k] for k in f) for f in files]
        wants = [[raws[k] for k in f] for f in files]
        sizes = [sum(len(w) for w in ws) for ws in wants]
        m = columns(units, sizes)
        n = m["n"]
        scap = np.array([len(f) + 1 for f in files], dtype=np.uint64)
        soff = np.concatenate([[0], np.cumsum(scap)[:-1]]).astype(np.uint64)
        m.update(ns=torch.zeros(n, dtype=torch.int64, device=dev), soff=t(soff), scap=t(scap),
                 send=torch.zeros(int(scap.sum()), dtype=torch.int64, device=dev),
                 sin=torch.zeros(int(scap.sum()), dtype=torch.int64, device=dev),
                 par=torch.zeros(n, dtype=torch.int32, device=dev))
        m["mb"] = sum(blocks_of(comp[k]) for f in files for k in f)
        # one slot per block where it fits SCRATCH_CAP (else the block stage runs in slices); the separate units share it
        nsep = sum(len(f) for f in files) if name in ("a", "b") else n
        full = max(L.swc_bzip2_stream_batch_scratch_bytes(k, m["mb"], m["total"] + 16 * nsep) for k in (n, nsep))
        m["scratch"] = torch.empty(min(full, SCRATCH_CAP), dtype=torch.uint8, device=dev)
        stages[name] = stage_ms(multi, m)
        # checks: statuses, sizes, stream counts, every stream from the block stage, bytes
        assert (m["st"] == 0).all().item() and m["ln"].cpu().tolist() == sizes
        assert m["ns"].cpu().tolist() == [len(f) for f in files] and m["par"].cpu().tolist() == [len(f) for f in files]
        host = m["out"].cpu().numpy()
        for i, ws in enumerate(wants):
            assert host[int(m["h_ooff"][i]):int(m["h_ooff"][i]) + sizes[i]].tobytes() == b"".join(ws), (name, i)
        del host
        r = dict(files=n, streams=sum(len(f) for f in files), blocks=m["mb"], multi_ms=[])
        # the same streams as separate units
        sep = None
        if name in ("a", "b"):
            flat = [k for f in files for k in f]
            sep = columns([comp[k] for k in flat], [len(raws[k]) for k in flat])
            sep["mb"] = m["mb"]
            r.update(stream_ms=[], warp_ms=[] if name == "a" else None)
        for _ in range(args.steps):                                       # alternating
            r["multi_ms"] += timed(multi, m, 1 + args.warmup)[-1:]
            if sep is not None:
                sep["scratch"] = m["scratch"]
                r["stream_ms"] += timed(stream_batch, sep, 1 + args.warmup)[-1:]
                assert (sep["st"] == 0).all().item()
                if name == "a":
                    warp_batch(sep)
                    r["warp_ms"] += timed(warp_batch, sep, 1)
                    assert (sep["st"] == 0).all().item()
                    L.swc_release_scratch()
        if sep is not None:
            stages[name + " separate units (stream batch)"] = stage_ms(stream_batch, sep)
            del sep
        med = lambda k: round(float(np.median(r[k])), 1)
        summary[name] = dict(multi_median_ms=med("multi_ms"), multi_GBps=round(m["total"] / med("multi_ms") / 1e6, 2))
        if "stream_ms" in r:
            summary[name].update(stream_units_median_ms=med("stream_ms"))
        if r.get("warp_ms"):
            summary[name].update(warp_units_median_ms=med("warp_ms"))
        if name == "a":
            # (d): the same call replayed from a CUDA graph
            cs = torch.cuda.Stream()
            cs.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(cs):
                with torch.cuda.graph(g, stream=cs):
                    multi(m)
            torch.cuda.synchronize()
            m["st"].fill_(-1)
            g.replay()
            torch.cuda.synchronize()
            assert (m["st"] == 0).all().item()
            ms_graph = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                ms_graph.append(e0.elapsed_time(e1))
            summary["d"] = dict(graph_median_ms=round(float(np.median(ms_graph)), 1))
            r["graph_ms"] = [round(x, 1) for x in ms_graph]
            del g
            # BZip2.multiDecompress file by file: host copy in, host loop, host copy out
            t0 = time.perf_counter()
            for i, u in enumerate(units):
                assert BZip2.multiDecompress(u) == wants[i]
            sec = time.perf_counter() - t0
            summary["a"].update(single_call_s_all_files=round(sec, 2))
        runs[name] = {k: ([round(x, 1) for x in v] if isinstance(v, list) else v) for k, v in r.items()}
        del m
        torch.cuda.empty_cache()
        L.swc_release_scratch()
    out.update(summary=summary, runs=runs, stage_ms=stages)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
