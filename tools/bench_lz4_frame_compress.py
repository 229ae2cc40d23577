#!/usr/bin/env python3
"""What the LZ4 frame layer costs on the compress side: the same 64 KiB blocks as raw blocks through
swc_lz4_block_compress_batch and as whole frames through swc_lz4_frame_compress_batch (caller scratch, exact max_blocks).
In one process, alternating, CUDA events around whole calls.  The input is 64 distinct 64 KiB blocks (80 % text-like, 10 %
zeros, 10 % random), tiled on the device; every frame of a shape is the same 16 MiB input, so every frame must equal the
first on the device, and the first equals the CPU restatement of LZ4.compress (oracle/swco_lz4c.py).

    python tools/bench_lz4_frame_compress.py [--blocks 65536] [--steps 5] [--warmup 1]

Shapes (T = --blocks): (raw) T raw blocks; (a) T/256 independent frames x 256 blocks, no checksums; (b) (a) with block and
content checksums; (c) (a) with dependent blocks; (d) the default options of LZ4.compress(data:) (4 MiB blocks, content
checksum) on the same bytes; (e) (a) replayed from a CUDA graph.  Prints one JSON line with the GPU's name and power limit,
per shape the median call time and GB/s of input, and the stage intervals of one call with swc_timing_enable."""
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

BLOCK = 64 << 10
PER_FRAME = 256
SCRATCH = 16 << 30


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def stage_names(k):
    """the intervals swc_timing_collect gives for one frame batch of s slices (k = 5 s + 3)"""
    s = (k - 3) // 5
    if k != 5 * s + 3 or s < 1:
        return [str(i) for i in range(k)]
    names = ["place+fill"]
    for i in range(s):
        names += (["slice gap"] if i else []) + ["chain", "parse", "layout", "emit"]
    return names + ["block xxh32", "content xxh32", "finish"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    T = args.blocks
    assert T % PER_FRAME == 0 and PER_FRAME % 64 == 0
    import helpers as H
    import swco_lz4c
    import torch
    from swcompression_b200 import LZ4, _lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    rng = random.Random(4)
    distinct = [bytes(BLOCK) if i % 10 == 8 else H.random_bytes(rng, BLOCK) if i % 10 == 9 else H.textlike(BLOCK, 500 + i)
                for i in range(64)]
    frame_in = b"".join(distinct) * (PER_FRAME // 64)
    nf, total = T // PER_FRAME, T * BLOCK
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)
    d_in = torch.cat([t(np.frombuffer(frame_in, dtype=np.uint8)).repeat(nf), torch.zeros(64, dtype=torch.uint8, device=dev)])
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    scratch = torch.empty(SCRATCH, dtype=torch.uint8, device=dev)   # the calls follow each other on one stream and share it

    blk_off, blk_len = t(np.arange(T, dtype=np.uint64) * np.uint64(BLOCK)), t(np.full(T, BLOCK, dtype=np.uint64))
    blk_cap = BLOCK + BLOCK // 255 + 64
    raw = dict(ooff=t(np.arange(T, dtype=np.uint64) * np.uint64(blk_cap)), ocap=t(np.full(T, blk_cap, dtype=np.uint64)),
               ln=torch.zeros(T, dtype=torch.int64, device=dev), st=torch.zeros(T, dtype=torch.int32, device=dev))
    opts = {
        "a_independent": dict(independentBlocks=True, blockChecksums=False, contentChecksum=False, contentSize=False, blockSize=BLOCK),
        "b_checksums": dict(independentBlocks=True, blockChecksums=True, contentChecksum=True, contentSize=False, blockSize=BLOCK),
        "c_dependent": dict(independentBlocks=False, blockChecksums=False, contentChecksum=False, contentSize=False, blockSize=BLOCK),
        "d_defaults": dict(independentBlocks=True, blockChecksums=False, contentChecksum=True, contentSize=False, blockSize=4 << 20),
    }
    f_off, f_len = t(np.arange(nf, dtype=np.uint64) * np.uint64(len(frame_in))), t(np.full(nf, len(frame_in), dtype=np.uint64))
    frames = {}
    for name, o in opts.items():
        cap = LZ4.max_compressed_size(len(frame_in), o["blockChecksums"], o["contentChecksum"], o["contentSize"], o["blockSize"])
        stride = (cap + 15) // 16 * 16
        frames[name] = dict(o=o, cap=cap, stride=stride, nblk=nf * -(-len(frame_in) // o["blockSize"]),
                            ooff=t(np.arange(nf, dtype=np.uint64) * np.uint64(stride)), ocap=t(np.full(nf, cap, dtype=np.uint64)),
                            ln=torch.zeros(nf, dtype=torch.int64, device=dev), st=torch.zeros(nf, dtype=torch.int32, device=dev))
    d_out = torch.empty(max(T * blk_cap, max(f["stride"] * nf for f in frames.values())) + 64, dtype=torch.uint8, device=dev)

    def run(name):
        if name == "raw_blocks":
            rc = L.swc_lz4_block_compress_batch(p(d_in), p(blk_off), p(blk_len), None, None, p(d_out), p(raw["ooff"]), p(raw["ocap"]),
                                                p(raw["ln"]), p(raw["st"]), T, p(scratch), scratch.numel(), stream())
        else:
            f = frames[name]
            o = f["o"]
            rc = L.swc_lz4_frame_compress_batch(p(d_in), p(f_off), p(f_len), int(o["independentBlocks"]), int(o["blockChecksums"]),
                                                int(o["contentChecksum"]), int(o["contentSize"]), o["blockSize"], None, 0, 0, 0,
                                                p(d_out), p(f["ooff"]), p(f["ocap"]), p(f["ln"]), p(f["st"]), nf, f["nblk"],
                                                p(scratch), scratch.numel(), stream())
        assert rc == 0, (name, rc)

    stages = {}
    for name in ["raw_blocks"] + list(frames):                       # correctness, warm-up and stage intervals of every shape
        L.swc_timing_enable(1)
        run(name)
        torch.cuda.synchronize()
        tb = (C.c_float * 256)()
        k = L.swc_timing_collect(tb, 256)
        L.swc_timing_enable(0)
        if name == "raw_blocks":
            assert (raw["st"] == 0).all().item()
            continue
        f = frames[name]
        names = stage_names(k)
        agg = {}
        for i in range(k):
            agg[names[i]] = round(agg.get(names[i], 0.0) + tb[i], 3)
        stages[name] = agg
        ln = int(f["ln"][0].item())
        assert (f["st"] == 0).all().item() and (f["ln"] == ln).all().item(), name
        out = d_out[: nf * f["stride"]].view(nf, f["stride"])[:, :ln]
        assert bool((out == out[0:1]).all()), name
        assert bytes(out[0].cpu().numpy()) == swco_lz4c.lz4_compress(frame_in, **f["o"])[1], name
        del out
    # (e): (a) captured once, then replayed
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            run("a_independent")
    torch.cuda.synchronize()
    shapes = ["raw_blocks"] + list(frames) + ["e_graph_replay"]

    def timed(name):
        if name == "e_graph_replay":
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
    assert (frames["a_independent"]["st"] == 0).all().item()
    med = {name: float(np.median(times[name])) for name in shapes}
    print(json.dumps({
        "workload": "%d blocks of 64 KiB (64 distinct: 80%% text-like, 10%% zeros, 10%% random), %.1f GiB of input per call, "
                    "%d frames of %d MiB" % (T, total / 2 ** 30, nf, len(frame_in) >> 20),
        "gpu": gpu_identity(),
        "median_ms": {k: round(v, 3) for k, v in med.items()},
        "all_ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "input_GBps": {k: round(total / v / 1e6, 3) for k, v in med.items()},
        "vs_raw_pct": {k: round(100 * (v / med["raw_blocks"] - 1), 1) for k, v in med.items()},
        "frame_bytes": {k: int(f["ln"][0].item()) for k, f in frames.items()},
        "stage_ms": stages,
    }))


if __name__ == "__main__":
    main()
