#!/usr/bin/env python3
"""What the LZ4 frame layer costs on the device: the same 64 KiB blocks as raw blocks through swc_lz4_block_decompress_batch
and as frames of several shapes through swc_lz4_frame_decompress_batch (caller scratch, exact max_blocks: the form a CUDA
graph can hold).  In one process, alternating, CUDA events around whole calls.  The blocks are 32 distinct text-like 64 KiB
inputs, tiled; the frames are written by the product's LZ4.compress.  Every unit's status and length is checked and every
shape's whole output is compared with the raw batch's.

    python tools/bench_lz4_frame_batch.py [--blocks 65536] [--steps 5] [--warmup 1]

Shapes (T = --blocks): (a) T raw blocks; (b) T/64 independent frames x 64 blocks; (c) with block checksums; (d) with content
checksum; (e) T/64 dependent frames x 64 blocks; (f) 16 independent frames x T/16 blocks with content checksum; (g) T one-block
frames; (h) 256 frames of (b) one by one through swc_lz4_decompress (host memory in and out), per frame.
Prints one JSON line with the GPU's name and power limit, per shape the median call time and GB/s of decoded bytes, and the
stage intervals of one call with swc_timing_enable."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BLOCK = 64 << 10
DISTINCT = 32
STAGES = ["walk+place+fill", "parse", "block xxh32", "chain", "resolve", "exec", "fallback", "content xxh32"]


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    T = args.blocks
    assert T % 1024 == 0
    import helpers as H
    import torch
    from swcompression_b200 import _lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    pieces = [H.textlike(BLOCK, 4100 + k) for k in range(DISTINCT)]
    round32 = b"".join(pieces)

    def compress(data, independent, block_ck=False, content_ck=False):
        buf, n = _lib.inbuf(data)
        out, ol = C.c_void_p(), C.c_size_t()
        assert L.swc_lz4_compress(buf, n, independent, block_ck, content_ck, 0, BLOCK, None, 0, 0, 0, C.byref(out), C.byref(ol)) == 0
        return _lib.take(out, ol)

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)

    def tiled(blobs, n):
        """n units, unit u = blobs[u % len(blobs)], 16-byte aligned -> device (buffer, offsets, lengths), input bytes"""
        k = len(blobs)
        stride = [(len(b) + 15) // 16 * 16 for b in blobs]
        one = np.zeros(sum(stride), dtype=np.uint8)
        starts = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint64)
        for b, s in zip(blobs, starts):
            one[int(s):int(s) + len(b)] = np.frombuffer(b, dtype=np.uint8)
        assert n % k == 0
        d_one = t(one)
        d_buf = torch.cat([d_one.repeat(n // k), torch.zeros(64, dtype=torch.uint8, device=dev)])
        u = np.arange(n, dtype=np.uint64)
        offs = (u // np.uint64(k)) * np.uint64(len(one)) + starts[(u % np.uint64(k)).astype(np.int64)]
        lens = np.array([len(b) for b in blobs], dtype=np.uint64)[(u % np.uint64(k)).astype(np.int64)]
        return d_buf, t(offs), t(lens), int(lens.sum())

    one_block = [compress(p, True) for p in pieces]
    raw_blocks = [f[11:-4] for f in one_block]                          # magic, FLG, BD, HC, block mark | payload | EndMark
    shapes = {
        "a_raw_blocks": (tiled(raw_blocks, T), T, 1),
        "b_independent_64": (tiled([compress(round32 * 2, True)], T // 64), T // 64, 64),
        "c_block_checksums": (tiled([compress(round32 * 2, True, block_ck=True)], T // 64), T // 64, 64),
        "d_content_checksum": (tiled([compress(round32 * 2, True, content_ck=True)], T // 64), T // 64, 64),
        "e_dependent_64": (tiled([compress(round32 * 2, False)], T // 64), T // 64, 64),
        "f_16_huge_frames": (tiled([compress(round32 * (T // 16 // 32), True, content_ck=True)], 16), 16, T // 16),
        "g_one_block_frames": (tiled(one_block, T), T, 1),
    }
    host_frame = compress(round32 * 2, True)
    total = T * BLOCK
    d_out = torch.empty(total + 64, dtype=torch.uint8, device=dev)
    p = lambda x: None if x is None else C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    state = {}
    # the calls follow each other on one stream: one scratch, sized for the largest shape, serves them all
    scratch = torch.empty(max(L.swc_lz4_frame_batch_scratch_bytes(n, c[3], T) for c, n, _ in shapes.values()), dtype=torch.uint8,
                          device=dev)
    for name, ((d_in, d_off, d_len, in_bytes), n, per) in shapes.items():
        size = per * BLOCK
        state[name] = dict(ooff=t(np.arange(n, dtype=np.uint64) * np.uint64(size)), ocap=t(np.full(n, size, dtype=np.uint64)),
                           ln=torch.zeros(n, dtype=torch.int64, device=dev), used=torch.zeros(n, dtype=torch.int64, device=dev),
                           st=torch.zeros(n, dtype=torch.int32, device=dev), scratch=scratch, size=size)

    def run(name):
        (d_in, d_off, d_len, _), n, _ = shapes[name]
        s = state[name]
        if name == "a_raw_blocks":
            rc = L.swc_lz4_block_decompress_batch(p(d_in), p(d_off), p(d_len), None, 0, p(d_out), p(s["ooff"]), p(s["ocap"]),
                                                  p(s["ln"]), p(s["st"]), n, stream())
        else:
            rc = L.swc_lz4_frame_decompress_batch(p(d_in), p(d_off), p(d_len), None, 0, 0, 0, p(d_out), p(s["ooff"]), p(s["ocap"]),
                                                  p(s["ln"]), p(s["used"]), p(s["st"]), n, T, p(s["scratch"]),
                                                  s["scratch"].numel(), stream())
        assert rc == 0, (name, rc)

    reference = None
    stages = {}
    for name in shapes:                                                # correctness, warm-up and stage intervals of every shape
        s = state[name]
        s["st"].fill_(-1)
        d_out.zero_()
        L.swc_timing_enable(1)
        run(name)
        torch.cuda.synchronize()
        tb = (C.c_float * 64)()
        k = L.swc_timing_collect(tb, 64)
        L.swc_timing_enable(0)
        if name != "a_raw_blocks":
            stages[name] = {STAGES[i] if k == len(STAGES) else str(i): round(tb[i], 3) for i in range(k)}
        assert (s["st"] == 0).all().item() and (s["ln"] == s["size"]).all().item(), name
        if name != "a_raw_blocks":
            assert (s["used"] == shapes[name][0][2]).all().item(), name
        if reference is None:
            reference = d_out[:total].clone()
            host = reference.view(T, BLOCK)[:DISTINCT].cpu().numpy()
            assert all(host[i].tobytes() == pieces[i] for i in range(DISTINCT))
        assert torch.equal(d_out[:total], reference), name
    for _ in range(args.warmup - 1):
        for name in shapes:
            run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in shapes}
    for _ in range(args.steps):
        for name in shapes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(name)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    buf, n = _lib.inbuf(host_frame)
    host_ms = []
    for i in range(256 + 8):                                           # (h): the host path, one frame per call
        out, ol, used = C.c_void_p(), C.c_size_t(), C.c_size_t()
        t0 = time.perf_counter()
        assert L.swc_lz4_decompress(buf, n, None, 0, 0, 0, C.byref(out), C.byref(ol), C.byref(used)) == 0
        host_ms.append((time.perf_counter() - t0) * 1e3)
        assert ol.value == 64 * BLOCK
        L.swc_free(out)
    med = {name: float(np.median(times[name])) for name in shapes}
    print(json.dumps({
        "workload": "%d blocks of 64 KiB text (%d distinct), %.1f GiB decoded per call" % (T, DISTINCT, total / 2 ** 30),
        "gpu": gpu_identity(),
        "median_ms": {k: round(v, 3) for k, v in med.items()},
        "all_ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "output_GBps": {k: round(total / v / 1e6, 1) for k, v in med.items()},
        "vs_raw_pct": {k: round(100 * (v / med["a_raw_blocks"] - 1), 1) for k, v in med.items()},
        "input_bytes": {k: v[0][3] for k, v in shapes.items()},
        "stage_ms": stages,
        "h_host_call_ms_per_4MiB_frame": round(float(np.median(host_ms[8:])), 3),
        "h_host_GBps": round(64 * BLOCK / float(np.median(host_ms[8:])) / 1e6, 2),
    }))


if __name__ == "__main__":
    main()
