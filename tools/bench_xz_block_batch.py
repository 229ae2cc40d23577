#!/usr/bin/env python3
"""The block-parallel XZ batch (swc_xz_block_unarchive_batch) against the one-warp-per-file batch (swc_xz_unarchive_batch)
on the shape multi-threaded `xz` writes: independent 1 MiB blocks (LZMA2 preset 6, 1 MiB dictionary, CRC-64, both size
fields in every block header), framed by hand from a few distinct compressed blocks so the CPU side takes seconds.

  (a) config 5: 1 184 single-block 1 MiB files, old and new alternated in one process;
  (b) 16 files of 64 MiB in 1 MiB blocks (1 024 blocks): the new batch per step, the old batch once (--old-big 0 skips it);
  (c) (b) captured once into a CUDA graph with a caller scratch and max_blocks = 1 024, then replayed.

Whole calls are timed with CUDA events; every unit's status, out_len and parallel_blocks is checked and every output is
compared with its source on the device.  Per-stage intervals of the new batch come from swc_timing_collect.  --other-lib
adds swc_xz_unarchive_batch of another build (for example the previous commit's) to (a), alternated with this build's, so a
change to xz_kernel can be compared in one session.

    python tools/bench_xz_block_batch.py [--steps 5] [--warmup 1] [--distinct 8] [--old-big 1] [--other-lib PATH]

Prints one JSON line with the GPU's name and power limit."""
import argparse
import ctypes as C
import json
import os
import struct
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

UNIT = 1 << 20


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
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--old-big", type=int, default=1)
    ap.add_argument("--other-lib", default=None)
    args = ap.parse_args()
    import helpers as H
    import swco
    import xz_block_cases as XB
    import xz_cases as X
    # the checks of the distinct blocks, once each, by the oracle's CRC-64 (the test helper's is bitwise Python)
    checks = {}
    X.check_bytes = lambda check, raw: checks.setdefault(raw, struct.pack("<Q", swco.crc64(raw)))
    log = lambda *m: print(*m, file=sys.stderr, flush=True)
    raws = [H.textlike(UNIT, 40 + k) for k in range(args.distinct)]
    blocks = [(X.lzma2_raw(r, preset=6, dict_size=UNIT), 0x10, r) for r in raws]
    small_pick = [i % args.distinct for i in range(1184)]
    small = [XB.stream([blocks[i]], X.CHECK_CRC64, sizes=[True]) for i in range(args.distinct)]
    big_pick = [[(f + k) % args.distinct for k in range(64)] for f in range(16)]
    big = [XB.stream([blocks[i] for i in pk], X.CHECK_CRC64, sizes=[True] * 64) for pk in big_pick]

    log("inputs framed")
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import pack_units
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    L = _lib.lib()
    vp, u64 = C.c_void_p, C.c_uint64
    O = None
    if args.other_lib:
        O = C.CDLL(os.path.abspath(args.other_lib))
        O.swc_xz_unarchive_batch.argtypes = [vp] * 8 + [u64, vp]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    src = torch.from_numpy(np.frombuffer(b"".join(raws), dtype=np.uint8).copy()).to(dev).view(args.distinct, UNIT)

    class Shape:
        def __init__(self, files, pick_rows, unit_out):
            buf, offs, lens = pack_units(files)
            self.n = len(files)
            self.d_in, self.d_off, self.d_len = t(buf), t(offs), t(lens)
            self.unit_out = unit_out
            self.d_out = torch.empty(self.n * unit_out + 64, dtype=torch.uint8, device=dev)
            self.d_ooff = t(np.arange(self.n, dtype=np.uint64) * np.uint64(unit_out))
            self.d_ocap = t(np.full(self.n, unit_out, dtype=np.uint64))
            self.d_len_out = torch.zeros(self.n, dtype=torch.int64, device=dev)
            self.d_st = torch.zeros(self.n, dtype=torch.int32, device=dev)
            self.d_par = torch.zeros(self.n, dtype=torch.int32, device=dev)
            self.rows = torch.tensor(pick_rows, device=dev).view(-1)
            self.scratch = None
            self.input_bytes = int(lens.sum())

        def io(self):
            return (p(self.d_in), p(self.d_off), p(self.d_len), p(self.d_out), p(self.d_ooff), p(self.d_ocap), p(self.d_len_out),
                    p(self.d_st))

        def old(self, lib=None):
            assert (lib or L).swc_xz_unarchive_batch(*self.io(), self.n, stream()) == 0

        def new(self, max_blocks=0):
            sc = self.scratch
            assert L.swc_xz_block_unarchive_batch(*self.io(), p(self.d_par), self.n, max_blocks, None if sc is None else p(sc),
                                                  0 if sc is None else sc.numel(), stream()) == 0

        def check(self, blocks_each):
            torch.cuda.synchronize()
            assert (self.d_st == 0).all().item() and (self.d_len_out == self.unit_out).all().item()
            if blocks_each is not None:
                assert (self.d_par == blocks_each).all().item()
            got = self.d_out[: self.n * self.unit_out].view(-1, UNIT)
            assert torch.equal(got, src[self.rows])
            self.d_st.fill_(-1); self.d_len_out.zero_(); self.d_par.zero_(); self.d_out.zero_()

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    def stages(fn):
        L.swc_timing_enable(1)
        fn()
        torch.cuda.synchronize()
        ms = (C.c_float * 16)()
        k = L.swc_timing_collect(ms, 16)
        L.swc_timing_enable(0)
        return [round(ms[i], 3) for i in range(k)]

    # (a) config 5
    a = Shape([small[i] for i in small_pick], small_pick, UNIT)
    legs = {"old": lambda: a.old(), "new": lambda: a.new()}
    if O is not None:
        legs["old_other_lib"] = lambda: a.old(O)
    for name, fn in legs.items():
        fn()
        a.check(1 if name == "new" else None)
    for _ in range(args.warmup - 1):
        for fn in legs.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(args.steps):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    a.check(None)
    a_stages = stages(legs["new"])
    a.check(1)
    med_a = {k: float(np.median(v)) for k, v in times.items()}
    log("(a)", med_a)
    del a

    # (b) 16 x 64 MiB in 1 MiB blocks, (c) the same from a CUDA graph
    b = Shape(big, big_pick, 64 * UNIT)
    b.new()
    b.check(64)
    tb = []
    for _ in range(args.steps):
        tb.append(timed(lambda: b.new()))
    b.check(64)
    b_stages = stages(lambda: b.new())
    b.check(64)
    b.scratch = torch.empty(L.swc_xz_block_batch_scratch_bytes(b.n, 1024), dtype=torch.uint8, device=dev)
    b.new(1024)
    b.check(64)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.new(1024)
    torch.cuda.synchronize()
    tc = []
    for _ in range(args.steps):
        tc.append(timed(g.replay))
    b.check(64)
    log("(b)", tb, "(c)", tc)
    old_big = None
    if args.old_big:
        old_big = timed(lambda: b.old())
        b.check(None)

    med_b, med_c = float(np.median(tb)), float(np.median(tc))
    print(json.dumps({
        "gpu": gpu_identity(),
        "blocks": "%d distinct 1 MiB text blocks, LZMA2 preset 6, 1 MiB dictionary, CRC-64, both size fields" % args.distinct,
        "a_config5_1184x1MiB": {
            "median_ms": {k: round(v, 2) for k, v in med_a.items()},
            "all_ms": {k: [round(x, 2) for x in v] for k, v in times.items()},
            "new_vs_old_pct": round(100 * (med_a["new"] / med_a["old"] - 1), 2),
            "old_vs_other_lib_pct": round(100 * (med_a["old"] / med_a["old_other_lib"] - 1), 2) if O is not None else None,
            "new_stage_ms": a_stages,
        },
        "b_16x64MiB_1MiB_blocks": {
            "new_median_ms": round(med_b, 2), "new_all_ms": [round(x, 2) for x in tb],
            "old_once_ms": None if old_big is None else round(old_big, 1),
            "speedup": None if old_big is None else round(old_big / med_b, 1),
            "new_stage_ms": b_stages,
            "output_GBps": round(16 * 64 * UNIT / med_b / 1e6, 2), "input_bytes": b.input_bytes,
        },
        "c_graph_replay_of_b": {"median_ms": round(med_c, 2), "all_ms": [round(x, 2) for x in tc]},
        "stage_order": "walk+place+fill+order | blocks | resolve | fallback",
    }))


if __name__ == "__main__":
    main()
