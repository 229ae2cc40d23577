#!/usr/bin/env python3
"""Secondary benchmarks for BASELINE.json configs 3-5 (LZ4 blocks, BZip2 900 KB blocks, XZ/LZMA2 1 MiB streams) on ONE GPU.

bench.py stays the headline (config 2, Deflate).  Each workload prints one JSON line with the same keys: decompressed GB/s
with the batch resident in HBM, the HBM roofline fraction of the (single) kernel, and the CPU restatement's throughput.
Unit counts are scaled to one GPU / a few minutes (stated in `config`); distinct units are tiled on the device.
`--workload lz4c` is the compress direction (LZ4.compress, LZ4+Compress.swift): it reports INPUT GB/s and prints a second
line for single LZ4.compress(data:) calls of 256 MiB.
"""
import argparse
import ctypes as C
import bz2
import json
import lzma
import os
import sys
import time
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _lz4_unit(seed):
    import helpers as H
    rng = np.random.Generator(np.random.PCG64(seed))
    k = rng.random()
    raw = bytes(65536) if k < 0.1 else rng.integers(0, 256, 65536, dtype=np.uint8).tobytes() if k < 0.2 else H.textlike(65536, seed)
    return H.lz4_block_compress(raw), raw


def _bz2_unit(seed):
    import helpers as H
    raw = H.textlike(900000, seed)
    return bz2.compress(raw, 9), raw


def _xz_unit(seed):
    import helpers as H
    raw = H.textlike(1 << 20, seed)
    # the unit handed to the batched kernel is the raw LZMA2 stream of the block (XZ framing is parsed on the host)
    return lzma.compress(raw, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "preset": 6, "dict_size": 1 << 20}]), raw


WORKLOADS = {
    "lz4": dict(gen=_lz4_unit, seed0=3, codec="lz4_block", unit=65536, distinct=2048, units=262144, kernel="lz4_parse_kernel + lz4_exec_kernel",
                desc="LZ4 block mode: independent 64 KiB blocks (80 % text-like, 10 % zeros, 10 % incompressible), LZ4_compress_default"),
    "bzip2": dict(gen=_bz2_unit, seed0=4, codec="bzip2", unit=900000, distinct=64, units=2048, kernel="bzip2_kernel",
                  desc="BZip2: independent single-block 900 KB streams, bz2 level 9"),
    "xz": dict(gen=_xz_unit, seed0=5, codec="lzma2", unit=1 << 20, distinct=32, units=1184, kernel="lzma_kernel",
               desc="XZ/LZMA2: independent 1 MiB streams, preset 6, 1 MiB dictionary (raw LZMA2 payload of each XZ block)"),
}


def oracle_fn(name):
    import swco
    if name == "lz4":
        return lambda u: swco.lz4_block(u)
    if name == "bzip2":
        return lambda u: swco.bzip2_decompress(u)
    return lambda u: swco.lzma2_decompress_raw(u, 18)


def cpu_throughput(name, units, budget, threads):
    """pthreads inside oracle/batch_mt.c (no interpreter in the timed loop)"""
    import swco
    codec, aux = {"lz4": ("lz4_block", 0), "bzip2": ("bzip2", 0), "xz": ("lzma2", 18)}[name]
    sec, nbytes, fails = swco.batch_mt(codec, units, max(threads, 4), threads, aux)
    assert fails == 0
    total = max(int(budget / (sec / max(threads, 4))), threads)
    sec, nbytes, fails = swco.batch_mt(codec, units, total, threads, aux)
    assert fails == 0
    return nbytes / sec / 1e9, total, sec


def best_threads(name, units):
    ncpu = os.cpu_count() or 1
    sweep = {th: cpu_throughput(name, units, 1.0, th)[0] for th in sorted({max(1, ncpu >> k) for k in range(5)} | {min(ncpu, 16), min(ncpu, 24)})}
    return max(sweep, key=sweep.get), {str(k): round(v, 3) for k, v in sweep.items()}


def _raw64k(seed):
    return _lz4_unit(seed)[1]


def run_lz4c(args):
    """LZ4 compression: independent 64 KiB blocks of the lz4 mix, no dictionary, through swc_lz4_block_compress_batch"""
    import torch
    import swco_lz4c
    from swcompression_b200 import LZ4, _lib
    from swcompression_b200.batch import Batch
    n_units = args.units or 262144
    distinct = min(2048, n_units)
    tile = max(n_units // distinct, 1)
    n_units = tile * distinct
    with Pool(min(os.cpu_count() or 1, 32)) as pool:
        raws = pool.map(_raw64k, range(3, 3 + distinct), chunksize=1)
    dev = torch.device("cuda:0")
    L = _lib.lib()
    one = torch.from_numpy(np.frombuffer(b"".join(raws), dtype=np.uint8).copy()).to(dev)
    d_in = torch.cat([one.repeat(tile), torch.zeros(64, dtype=torch.uint8, device=dev)])
    del one
    offs = np.arange(n_units, dtype=np.uint64) * np.uint64(65536)
    cap = 65536 + 65536 // 255 + 64
    b = Batch("lz4_block_compress", np.zeros(1, dtype=np.uint8), offs, np.full(n_units, 65536, dtype=np.uint64), cap, device=str(dev))
    b.d_in = d_in
    for _ in range(args.warmup):
        b.run()
    st, ln, _ = b.results()
    assert (st == 0).all()
    pc = (cap + 15) // 16 * 16
    host = b.d_out[: min(distinct, 8) * pc].cpu().numpy()
    for i in range(min(distinct, 8)):
        assert bytes(host[i * pc:i * pc + int(ln[i])]) == swco_lz4c.lz4_block_compress(raws[i])[1], "parity vs oracle failed"
    total_in, total_out = n_units * 65536, int(ln.sum())
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    L.swc_timing_enable(1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.steps):
        b.run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    tbuf = (C.c_float * 4096)()
    nint = L.swc_timing_collect(tbuf, 4096)
    L.swc_timing_enable(0)
    # every slice of a batch drops marks before lz4c_chain_kernel and after each of the three kernels: the intervals run
    # chain, parse, emit, then the host's planning of the next slice
    per = [sum(float(tbuf[i]) for i in range(k, nint, 4)) / args.steps for k in range(4)]
    peak = 3350.0
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    achieved = (total_in + total_out) / (ms * 1e-3) / 1e9
    cpu = None
    if not args.no_cpu:
        threads = os.cpu_count() or 1
        sec, _, fails = swco_lz4c.batch_mt(raws, max(threads * 4, 64), threads)
        total = max(int(8.0 / (sec / max(threads * 4, 64))), threads)
        sec, _, fails = swco_lz4c.batch_mt(raws, total, threads)
        assert fails == 0
        cpu = {"value": total * 65536 / sec / 1e9, "unit": "GB/s (input)", "cores": threads, "kind": "port",
               "sample": f"{total} units in {sec:.1f} s on {threads} pthreads (oracle/lz4_compress.c)"}
    del b, d_in
    torch.cuda.empty_cache()
    print(json.dumps({
        "metric": "compressed_input_GB_per_s", "value": total_in / (ms * 1e-3) / 1e9, "unit": "GB/s", "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "data": "synthetic",
        "config": {"workload": "LZ4 compression, LZ4+Compress.swift parse: independent 64 KiB blocks (80 % text-like, 10 % zeros, "
                               "10 % incompressible), no dictionary", "units": n_units, "distinct_units": distinct,
                   "input_bytes": total_in, "compressed_bytes": total_out},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "kernel": "lz4c_chain_kernel + lz4c_parse_kernel + lz4c_emit_kernel", "kernel_ms": ms,
                     "kernel_ms_chain_parse_emit": [round(x, 3) for x in per[:3]], "between_slices_ms": round(per[3], 3)},
        "cpu_baseline": cpu}))
    # one LZ4.compress(data:) call of 256 MiB: few blocks means few parse lanes
    data = b"".join(raws[i % distinct] for i in range(4096))
    single = {}
    for label, kw in (("default_4MiB_blocks", {}), ("dependent_64KiB_blocks", dict(independentBlocks=False, blockSize=65536))):
        out = LZ4.compress(data, **kw)
        assert out == swco_lz4c.lz4_compress(data, **kw)[1], "parity vs oracle failed"
        t0 = time.perf_counter()
        for _ in range(max(args.steps // 2, 1)):
            out = LZ4.compress(data, **kw)
        dt = (time.perf_counter() - t0) / max(args.steps // 2, 1)
        single[label] = {"seconds": round(dt, 3), "input_GB_per_s": len(data) / dt / 1e9, "compressed_bytes": len(out)}
    print(json.dumps({"metric": "single_call_input_GB_per_s", "unit": "GB/s", "input_bytes": len(data),
                      "host_buffers": True, "calls": single}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=list(WORKLOADS) + ["lz4c"], required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--units", type=int, default=0)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if args.workload == "lz4c":
        return run_lz4c(args)
    W = WORKLOADS[args.workload]
    n_units = args.units or W["units"]
    distinct = min(W["distinct"], n_units)
    tile = max(n_units // distinct, 1)
    n_units = tile * distinct
    with Pool(min(os.cpu_count() or 1, 32)) as pool:
        pairs = pool.map(W["gen"], range(W["seed0"], W["seed0"] + distinct), chunksize=1)
    units = [p[0] for p in pairs]
    raws = [p[1] for p in pairs]

    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import Batch, pack_units
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    L = _lib.lib()
    buf, offs, lens = pack_units(units)
    stride = len(buf) - 64
    d_in = torch.cat([torch.from_numpy(buf[:stride]).to(dev).repeat(tile), torch.zeros(64, dtype=torch.uint8, device=dev)])
    all_off = (offs[None, :] + (np.arange(tile, dtype=np.uint64) * np.uint64(stride))[:, None]).reshape(-1)
    all_len = np.tile(lens, tile)
    aux = bytes([18] * n_units) if W["codec"] == "lzma2" else None
    b = Batch(W["codec"], np.zeros(1, dtype=np.uint8), all_off, all_len, W["unit"], device=str(dev), aux=aux)
    b.d_in = d_in
    total_in = int(lens.sum()) * tile
    total_out = n_units * W["unit"]
    for _ in range(args.warmup):
        b.run()
    st, ln, used = b.results()
    assert (st == 0).all() and (ln == W["unit"]).all(), (st[:8], ln[:8])
    fn = oracle_fn(args.workload)
    host = b.d_out[: min(distinct, 8) * ((W["unit"] + 15) // 16 * 16)].cpu().numpy()
    pu = (W["unit"] + 15) // 16 * 16
    for i in range(min(distinct, 8)):
        ost, oout, _ = fn(units[i])
        assert ost == 0 and oout == raws[i] and bytes(host[i * pu:i * pu + W["unit"]]) == oout, "parity vs oracle failed"
    launches0 = L.swc_kernel_launches()
    L.swc_timing_collect.argtypes = [C.c_void_p, C.c_int32]
    L.swc_timing_enable(1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.steps):
        b.run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    tbuf = (C.c_float * 64)()
    nint = L.swc_timing_collect(tbuf, 64)
    L.swc_timing_enable(0)
    marks = [round(float(x), 3) for x in list(tbuf)[:nint]]
    launches = L.swc_kernel_launches() - launches0
    peak = 3350.0                      # H100 SXM data sheet, HBM3
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    achieved = (total_in + total_out) / (ms * 1e-3) / 1e9
    cpu = None
    if not args.no_cpu:
        cores, sweep = best_threads(args.workload, units)
        v1, n1, d1 = cpu_throughput(args.workload, units, 4.0, 1)
        vN, nN, dN = cpu_throughput(args.workload, units, 8.0, cores)
        cpu = {"value": vN, "unit": "GB/s", "cores": cores, "logical_cpus": os.cpu_count(), "thread_sweep_GBps": sweep, "kind": "port",
               "single_thread_value": v1, "sample": f"{nN} units in {dN:.1f} s on {cores} pthreads (oracle/batch_mt.c)"}
    print(json.dumps({
        "metric": "decompressed_GB_per_s", "value": total_out / (ms * 1e-3) / 1e9, "unit": "GB/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8",
        "data": "synthetic",
        "config": {"workload": W["desc"], "units": n_units, "unit_bytes": W["unit"], "distinct_units": distinct,
                   "compressed_bytes": total_in, "decompressed_bytes": total_out},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                     "kernel": W["kernel"], "kernel_ms": ms, "algorithmic_bytes_per_launch": total_in + total_out,
                     "intervals_between_timing_marks_ms": marks},
        "cpu_baseline": cpu, "gpu_launches": int(launches)}))


if __name__ == "__main__":
    main()
