#!/usr/bin/env python3
"""What walking TAR archives on the device costs: WebDataset-shaped shards (64 MiB, entries of 1-64 KiB) as plain tar
through a 'tar' batch (swc_tar_walk_batch), and the same shards as .tar.gz through a 'gzip' batch followed by a 'tar'
batch over its outputs, alternated in one process against the 'gzip' batch alone.  CUDA events around whole calls;
every unit's statuses and entry count are checked against the CPU restatement (oracle/tar.c), whose walk is also timed
on the CPU threads
(the C walk alone: buffers and record tables are prepared before the clock starts).

    python tools/bench_tar_batch.py [--shards 16] [--steps 5] [--warmup 1] [--level 6]

Prints one JSON line with the GPU's name and power limit, headers per second of the walk, the walk's share of the
.tar.gz path, and the CPU walk's headers per second."""
import argparse
import gzip
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SHARD = 64 << 20


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def shard(seed):
    """one WebDataset-style shard: samples of a .txt and a .bin member, 1-64 KiB each, up to 64 MiB"""
    import tar_writer as W
    rng = np.random.default_rng(seed)
    parts, size, k = [], 0, 0
    words = [b"alpha", b"beta", b"gamma", b"delta", b"tar", b"shard", b"sample"]
    while True:
        for ext in (b"txt", b"bin"):
            n = int(rng.integers(1024, 65537))
            if size + 512 + n + 511 + 1024 > SHARD:
                return b"".join(parts) + W.EOF_MARKER
            body = (b" ".join(words[int(i)] for i in rng.integers(0, len(words), n // 4 + 1)))[:n] if ext == b"txt" else \
                rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            e = W.entry(body, name=b"%08d.%s" % (k, ext), magic=W.USTAR)
            parts.append(e)
            size += len(e)
        k += 1


def timed(fn, torch):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--level", type=int, default=6)
    a = ap.parse_args()
    import torch
    import swco_tar
    from swcompression_b200.batch import Batch

    with ThreadPoolExecutor() as ex:
        shards = list(ex.map(shard, range(a.shards)))
        gz = list(ex.map(lambda s: gzip.compress(s, a.level, mtime=0), shards))
    want = [swco_tar.walk(s)[:3] for s in shards]
    headers = sum(w[0] for w in want)

    plain = Batch.from_units("tar", shards, None)
    g = Batch.from_units("gzip", gz, SHARD)
    t = Batch.tar_of(g)
    for _ in range(a.warmup):
        plain.run(); g.run(); t.run()
    torch.cuda.synchronize()
    tp, tg, tgt = [], [], []
    for _ in range(a.steps):
        tp.append(timed(plain.run, torch))
        tg.append(timed(g.run, torch))
        tgt.append(timed(lambda: (g.run(), t.run()), torch))
    for b in (plain, t):
        n, ist, ost, _, _ = b.tar_results()
        assert [(int(x), int(y), int(z)) for x, y, z in zip(n, ist, ost)] == want, "walk differs from the oracle"
    st, ln, _ = g.results()
    assert (st == 0).all() and [int(x) for x in ln] == [len(s) for s in shards]

    cpu_s = swco_tar.walk_seconds(shards, os.cpu_count())

    med = lambda v: float(np.median(v))
    walk_ms, gz_ms, chain_ms = med(tp), med(tg), med(tgt)
    print(json.dumps({
        "gpu": gpu_identity(), "shards": a.shards, "shard_bytes": SHARD, "headers": headers, "gzip_level": a.level,
        "tar_walk_ms": walk_ms, "tar_headers_per_s": headers / walk_ms * 1e3,
        "gzip_ms": gz_ms, "gzip_then_tar_ms": chain_ms, "walk_share_of_tar_gz": (chain_ms - gz_ms) / chain_ms,
        "cpu_oracle_walk_s": cpu_s, "cpu_threads": os.cpu_count(), "cpu_headers_per_s": headers / cpu_s,
        "samples_ms": {"tar": tp, "gzip": tg, "gzip_then_tar": tgt}}))


if __name__ == "__main__":
    main()
