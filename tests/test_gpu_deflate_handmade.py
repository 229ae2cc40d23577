"""The hand-built Deflate catalogue (tests/deflate_cases.py) on every Deflate decoder, unit by unit against the oracle:
status; for success the bytes, out_len and consumed bits; for overflow the required size.  The units are packed the
hostile way of tests/test_gpu_layout.py (unaligned, between foreign bytes, start bits, fenced outputs) and run twice:
with every output capacity exactly the decoded size and one byte short of it.

- K1w (inflate_warp_kernel): the catalogue is under 20 000 units, so it takes the warp decoder by default;
- K1L (inflate_lut_kernel): the same batch in a child process with SWC_DEFLATE_K1=lut;
- the truncation family (over 20 000 units) in-process, where it takes K1L, and in a child with SWC_DEFLATE_K1=warp;
- the generic kernel (inflate_slow_kernel) through the over-subscribed rewrites (family 7), from both;
- the single-stream API on every case outside family 7 and on a sample of family 7 (the batch tests run all of it)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import deflate_cases as D
import helpers as H
from test_gpu_layout import Layout, run_both, run_deflate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _caps(lay, short):
    """output regions of exactly the oracle's size minus `short` bytes (a failing unit gets room to spare), on 16-byte
    multiples with GUARD bytes around them"""
    sizes = [len(e[1]) if e[0] == 0 else None for e in lay.expect]
    spare = max([s for s in sizes if s is not None] + [0]) + 1024
    offs = np.zeros(lay.n, dtype=np.uint64)
    caps = np.zeros(lay.n, dtype=np.uint64)
    pos = H.GUARD
    for i, s in enumerate(sizes):
        cap = spare if s is None else max(s - short, 0)
        offs[i], caps[i] = pos, cap
        pos = (pos + cap + 1 + 15) // 16 * 16
    lay.out_off, lay.out_cap, lay.total = offs, caps, pos + H.GUARD


def catalogue_batches(oracle):
    cases = D.catalogue()
    units = [H.LayoutUnit(c.data, aux=c.start_bit, raw=c.expect) for c in cases]
    lay = Layout("deflate", oracle, units, 301)
    wrong = [(c.name, e[0]) for c, e in zip(cases, lay.expect) if e[0] != c.status or (e[0] == 0 and e[2] != c.nbits)]
    assert not wrong, f"the oracle disagrees with the catalogue: {wrong[:8]}"
    for short in (0, 1):
        _caps(lay, short)
        lay.check(*run_both(lay, run_deflate, start_bits=[u.aux for u in units]))


def truncation_batch(oracle):
    trunc = D.truncation_units()
    units = [H.LayoutUnit(t.data, tail=t.tail, aux=t.start_bit) for t in trunc]       # the rest of the stream behind each
    lay = Layout("deflate", oracle, units, 302)
    assert lay.n >= 20000 and all(e[0] != 0 for e in lay.expect)
    lay.check(*run_both(lay, run_deflate, start_bits=[u.aux for u in units]))


def _child(kernel, fn):
    env = dict(os.environ, SWC_DEFLATE_K1=kernel)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    code = f"import swco, test_gpu_deflate_handmade as T; T.{fn}(swco)"
    p = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]


def test_catalogue_warp_kernel(oracle):
    catalogue_batches(oracle)


def test_catalogue_lut_kernel():
    _child("lut", "catalogue_batches")


def test_truncations_lut_kernel(oracle):
    truncation_batch(oracle)


def test_truncations_warp_kernel():
    _child("warp", "truncation_batch")


def test_single_stream_api(oracle):
    """Deflate.decompress_from on every case of the catalogue outside family 7 and on every tenth over-subscribed rewrite
    (the serial generic kernel takes them one call at a time), Deflate.decompress on those without start bits, and a
    sample of the truncations"""
    import swcompression_b200 as S
    bad = []
    over = [c for c in D.catalogue() if c.family == 7]
    for c in [c for c in D.catalogue() if c.family != 7] + over[::10]:
        try:
            out, used = S.Deflate.decompress_from(c.data, c.start_bit)
            got = (0, out, used)
        except S.SWCompressionError as e:
            got = (e.code, None, None)
        if got != ((0, c.expect, c.nbits) if c.expect is not None else (c.status, None, None)):
            bad.append((c.name, got[0], c.status, got[2], c.nbits))
        elif c.start_bit == 0 and c.expect is not None and c.family != 7 and S.Deflate.decompress(c.data) != c.expect:
            bad.append((c.name, "decompress"))
    assert not bad, f"{len(bad)} cases differ: {bad[:8]}"
    rng = random.Random(303)
    for t in rng.sample(D.truncation_units(), 100):
        with pytest.raises(S.SWCompressionError) as e:
            S.Deflate.decompress_from(t.data, t.start_bit)
        assert e.value.code == oracle.deflate_decompress(t.data, t.start_bit)[0], t.name
