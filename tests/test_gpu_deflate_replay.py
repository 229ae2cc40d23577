"""Hand-built Deflate streams aimed at the batch boundaries of lz_resolve_kernel (K2, csrc/inflate.cu), decoded through
both Huffman stages (K1w by default, K1L in a child process with SWC_DEFLATE_K1=lut) at all 16 output phases and compared
with the oracle byte for byte.

A K2 batch is the longest run of at most 64 records whose output ends within SPAN = 1 KiB of the batch start; a literal
run longer than that is placed in pieces of SPAN bytes.  A match is read from the flushed output ("far") when its first
source byte lies more than RING = 2 KiB behind the batch end, and from the shared-memory ring otherwise.  `batches`
restates that rule so that the streams below can put records exactly on its edges; the CPU test checks that they do."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import deflate_writer as W
import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RING, SPAN, BATCH = 2048, 1024, 64
DELTAS = (-16, -1, 0, 1, 16)


def records(tokens):
    """tokens [(literal run, length, distance)] -> the Huffman stage's records [(advance, length, distance)]: a run over
    255 bytes is first cut down by an escape record (length 0) that advances by run & ~255"""
    recs = []
    for run, ln, d in tokens:
        if run > 255:
            recs.append((run & ~255, 0, 0))
            run &= 255
        recs.append((run + ln, ln, d))
    return recs


def batches(recs, total):
    """K2's batches -> [(first record, records, start, end)]; 0 records for a piece of a long literal run"""
    out, g, done, part = [], 0, 0, 0
    while True:
        cum = k = 0
        while k < BATCH and g + k < len(recs):
            a = recs[g + k][0] - (part if k == 0 else 0)
            if cum + a > SPAN:
                break
            cum, k = cum + a, k + 1
        if k:
            out.append((g, k, done, done + cum))
            g, part, done = g + k, 0, done + cum
            continue
        rem = recs[g][0] - part if g < len(recs) else total - done
        if rem == 0:
            return out
        s = min(rem, SPAN)
        if g < len(recs):
            part += s
        out.append((g, 0, done, done + s))
        done += s


def positions(recs):
    """output position at which each record's match starts"""
    pos, p = [], 0
    for adv, ln, _ in recs:
        p += adv
        pos.append(p - ln)
    return pos


class Stream:
    """A unit built from tokens; distances may be filled in after the batches are known (they do not move them)."""

    def __init__(self, name, tokens, tail):
        self.name, self.tokens, self.tail = name, [list(t) for t in tokens], tail

    def layout(self):
        recs = records(self.tokens)
        total = sum(r + ln for r, ln, _ in self.tokens) + self.tail
        return recs, batches(recs, total), total

    def token_of_record(self):
        out = []
        for i, (run, _, _) in enumerate(self.tokens):
            if run > 255:
                out.append(None)
            out.append(i)
        return out

    def encode(self, seed):
        rng = random.Random(seed)
        w = W.DeflateWriter()
        toks = []
        for run, ln, d in self.tokens:
            if run:
                toks.append(bytes(rng.randrange(97, 123) for _ in range(run)))
            toks.append(W.Match(ln, d))
        if self.tail:
            toks.append(bytes(rng.randrange(97, 123) for _ in range(self.tail)))
        w.dynamic(toks, final=True)
        data, _ = w.finish()
        return data, bytes(w.out)


def _group(n, total, near_at, far=False, periodic=()):
    """n tokens whose outputs sum to `total`; distances near (<= 40, from `near_at` on) or far (> RING + SPAN); the tokens
    at the indices in `periodic` copy 40 bytes at distance 3 (dist < len)"""
    out = []
    for i in range(n):
        a = total // n + (1 if i < total % n else 0)
        ln = 40 if i in periodic else 3 + i % 6
        d = 3 if i in periodic else (RING + SPAN + 64 + 17 * i if far else min(near_at + a - ln, 5 + (13 * i) % 36))
        out.append((a - ln, ln, d))
        near_at += a
    return out


def _prefix():
    """a 4 KiB + 40 B literal run, then records that close the batch after its pieces exactly at SPAN: the batches after
    it start with the next token and can reach 3 KiB back"""
    return [(4096 + 40, 3, 7), (255, 258, 1), (210, 258, 1)]


def cases():
    """-> [Stream]"""
    out = []
    cross = (255, 258, 1)                     # 513 bytes: no group below closes a batch with it
    for n in (31, 32, 33, 62, 63, 64, 65):
        for total in (SPAN, SPAN - 7):
            if total // n < 15:
                continue
            out.append(Stream(f"first_batch_{n}_{total}", [(40, 3, 7)] + _group(n - 1, total - 43, 43) + [cross]
                              + _group(20, 400, 2000), 33))
            out.append(Stream(f"far_batch_{n}_{total}", _prefix() + _group(n, total, 5120, far=True) + [cross]
                              + _group(20, 400, 6000, far=True), 5))
    # distances at the far/near threshold of a 64-record batch, measured from its end and from its start
    for end_side in (True, False):
        for tail_escape in (False, True):
            s = Stream(f"threshold_{'end' if end_side else 'start'}{'_escape_after' if tail_escape else ''}",
                       _prefix() + _group(64, SPAN, 5120, far=True) + ([(1500, 3, 1)] if tail_escape else [cross])
                       + _group(20, 400, 6000, far=True), 0)
            recs, bs, _ = s.layout()
            pos, tok = positions(recs), s.token_of_record()
            big = next(b for b in bs if b[1] == 64)
            for j, r in enumerate(range(big[0], big[0] + big[1])):
                if tok[r] is None or recs[r][1] == 0:
                    continue
                ref = big[3] if end_side else big[2]
                s.tokens[tok[r]][2] = pos[r] + RING - ref + DELTAS[j % len(DELTAS)]
            out.append(s)
    # dist < len at both ends of 64-record batches
    out.append(Stream("periodic_at_batch_ends", _prefix() + _group(64, SPAN, 5120, periodic=(0, 63))
                      + _group(64, SPAN, 6144, periodic=(0, 63)) + [(0, 258, 1), (0, 258, 2)], 21))
    out.append(Stream("periodic_first_batch", [(40, 3, 7)] + _group(63, SPAN - 43, 43, periodic=(1, 62))
                      + [(0, 258, 3)] * 4, 9))
    # literal runs longer than SPAN directly before and after a 64-record batch, and trailing literal runs
    # (an escape's last piece of at most SPAN bytes is a record of the batch after it: here 256 bytes, which with the
    # match behind it and 62 more records fill a 64-record batch)
    for run in (1300, 2350):
        rest = SPAN - 256 - (run & 255) - 3
        out.append(Stream(f"escapes_around_64_{run}", _prefix() + [(run, 3, 9)] + _group(62, rest, 5120 + run)
                          + [(run, 5, 2900)] + _group(64, SPAN, 9000, far=True), run))
    # near matches (read from the ring) across the ring's end: at output position k * RING (k = 1..8) one match whose
    # destination and one whose source cross it, starting k - 1 bytes later each time, so that at every output phase
    # some 8-byte copy trip is cut after each of its first 7 bytes
    toks, at = [], 0
    for k in range(1, 9):
        for ms, d in ((k * RING - 24 + k - 1, 40), (k * RING + 8 + k - 1, 32)):
            toks.append((ms - at, 24, d))
            at = ms + 24
    out.append(Stream("ring_wrap_near", toks, 3))
    for tail in (0, 1, 15, 16, 17, SPAN - 1, SPAN, SPAN + 1, 3000):
        out.append(Stream(f"trailing_literals_{tail}", [(40, 3, 7)] + _group(64, SPAN, 43), tail))
    return out


def _cpu_view():
    """per case: (records, batches, match positions)"""
    return [(s,) + s.layout()[:2] + (positions(s.layout()[0]),) for s in cases()]


def test_cases_reach_the_batch_edges():
    """CPU: the model's batches of the streams cover every edge the GPU tests are meant to reach"""
    sizes, capped, crossed, far_near, periodic, escapes, tails = set(), False, set(), set(), set(), set(), set()
    for s, recs, bs, pos in _cpu_view():
        for bi, (g, k, b0, b1) in enumerate(bs):
            sizes.add(k)
            if k == BATCH and g + k < len(recs) and b1 - b0 + recs[g + k][0] <= SPAN:
                capped = True                                   # a 65th record would still have fitted
            if k and g + k < len(recs) and k in (63, 64) and b1 - b0 + recs[g + k][0] > SPAN:
                crossed.add(k)                                  # the record after the 63rd / 64th crosses SPAN
            if k == BATCH:
                if bi > 0 and bs[bi - 1][1] == 0:
                    escapes.add("before")
                if bi + 1 < len(bs) and bs[bi + 1][1] == 0:
                    escapes.add("after")
            for r in range(g, g + k):
                adv, ln, d = recs[r]
                if ln == 0:
                    continue
                assert 1 <= d <= pos[r] and d <= 32768, (s.name, r)
                far_near.add((pos[r] - d + RING - b1, "end"))
                far_near.add((pos[r] - d + RING - b0, "start"))
                if d < ln and r in (g, g + k - 1):
                    periodic.add("first" if r == g else "last")
        tails.add(s.tail)
    assert {31, 32, 33, 62, 63, 64, 0} <= sizes
    assert capped and crossed == {63, 64}
    assert {(-d, side) for d in DELTAS for side in ("end", "start")} <= far_near
    assert periodic == {"first", "last"} and escapes == {"before", "after"}
    assert {0, 1, 15, 16, 17, SPAN, SPAN + 1} <= tails


def test_near_copies_cross_the_ring_end():
    """CPU: at every output phase, near matches copied 8 bytes per lane and trip (2-lane sub-groups: trips start at bytes
    0, 8, 16, ... of the match) have trips whose destination and trips whose source cross the ring's end after each
    of their first 7 bytes"""
    s = next(c for c in cases() if c.name == "ring_wrap_near")
    recs, bs, _ = s.layout()
    pos = positions(recs)
    for ph in range(16):
        dst, src = set(), set()
        for r, (adv, ln, d) in enumerate(recs):
            if ln == 0 or d < ln:
                continue
            for i in range(0, ln, 8):
                n = min(8, ln - i)
                for cut in range(1, n):
                    if (pos[r] + i + ph + cut) % RING == 0:
                        dst.add(cut)
                    if (pos[r] - d + i + ph + cut) % RING == 0:
                        src.add(cut)
        assert dst == src == set(range(1, 8)), (ph, dst, src)


def _run(oracle):
    """every case at output phases 0..15 as one batch, checked against the oracle"""
    from test_gpu_layout import Layout, run_deflate
    units = []
    for i, s in enumerate(cases()):
        data, raw = s.encode(1000 + i)
        units += [H.LayoutUnit(data, raw=raw)] * 16
    lay = Layout("deflate", oracle, units, 401)
    offs = np.zeros(lay.n, dtype=np.uint64)
    caps = np.zeros(lay.n, dtype=np.uint64)
    pos = H.GUARD
    for i, (st, raw, _) in enumerate(lay.expect):
        assert st == 0, (i, st)
        pos = (pos + 15) // 16 * 16 + i % 16                   # output phase i mod 16
        offs[i], caps[i] = pos, len(raw)
        pos += len(raw) + 1
    lay.out_off, lay.out_cap, lay.total = offs, caps, pos + H.GUARD
    lay.check(*run_deflate(lay))


@pytest.mark.gpu
def test_replay_edges_warp_kernel(oracle):
    _run(oracle)


@pytest.mark.gpu
def test_replay_edges_lut_kernel():
    env = dict(os.environ, SWC_DEFLATE_K1="lut")
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")] +
                                        ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    code = "import swco, test_gpu_deflate_replay as T; T._run(swco)"
    p = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
