"""The hand-built LZ4 catalogue (tests/lz4_cases.py) on every LZ4 decode path, against the writer's model and the oracle.

- Raw-block batch (lz4_parse_kernel + lz4_exec_kernel, lz4_fallback_kernel for units whose fields do not fit the 24-bit
  records): one hostile batch per dictionary, at capacities of exactly the decoded size and one byte short, where every
  unit that decodes must report OVERFLOW with its exact size; then every cut of the small blocks as one more batch.
- One-kernel path (lz4_block_kernel): every block of at most 4 MiB, the largest frame block, as the single block of a
  dependent B7 frame with the case's dictionary through LZ4.decompress; the same block as an independent frame and, without
  a dictionary, as a legacy frame (both through the two-phase path).  Larger blocks are raw-only.
- Family 8 (dependent chains, descriptor fields, several frames) through LZ4.decompress and LZ4.multiDecompress.
- A block that decodes to 4 GiB + 16 MiB, through the raw batch and a legacy frame."""

import numpy as np
import pytest

import helpers as H
import lz4_cases as D
import lz4_writer as W
from test_gpu_layout import Layout, _dev, _p, _stream, run_both, run_lz4

pytestmark = pytest.mark.gpu


def _caps(lay, short):
    """every unit's output region: the oracle's output length minus `short` (a failing unit's is empty)"""
    offs = np.zeros(lay.n, dtype=np.uint64)
    caps = np.zeros(lay.n, dtype=np.uint64)
    pos = H.GUARD
    for i, e in enumerate(lay.expect):
        cap = max(len(e[1]) - short, 0)
        offs[i], caps[i] = pos, cap
        pos = (pos + cap + 1 + 15) // 16 * 16
    lay.out_off, lay.out_cap, lay.total = offs, caps, pos + H.GUARD


def _by_dictionary(items, case_of):
    groups = {}
    for it in items:
        groups.setdefault(case_of(it).dict_key, []).append(it)
    return sorted(groups.items(), key=lambda kv: -1 if kv[0] is None else kv[0])


def test_catalogue_raw_batch(oracle):
    blocks = [c for c in D.catalogue() if c.form == "block"]
    groups = _by_dictionary(blocks, lambda c: c)
    assert [k for k, _ in groups] == [None] + list(D.DICT_LENGTHS)
    for j, (key, cs) in enumerate(groups):
        d = cs[0].dictionary
        units = [H.LayoutUnit(c.data, raw=c.out if c.status == W.OK else None) for c in cs]
        lay = Layout("lz4_block", oracle, units, 700 + j, dictionary=d)
        assert [e[0] for e in lay.expect] == [c.status for c in cs]
        _caps(lay, 0)
        lay.check(*run_both(lay, run_lz4, d), consumed=False)
        _caps(lay, 1)
        lay.check(*run_both(lay, run_lz4, d), consumed=False)


def test_truncations_raw_batch(oracle):
    cuts = D.truncations()
    assert len(cuts) > 5000
    for j, (key, ts) in enumerate(_by_dictionary(cuts, lambda t: t.case)):
        d = ts[0].case.dictionary
        units = [H.LayoutUnit(t.data, tail=t.tail) for t in ts]
        lay = Layout("lz4_block", oracle, units, 720 + j, dictionary=d)
        assert [e[0] for e in lay.expect] == [t.model.status for t in ts]
        _caps(lay, 0)
        lay.check(*run_both(lay, run_lz4, d), consumed=False)


def _decompress(data, d):
    import swcompression_b200 as S
    try:
        return W.OK, S.LZ4.decompress(data, d)
    except S.SWCompressionError as e:
        return e.code, e.payload


def _multi(data, d):
    import swcompression_b200 as S
    try:
        return W.OK, S.LZ4.multiDecompress(data, d)
    except S.SWCompressionError as e:
        return e.code, e.payload


def _want(status, out):
    return status, out if status in (W.OK, W.CHECKSUM) else None


def test_catalogue_through_frames():
    """the dependent frame takes lz4_block_kernel; the independent and legacy frames the two-phase path"""
    bad, forms = [], {}
    for c in D.catalogue():
        for form, data, d in D.wrapped(c):
            m = W.decode(data, d)
            forms[form] = forms.get(form, 0) + 1
            got = _decompress(data, d)
            if got != _want(m.status, m.out):
                bad.append((c.name, form, got[0], m.status))
    assert not bad, f"{len(bad)} of {sum(forms.values())} frames differ from the model: {bad[:8]}"
    assert forms["dependent"] > 900 and forms["legacy"] > 700


def test_chains_decompress_and_multi():
    bad, n = [], 0
    for c in D.catalogue():
        if c.form != "frame":
            continue
        n += 1
        got = _decompress(c.data, c.dictionary)
        if got != _want(c.status, c.out):
            bad.append((c.name, "decompress", got[0], c.status))
        got = _multi(c.data, c.dictionary)
        if got != _want(*c.multi):
            bad.append((c.name, "multiDecompress", got[0], c.multi[0]))
    assert not bad, f"{len(bad)} of {n} family 8 cases differ from the model: {bad[:8]}"


# ---------------------------------------------------------------------------------------------------------- past 4 GiB
def _need_memory():
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 10 << 30:
        pytest.skip(f"{free >> 20} MiB free on the device; the block needs about 10 GiB")
    with open("/proc/meminfo") as f:
        avail = next(int(l.split()[1]) << 10 for l in f if l.startswith("MemAvailable:"))
    if avail < 12 << 30:
        pytest.skip(f"{avail >> 20} MiB of host memory available; the block needs about 12 GiB")


RUN = 1 << 24


def test_block_past_4_gib_overflow_size():
    """the block alone at capacity 0 needs no large buffer: it reports OVERFLOW with its exact 64-bit size, 4 GiB + 16 MiB +
    12 bytes, and writes nothing"""
    import torch
    from swcompression_b200 import _lib
    blk, vals, tail = D.past_4gib_block()
    total = len(vals) * RUN + len(tail)
    d_in = _dev(np.frombuffer(b"\xFF" * 5 + blk + b"\xFF" * 64, dtype=np.uint8).copy())
    d_off, d_len = _dev(np.array([5], dtype=np.uint64)), _dev(np.array([len(blk)], dtype=np.uint64))
    d_ooff, d_ocap = _dev(np.array([H.GUARD], dtype=np.uint64)), _dev(np.array([0], dtype=np.uint64))
    d_out = torch.full((2 * H.GUARD,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len = torch.zeros(1, dtype=torch.int64, device="cuda")
    r_st = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    rc = _lib.lib().swc_lz4_block_decompress_batch(_p(d_in), _p(d_off), _p(d_len), None, 0, _p(d_out), _p(d_ooff), _p(d_ocap),
                                                   _p(r_len), _p(r_st), 1, _stream())
    assert rc == 0, _lib.status_name(rc)
    torch.cuda.synchronize()
    assert (r_st.item(), r_len.item()) == (W.OVERFLOW, total)
    assert bool((d_out == H.SENTINEL).all())


def test_block_past_4_gib_raw_batch():
    """one unit at its exact size and the same block at capacity 0: the first decodes to 4 GiB + 16 MiB + 12 bytes (runs
    compared on the device), the second reports OVERFLOW with that size, and no byte outside the regions changes"""
    import torch
    from swcompression_b200 import _lib
    _need_memory()
    blk, vals, tail = D.past_4gib_block()
    nrun = len(vals)
    total = nrun * RUN + len(tail)
    assert total > 1 << 32
    G = H.GUARD
    d_in = _dev(np.frombuffer(b"\xFF" * 13 + blk + b"\xFF" * 64, dtype=np.uint8).copy())
    d_off, d_len = _dev(np.array([13, 13], dtype=np.uint64)), _dev(np.array([len(blk)] * 2, dtype=np.uint64))
    d_ooff = _dev(np.array([G, G + total + G], dtype=np.uint64))
    d_ocap = _dev(np.array([total, 0], dtype=np.uint64))
    d_out = torch.full((total + 3 * G,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    r_len = torch.zeros(2, dtype=torch.int64, device="cuda")
    r_st = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    rc = _lib.lib().swc_lz4_block_decompress_batch(_p(d_in), _p(d_off), _p(d_len), None, 0, _p(d_out), _p(d_ooff), _p(d_ocap),
                                                   _p(r_len), _p(r_st), 2, _stream())
    assert rc == 0, _lib.status_name(rc)
    torch.cuda.synchronize()
    st, ln = r_st.cpu().tolist(), r_len.cpu().tolist()
    assert st == [W.OK, W.OVERFLOW] and ln == [total, total]
    v = torch.tensor(vals, dtype=torch.uint8, device="cuda")
    bad = []
    for k0 in range(0, nrun, 16):
        k1 = min(k0 + 16, nrun)
        got = d_out[G + k0 * RUN:G + k1 * RUN]
        if not torch.equal(got, v[k0:k1].repeat_interleave(RUN)):
            bad += [k for k in range(k0, k1) if not torch.equal(got[(k - k0) * RUN:(k - k0 + 1) * RUN], v[k].expand(RUN))]
    assert not bad, f"runs {bad[:8]} of {nrun} hold wrong bytes"
    assert bytes(d_out[G + nrun * RUN:G + total].cpu().numpy()) == tail
    fence = torch.cat([d_out[:G], d_out[G + total:]])
    assert bool((fence == H.SENTINEL).all()), "bytes changed outside the output region"


def test_block_past_4_gib_legacy_frame():
    """LZ4.decompress of a legacy frame holding the block: the first attempt overflows the 8 MiB guess, the exact-size
    retry decodes it again; every run checked on the host"""
    import swcompression_b200 as S
    _need_memory()
    blk, vals, tail = D.past_4gib_block()
    out = S.LZ4.decompress(W.legacy_frame([blk]))
    nrun = len(vals)
    assert len(out) == nrun * RUN + len(tail)
    a = np.frombuffer(out, dtype=np.uint8)
    bad = [k for k, v in enumerate(vals) if not (a[k * RUN:(k + 1) * RUN] == v).all()]
    assert not bad, f"runs {bad[:8]} of {nrun} hold wrong bytes"
    assert out[nrun * RUN:] == tail
