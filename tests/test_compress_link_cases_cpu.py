"""The link-builder and emit-chunk catalogue (compress_link_cases.py) on the CPU: every case reaches the edges it names in
the model of the GPU machinery, the model and the CPU restatement of the reference agree with the plain statements on
every case, and each near miss of the model gets at least the case aimed at it wrong."""
import functools

import pytest

import compress_link_cases as K
import lz4c_cases as LK
from test_deflate_compress_cpu import statement

DCASES = K.deflate_cases()
LCASES = K.lz4_cases()
DBY = {c[0]: c for c in DCASES}
LBY = {c[0]: c for c in LCASES}


@functools.lru_cache(maxsize=None)
def dmodel(name, variant=None):
    return K.DeflateModel(DBY[name][1], variant)


@functools.lru_cache(maxsize=None)
def lmodel(name, variant=None):
    _, block, dictionary, _ = LBY[name]
    return K.LZ4Model(block, dictionary, variant)


@pytest.mark.parametrize("name", list(DBY))
def test_deflate_case_reaches_its_edges(name):
    m = dmodel(name)
    missed = [e for e in DBY[name][2] if not K.deflate_edge(m, e)]
    assert not missed, missed


@pytest.mark.parametrize("name", list(DBY))
def test_deflate_model_statement_and_oracle_agree(name):
    import swco_deflatec
    data = DBY[name][1]
    ref = statement(data)
    assert dmodel(name).out == ref
    assert swco_deflatec.deflate_compress(data) == (0, ref, None)


def test_deflate_catalogue_covers_the_geometry():
    names = set(DBY)
    assert {f"halo_x{x}_d{d}" for x in (0, 1, 31, 32, 33) for d in (K.REACH, K.REACH + 1)} <= names
    assert {f"phase_{v}" for v in range(32)} <= names
    assert {f"out_len_mod4_{r}" for r in range(4)} | {"bits_mod32_0"} <= names
    groups = [len(e[1]) for _, _, edges in DCASES for e in edges if e[0] == "group"]
    assert set(range(2, 9)) <= set(groups)
    assert {e[0] for _, _, edges in DCASES for e in edges} >= {
        "halo", "hidden", "nearest_bucket", "chain_past_reach", "chunk_at_match", "chunk_in_match",
        "chunk_in_literals", "eob_only", "end_match"}
    assert {e[1] for _, _, edges in DCASES for e in edges if e[0] == "end_match"} == {0, 1, 2}


# each near miss and the case built to catch it
DEFLATE_AIMED = {"halo_short": "halo_x0_d32768", "bucket": "bucket_reach", "late_checkpoint": "chunk_boundaries"}


@pytest.mark.parametrize("variant", K.DEFLATE_VARIANTS)
def test_deflate_near_miss_is_caught(variant):
    name = DEFLATE_AIMED[variant]
    assert dmodel(name, variant).out != dmodel(name).out


def test_deflate_halo_short_misses_only_lane_zero():
    """the halo one position short loses exactly the source at the window's first position"""
    for x in (0, 1, 31, 32, 33):
        name = f"halo_x{x}_d{K.REACH}"
        assert (dmodel(name, "halo_short").out != dmodel(name).out) == (x == 0), name


@pytest.mark.parametrize("name", list(LBY))
def test_lz4_case_reaches_its_edges(name):
    m = lmodel(name)
    missed = [e for e in LBY[name][3] if not K.lz4_edge(m, e)]
    assert not missed, missed


@pytest.mark.parametrize("name", list(LBY))
def test_lz4_model_statement_and_oracle_agree(name):
    import swco_lz4c
    _, block, dictionary, _ = LBY[name]
    ref = LK.py_block(block, dictionary)
    assert lmodel(name).out == ref
    assert swco_lz4c.lz4_block_compress(block, dictionary) == (0, ref, None)


def test_lz4_catalogue_covers_the_geometry():
    assert {K.lz4_edge(lmodel(n), ("align", s)) for n, s in ((f"seam_align_{s}", s) for s in range(1, 32))} == {True}
    assert {len(LBY[f"seam_dict_{d}"][2]) for d in (K.MAX_DICT - 1, K.MAX_DICT, K.MAX_DICT + 1)} == {
        K.MAX_DICT - 1, K.MAX_DICT, K.MAX_DICT + 1}
    steps = [e[1:] for _, _, _, edges in LCASES for e in edges if e[0] == "steps"]
    assert any(lp == 31 and apart == 0 for _, lp, _, _, apart in steps)
    assert any(lp == 0 and apart == 1 for _, lp, _, _, apart in steps)
    assert any(lq == 0 and apart == 0 for _, _, _, lq, apart in steps)
    assert any(lq == 31 and apart >= 1 for _, _, _, lq, apart in steps)
    groups = [len(e[1]) for _, _, _, edges in LCASES for e in edges if e[0] == "group"]
    assert set(range(2, 9)) <= set(groups)


LZ4_AIMED = {"write_first": "between_in_step", "front_to_back": "between_across_steps", "bucket": "bucket_groups"}


@pytest.mark.parametrize("variant", K.LZ4_VARIANTS)
def test_lz4_near_miss_is_caught(variant):
    name = LZ4_AIMED[variant]
    assert lmodel(name, variant).out != lmodel(name).out

