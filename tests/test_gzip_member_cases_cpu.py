"""Pins the multi-member gzip cases (tests/gzip_member_cases.py) on the CPU: every stated status and member list is the
oracle's (swco_gzip_multi_unarchive), the member starts the oracle's walk gives are the ones Python's zlib finds in every
valid file, every BGZF case is a chain of BSIZE hints except those built to lie, and the byte cuts cover each status the
batch must reproduce."""
import gzip_member_cases as G


def test_statuses_and_members_match_oracle(oracle):
    bad = []
    for c in G.cases():
        st, out, ends, starts, consumed = G.expect(oracle, c.data)
        if c.status is not None and st != c.status:
            bad.append((c.name, st, c.status))
        elif c.members is not None and (out != b"".join(c.members) or len(ends) != len(c.members)):
            bad.append((c.name, "members"))
    assert not bad, bad


def test_member_starts_match_zlib(oracle):
    checked = 0
    for c in G.cases():
        st, _, _, starts, consumed = G.expect(oracle, c.data)
        if st != G.OK:
            continue
        z = G.zlib_starts(c.data)
        if z is None:
            continue
        assert z == starts, c.name
        assert consumed == len(c.data), c.name
        checked += 1
    assert checked > 20


def _bsize_chain(data):
    """member starts following the BC subfields' BSIZE from 0, or None when a member has none or it leaves the file"""
    at, out = 0, []
    while at < len(data):
        if at + 12 > len(data) or not data[at + 3] & 4:
            return None
        x, end, nxt = at + 12, at + 12 + int.from_bytes(data[at + 10:at + 12], "little"), None
        while x + 4 <= end:
            ln = int.from_bytes(data[x + 2:x + 4], "little")
            if data[x:x + 2] == b"BC" and ln == 2:
                nxt = at + int.from_bytes(data[x + 4:x + 6], "little") + 1
            x += 4 + ln
        if nxt is None or nxt > len(data):
            return None
        out.append(at)
        at = nxt
    return out


def test_bgzf_hints(oracle):
    for c in G.bgzf_cases():
        chain = _bsize_chain(c.data)
        starts = G.expect(oracle, c.data)[3]
        if "BSIZE" in c.name:
            assert chain != starts, c.name
        else:
            assert chain == starts, c.name


def test_cuts_cover_the_statuses(oracle):
    seen = {G.expect(oracle, d)[0] for _, d in G.cuts()}
    assert {G.OK, G.GZ_MAGIC} <= seen and len(seen) >= 4, seen
