"""CPU checks of the DEFLATE reference (tests/deflate_ref.py) and, through the emulated decoder core, of the gzip
reader's logic on streams zlib never writes: the reference parser must equal zlib on zlib's own streams, agree with
zlib on accept versus refuse over the crafted corpus, and the emulated pipeline must decode every crafted stream to
zlib's bytes or refuse it exactly when zlib does, at span sizes from 64 B to 64 KB."""
import zlib

import pytest

import deflate_ref as R
import inflate_streams as IS
from test_inflate_emulated import Emu


def zlib_or_none(body):
    try:
        return zlib.decompress(body, -15)
    except zlib.error:
        return None


def parse_or_none(body):
    try:
        return R.parse(body, keep_tokens=False)[0]
    except R.DeflateError:
        return None


@pytest.fixture(scope="module")
def corpus():
    """every item at the span start at all 8 bit phases, and 3 bytes before / 5 bytes after it at phases 0 and 5"""
    out = R.crafted(deltas=(0,)) + R.crafted(deltas=(-3, 5), phases=(0, 5))[:-len(R.unplaced())]
    return [(name, body, zlib_or_none(body)) for name, body in out]


@pytest.fixture(scope="module")
def emu():
    return Emu()


def test_parse_equals_zlib_on_stream_matrix():
    for name, body, data in IS.matrix(48 << 10):
        out, blocks, end = R.parse(body)
        assert out == data, name
        assert (end + 7) // 8 == len(body), name
        assert blocks[-1]["final"] and not any(b["final"] for b in blocks[:-1]), name


def test_crafted_corpus_covers_accept_and_refuse(corpus):
    kinds = {}
    for name, _, want in corpus:
        kinds.setdefault(name.split("@")[0], set()).add(want is not None)
    refused = {"sofar_plus1", "sofar_plus1_fixed", "sofar_plus1_span0", "fixed_286", "fixed_287", "fixed_dist30",
               "fixed_dist31", "over_lit", "incomplete_lit", "over_dist", "incomplete_dist", "over_cl",
               "incomplete_cl", "one_cl_code", "missing_eob_len", "hclen4", "hlit287", "hdist31", "rep16_at_start",
               "rep_overrun", "btype3"}
    for k, v in kinds.items():
        if k == "missing_eob_end":   # zero padding after the last literal can read as the fixed end-of-block code
            assert False in v, k
        else:
            assert v == {k not in refused}, (k, v)


def test_parse_agrees_with_zlib_on_crafted_corpus(corpus):
    for name, body, want in corpus:
        assert parse_or_none(body) == want, name


def test_crafted_structure():
    """the corpus holds what its names say: parse sees the trees and symbols"""
    def blocks(name):
        return [b for b in R.parse(R.place(name, 0, 3))[1] if b["type"] == "dynamic"]
    far = R.parse(R.place("far_dynamic", 0, 0))[1]
    toks = [t for b in far for t in b.get("tokens", []) if isinstance(t, tuple)]
    assert {t[1] for t in toks} >= set(range(32507, 32769)) and (258, 32768, 284) in toks and (258, 32768, 285) in toks
    syms = R.parse(R.place("all_syms_fixed", 0, 0))[1]
    toks = [t for b in syms if b["type"] == "fixed" for t in b["tokens"] if isinstance(t, tuple)]
    assert {t[2] for t in toks} == set(range(257, 286)) and {R.dist_sym(t[1])[0] for t in toks} == set(range(30))
    b, = blocks("all_syms_dynamic")
    assert b["hlit"] == 286 and b["hdist"] == 30
    b, = blocks("one_dist_code")
    assert [l for l in b["dlens"] if l] == [1]
    b, = blocks("empty_dist_tree")
    assert not any(b["dlens"])
    b, = blocks("eob_only")
    assert [i for i, l in enumerate(b["llens"]) if l] == [256] and b["tokens"] == []
    b, = blocks("rep16_first_dist")
    at, i = 0, 0
    while at < b["hlit"]:
        s, x = b["rle"][i]
        at += 1 if s < 16 else 3 + x if s == 16 else 3 + x if s == 17 else 11 + x
        i += 1
    assert at == b["hlit"] and b["rle"][i][0] == 16
    for name, sym in (("rep16_across", 16), ("rep18_across", 18), ("rep17_across", 17)):
        b, = blocks(name)
        at, crossed = 0, set()
        for s, x in b["rle"]:
            n = 1 if s < 16 else 3 + x if s in (16, 17) else 11 + x
            if at < b["hlit"] < at + n:
                crossed.add(s)
            at += n
        assert sym in crossed, name
    assert blocks("hclen5")[0]["hclen"] == 5 and blocks("hclen19")[0]["hclen"] == 19
    assert blocks("hlit257_one_code")[0]["hlit"] == 257 and blocks("hlit257_one_code")[0]["hdist"] == 1
    b, = blocks("deep15")
    used = {t if isinstance(t, int) else t[2] for t in b["tokens"]} | {256}
    assert max(b["llens"][s] for s in used) == 15
    assert max(b["dlens"][R.dist_sym(t[1])[0]] for t in b["tokens"] if isinstance(t, tuple)) == 15
    b, = blocks("cl7")
    assert max(b["cllens"]) == 7 and max(b["cllens"][s] for s, _ in b["rle"]) == 7
    blk = R.parse(R.place("stored_final_padded", 0, 2))[1][-1]
    assert blk["type"] == "stored" and blk["final"] and (blk["start"] + 3) % 8 != 0
    assert all(b["type"] == "fixed" for b in R.parse(dict(R.unplaced())["fixed_only_run"])[1])


@pytest.mark.parametrize("span", [64, 1024, 3000, 8192, 65536])
def test_emulated_core_on_crafted_corpus(emu, corpus, span):
    for name, body, want in corpus:
        st, got, stats = emu.inflate(body, span)
        if want is None:
            assert st != 0 and got is None, (name, st, stats)
        else:
            assert st == 0 and got == want, (name, st, stats)
            assert stats["in_bytes"] == len(body), (name, stats)


def test_far_distance_chain_rounds(emu):
    """stored 32 KB blocks, each followed by a fixed block of distance-32 768 matches: every span start after the
    first is a stored block the chain has to confirm (the count is recorded, not bounded)"""
    body = R.far_chain()
    for span in (1024, 8192):
        st, got, stats = emu.inflate(body, span)
        assert st == 0 and got == zlib.decompress(body, -15), stats
        print("far_chain span %d: %s" % (span, stats))
