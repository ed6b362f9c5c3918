"""GPU checks of the gzip reader and writer against the plain-Python DEFLATE reference (tests/deflate_ref.py).

* reader (lb2_inflate_run, gunzip): the crafted corpus -- distances up to 32 768 at and through span starts, every
  length and distance symbol, one-code and empty trees, repeats across HLIT / HDIST, 15-bit and 7-bit codes, fixed-only
  runs, stored edge cases, and the refusals next to them -- at the default span and at 1, 2 and 8 KB spans.  Accepted
  streams equal zlib's bytes, CRC-32 and input length; refused ones return LB2_E_DATA.
* writer (lb2_gzip_*): every output is parsed.  Its block structure, the completeness and limits of its codes, the
  choice of block type by the kernel's byte formula, the optimality of its codes, and that the hard paths (length
  limiting, fixed blocks with matches, distance 32 768, chunk-end truncation, all lengths and distance codes) ran.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

import deflate_ref as R

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- reader
def run(ctx, body):
    """raw DEFLATE body through lb2_inflate_run / read -> (rc, bytes or None, stats)"""
    from lambdipy_b200 import _native as N
    lib = ctx.lib
    d = C.c_void_p()
    ctx.check(lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    try:
        n, st = C.c_uint64(), N.InflateStats()
        buf = C.create_string_buffer(body, max(len(body), 1))
        rc = lib.lb2_inflate_run(d, buf, len(body), C.byref(n), C.byref(st))
        if rc:
            return rc, None, st.as_dict()
        out = C.create_string_buffer(max(n.value, 1))
        ctx.check(lib.lb2_inflate_read(d, out, n.value))
        return 0, out.raw[:n.value], st.as_dict()
    finally:
        lib.lb2_inflate_destroy(d)


def zlib_or_none(body):
    try:
        return zlib.decompress(body, -15)
    except zlib.error:
        return None


@pytest.fixture(scope="module")
def corpus():
    return [(name, body, zlib_or_none(body)) for name, body in R.crafted()]


@pytest.mark.parametrize("span_kb", [None, "1", "2", "8"])
def test_reader_crafted_corpus(gpu_ctx, monkeypatch, corpus, span_kb):
    from lambdipy_b200 import _native as N
    if span_kb:
        monkeypatch.setenv("LB2_INFLATE_SPAN_KB", span_kb)
    else:
        monkeypatch.delenv("LB2_INFLATE_SPAN_KB", raising=False)
    n_ok = n_refused = 0
    for name, body, want in corpus:
        rc, got, st = run(gpu_ctx, body)
        if want is None:
            assert rc == N.LB2_E_DATA and got is None, (name, rc, st)
            n_refused += 1
        else:
            assert rc == 0 and got == want, (name, rc, st)
            assert st["crc32"] == zlib.crc32(want) and st["in_bytes"] == len(body), (name, st)
            n_ok += 1
    assert n_ok > 400 and n_refused > 400, (n_ok, n_refused)


def test_reader_crafted_in_gzip_framing(gpu_ctx, tmp_path):
    from lambdipy_b200.tarball import gunzip
    names = ["far_dynamic@+0.0", "all_syms_dynamic@-3.5", "rep16_first_dist@+5.3", "deep15@+0.7", "eob_only@+0.1",
             "stored_final_padded@+0.2", "fixed_only_run", "sofar_plus1@+0.0", "fixed_dist31@+5.0", "over_cl@-3.0"]
    crafted = dict(R.crafted())
    for name in names:
        body = crafted[name]
        want = zlib_or_none(body)
        data = want or b""
        raw = b"\x1f\x8b\x08\x00\0\0\0\0\x00\xff" + body + zlib.crc32(data).to_bytes(4, "little") + \
            (len(data) & 0xFFFFFFFF).to_bytes(4, "little")
        p = tmp_path / "c.gz"
        p.write_bytes(raw)
        if want is None:
            with pytest.raises(Exception):
                gunzip(str(p), gpu_ctx)
        else:
            assert gunzip(str(p), gpu_ctx) == want, name


def test_reader_fixed_only_run_is_one_span(gpu_ctx, monkeypatch):
    """no block-start candidates: every nominal span is absorbed into span 0"""
    monkeypatch.setenv("LB2_INFLATE_SPAN_KB", "1")
    body = dict(R.unplaced())["fixed_only_run"]
    rc, got, st = run(gpu_ctx, body)
    assert rc == 0 and got == zlib.decompress(body, -15)
    assert st["n_spans"] == 1 and st["n_absorbed"] == (len(body) + 1023) // 1024 - 1, st


@pytest.mark.parametrize("span_kb", ["1", "8"])
def test_reader_far_chain_rounds(gpu_ctx, monkeypatch, span_kb):
    """32 KB stored blocks, each followed by distance-32 768 matches; the chain's round count is printed"""
    monkeypatch.setenv("LB2_INFLATE_SPAN_KB", span_kb)
    body = R.far_chain()
    rc, got, st = run(gpu_ctx, body)
    assert rc == 0 and got == zlib.decompress(body, -15), st
    print("far_chain span %s KB: rounds %d, rejected %d, spans %d" % (span_kb, st["n_rounds"], st["n_rejected"],
                                                                      st["n_spans"]))


# ---------------------------------------------------------------------------------------------------- writer
def gzip_pieces(ctx, pieces):
    """Raw API: DEFLATE the concatenation of `pieces`, one submission each (two in flight).  Returns
    (gzip file bytes, crc32, isize, stats)."""
    from lambdipy_b200 import _native as N
    from lambdipy_b200.tarball import gzip_header
    lib = ctx.lib
    g = C.c_void_p()
    ctx.check(lib.lb2_gzip_create(ctx.h, 0, C.byref(g)))
    cap = max([N.gzip_bound(len(p)) for p in pieces] + [16])
    bufs = [ctx.pinned_alloc(max([len(p) for p in pieces] + [16])) for _ in range(2)]
    out = ctx.pinned_alloc(cap)
    body, in_flight = [], []
    n = C.c_uint64()
    try:
        for i, p in enumerate(pieces):
            if len(in_flight) == 2:
                ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
                body.append(C.string_at(out, n.value))
                in_flight.pop(0)
            buf = bufs[i & 1]
            C.memmove(buf, p, len(p))
            ctx.check(lib.lb2_gzip_submit(g, buf, len(p)))
            in_flight.append(i)
        for _ in in_flight:
            ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
            body.append(C.string_at(out, n.value))
        crc, isize, st = C.c_uint32(), C.c_uint64(), N.GzipStats()
        ctx.check(lib.lb2_gzip_finish(g, out, cap, C.byref(n), C.byref(crc), C.byref(isize), C.byref(st)))
        body.append(C.string_at(out, n.value))
    finally:
        lib.lb2_gzip_destroy(g)
        for b in bufs:
            ctx.pinned_free(b)
        ctx.pinned_free(out)
    data = gzip_header("t.gz", 0) + b"".join(body) + crc.value.to_bytes(4, "little") + (isize.value & 0xFFFFFFFF).to_bytes(4, "little")
    return data, crc.value, isize.value, st.as_dict()


def kernel_lengths(freq, maxbits):
    """deflate.cu's build_lengths restated: Moffat-Katajainen over the weights sorted by (weight, symbol), depths
    clamped to maxbits and the over-subscription repaired by lengthening the shortest leaves that fit"""
    order = sorted((t for t in range(len(freq)) if freq[t]), key=lambda t: (freq[t], t))
    m, out = len(order), [0] * len(freq)
    if m == 1:
        out[order[0]] = 1
    if m < 2:
        return out
    A = [freq[s] for s in order]
    A[0] += A[1]
    root, leaf = 0, 2
    for nxt in range(1, m - 1):
        if leaf >= m or A[root] < A[leaf]:
            A[nxt], A[root], root = A[root], nxt, root + 1
        else:
            A[nxt], leaf = A[leaf], leaf + 1
        if leaf >= m or (root < nxt and A[root] < A[leaf]):
            A[nxt] += A[root]
            A[root], root = nxt, root + 1
        else:
            A[nxt], leaf = A[nxt] + A[leaf], leaf + 1
    A[m - 2] = 0
    for nxt in range(m - 3, -1, -1):
        A[nxt] = A[A[nxt]] + 1
    avbl, used, dpth, root, nxt = 1, 0, 0, m - 2, m - 1
    while avbl > 0:
        while root >= 0 and A[root] == dpth:
            used, root = used + 1, root - 1
        while avbl > used:
            A[nxt], nxt, avbl = dpth, nxt - 1, avbl - 1
        avbl, dpth, used = 2 * used, dpth + 1, 0
    cnt = [0] * (maxbits + 1)
    for a in A:
        cnt[min(a, maxbits)] += 1
    total = sum(cnt[i] << (maxbits - i) for i in range(1, maxbits + 1))
    while total > 1 << maxbits:
        cnt[maxbits] -= 1
        for i in range(maxbits - 1, 0, -1):
            if cnt[i]:
                cnt[i] -= 1
                cnt[i + 1] += 2
                break
        total -= 1
    j = m
    for i in range(1, maxbits + 1):
        for _ in range(cnt[i]):
            j -= 1
            out[order[j]] = i
    return out


def two_codes(freq):
    """the kernel's rule for the distance and code-length codes: at least two codes"""
    f = list(freq)
    nz = sum(1 for x in f if x)
    if nz < 2:
        if not f[0]:
            f[0] = 1
        else:
            f[1] = 1
    if nz == 0:
        f[1] = 1
    return f


def block_freqs(tokens):
    lf, df, extra = [0] * 286, [0] * 30, 0
    for t in tokens:
        if isinstance(t, int):
            lf[t] += 1
        else:
            length, dist, ls = t
            lf[ls] += 1
            ds = R.dist_sym(dist)[0]
            df[ds] += 1
            extra += R.LEXT[ls - 257] + R.DEXT[ds]
    lf[256] = 1
    return lf, df, extra


def kernel_dynamic(lf, df):
    """the dynamic block the kernel would write for these frequencies: (llens, dlens, cllens, rle, header bits)"""
    ll = kernel_lengths(lf, 15)
    dl = kernel_lengths(two_codes(df), 15)
    hlit, hdist = 286, 30
    while hlit > 257 and not ll[hlit - 1]:
        hlit -= 1
    while hdist > 1 and not dl[hdist - 1]:
        hdist -= 1
    rle = R.rle_lengths(ll[:hlit] + dl[:hdist])
    cf = [0] * 19
    for s, _ in rle:
        cf[s] += 1
    cl = kernel_lengths(two_codes(cf), 7)
    hclen = 19
    while hclen > 4 and not cl[R.CLORDER[hclen - 1]]:
        hclen -= 1
    hdr = 17 + 3 * hclen + sum(cl[s] + {16: 2, 17: 3, 18: 7}.get(s, 0) for s, _ in rle)
    return ll[:hlit], dl[:hdist], cl, rle, hdr


def analyse(gz, pieces, st):
    """Parse the writer's output and check it chunk by chunk.  Returns the list of (mode, block) per chunk."""
    whole = b"".join(pieces)
    assert zlib.decompress(gz, wbits=31) == whole
    from lambdipy_b200.tarball import gzip_header
    body = gz[len(gzip_header("t.gz", 0)):-8]
    out, blocks, end = R.parse(body)
    assert out == whole and (end + 7) // 8 == len(body)
    assert body[-2:] == b"\x03\x00" and blocks[-1]["type"] == "fixed" and blocks[-1]["tokens"] == []
    assert blocks[-1]["start"] == 8 * (len(body) - 2)
    assert not any(b["final"] for b in blocks[:-1]) and blocks[-1]["final"]
    sizes = [min(65536, len(p) - i) for p in pieces for i in range(0, len(p), 65536)]
    chunks, k = [], 0
    for clen in sizes:
        b = blocks[k]
        start = b["start"]
        if b["type"] == "stored":
            n = -(-clen // 65535)
            got = [blocks[k + i]["len"] for i in range(n)]
            assert all(blocks[k + i]["type"] == "stored" for i in range(n)) and sum(got) == clen
            assert got == [65535] * (n - 1) + [clen - 65535 * (n - 1)]
            k += n
            mode = 0
        else:
            assert sum(R.token_len(t if isinstance(t, int) else t[:2]) for t in b["tokens"]) == clen
            k += 1
            mode = 1 if b["type"] == "fixed" else 2
        e = blocks[k]
        assert e["type"] == "stored" and e["len"] == 0 and e["end"] % 8 == 0
        assert start % 8 == 0     # every chunk starts byte-aligned
        k += 1
        chunks.append((mode, b, clen, (e["end"] - start) // 8))
        if mode == 2:
            for lens, kind, limit in ((b["llens"], "lens", 15), (b["dlens"], "dists", 15), (b["cllens"], "codes", 7)):
                assert max(lens) <= limit
                nz = [l for l in lens if l]
                assert R.kraft(nz) == 1 << 15 or (kind != "codes" and nz == [1]), (kind, nz)
    assert k == len(blocks) - 1
    assert st["n_chunks"] == len(sizes)
    assert st["n_stored_chunks"] == sum(m == 0 for m, *_ in chunks)
    assert st["n_fixed_chunks"] == sum(m == 1 for m, *_ in chunks)
    return chunks


def check_pricing_and_optimality(chunks):
    """A Huffman chunk is the smallest of dynamic, fixed and stored by the kernel's byte formula (ties: stored, then
    fixed, then dynamic), and its dynamic code, when it has one, is the kernel's and costs what an optimal Huffman code
    costs wherever the optimal code fits the length limit.  Stored chunks are not checked: their tokens are not in the
    output."""
    n_opt = 0
    for mode, b, clen, size in chunks:
        if mode == 0:
            continue
        lf, df, extra = block_freqs(b["tokens"])
        ll, dl, cl, rle, hdr = kernel_dynamic(lf, df)
        fix = 3 + sum(f * l for f, l in zip(lf, R.FIXED_L)) + 5 * sum(df) + extra
        dyn = hdr + R.code_cost(lf, ll) + R.code_cost(df, dl) + extra
        fix_b, dyn_b = (fix + 10) // 8 + 4, (dyn + 10) // 8 + 4
        stored_b = clen + 5 * (-(-clen // 65535)) + 5
        if mode == 1:
            assert fix_b < stored_b and fix_b <= dyn_b and size == fix_b, (fix_b, dyn_b, stored_b, size)
            continue
        assert (b["llens"], b["dlens"], b["cllens"], b["rle"]) == (ll, dl, cl, rle)
        assert b["end"] - b["start"] == dyn
        assert dyn_b < fix_b and dyn_b < stored_b and size == dyn_b, (fix_b, dyn_b, stored_b, size)
        cf = [0] * 19
        for s, _ in rle:
            cf[s] += 1
        for freq, lens, limit in ((lf, ll, 15), (two_codes(df), dl, 15), (two_codes(cf), cl, 7)):
            opt = R.huffman_lengths(freq)
            if max(opt) <= limit:
                assert R.code_cost(freq, lens[:len(freq)] + [0] * (len(freq) - len(lens))) == R.code_cost(freq, opt)
                n_opt += 1
    return n_opt


def gzip_and_check(ctx, pieces):
    gz, crc, isize, st = gzip_pieces(ctx, pieces)
    whole = b"".join(pieces)
    assert crc == zlib.crc32(whole) and isize == len(whole)
    chunks = analyse(gz, pieces, st)
    check_pricing_and_optimality(chunks)
    return chunks


def _text(n, seed):
    import inflate_streams as IS
    return IS.text(n, seed)


def _rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _hist_depths(chunk):
    """optimal literal/length and code-length code depths a chunk's byte histogram alone would give (the kernel's
    matches perturb them a little)"""
    lf = np.bincount(np.frombuffer(chunk, np.uint8), minlength=256).tolist() + [1] + [0] * 29
    ll = kernel_lengths(lf, 15)
    n = 286
    while n > 257 and not ll[n - 1]:
        n -= 1
    cf = [0] * 19
    for s, _ in R.rle_lengths(ll[:n] + [1, 1]):
        cf[s] += 1
    return max(R.huffman_lengths(lf)), max(R.huffman_lengths(cf))


def geometric_chunks():
    """64 KB chunks of shuffled bytes: a tail of 14 symbols with counts 2^k (p_k ~ 2^-k) under a flat body of 242
    symbols.  The body is near-random, so the kernel finds few matches and the tail keeps the optimal literal code
    deeper than 15.  (Bytes drawn from p_k ~ 2^-k alone repeat so much that the matches flatten the literal code.)"""
    counts = [1 << k for k in range(13)] + [1]
    body = (65536 - sum(counts)) // 242
    counts += [body] * 242
    counts[-1] += 65536 - sum(counts)
    sym = np.repeat(np.arange(256, dtype=np.uint8), counts)
    out = [np.random.default_rng(seed).permutation(sym).tobytes() for seed in range(6)]
    assert all(_hist_depths(c)[0] > 15 for c in out)
    return out


def deep_cl_chunks():
    """64 KB chunks of i.i.d. bytes with weights 2^-U(0, s) (entropy about 7 bits, so few matches), kept where the
    histogram's optimal code-length code is deeper than 7"""
    out = []
    for seed in (112, 7, 37, 160):
        rng = np.random.default_rng(seed)
        w = 2.0 ** -(rng.uniform(0, rng.uniform(4, 12), 256))
        w /= w.sum()
        r2 = np.random.default_rng(1000 + seed)
        for _ in range(16):
            c = r2.choice(256, 65536, p=w).astype(np.uint8).tobytes()
            if _hist_depths(c)[1] > 7:
                out.append(c)
    return out


def test_writer_structure_and_pricing(gpu_ctx):
    import inflate_streams as IS
    n_opt = 0
    for pieces in ([_text(300_000, 1)], [IS.so_bytes(1 << 20)], [_rand(150_000, 2)], [b"\x00"], [b"ab" * 40],
                   [_text(70_000, 3), _rand(3000, 4), _text(100, 5)], [bytes(200_000)]):
        gz, crc, isize, st = gzip_pieces(gpu_ctx, pieces)
        n_opt += check_pricing_and_optimality(analyse(gz, pieces, st))
    assert n_opt > 50


def check_length_limited(chunks, which, limit):
    deep = 0
    for mode, b, *_ in chunks:
        if mode != 2:
            continue
        lf, df, _ = block_freqs(b["tokens"])
        if which == "lit":
            freq, lens = lf, b["llens"]
        else:
            cf = [0] * 19
            for s, _ in b["rle"]:
                cf[s] += 1
            freq, lens = two_codes(cf), b["cllens"]
        if max(R.huffman_lengths(freq)) > limit:
            deep += 1
            assert max(lens) <= limit and R.kraft(lens) == 1 << 15
    return deep


def test_writer_length_limit_15(gpu_ctx):
    pieces = geometric_chunks()
    assert len(pieces) >= 4
    chunks = gzip_and_check(gpu_ctx, [b"".join(pieces)])
    assert check_length_limited(chunks, "lit", 15) >= 1


def test_writer_length_limit_7(gpu_ctx):
    pieces = deep_cl_chunks()
    assert len(pieces) >= 4
    chunks = gzip_and_check(gpu_ctx, [b"".join(pieces)])
    assert check_length_limited(chunks, "cl", 7) >= 1


def periodic_tails():
    rng = np.random.default_rng(9)
    out = []
    for period in range(1, 41):
        pat = rng.integers(0, 256, period, dtype=np.uint8).tobytes()
        n = int(rng.integers(period + 115, 301))
        out.append((pat * (n // period + 1))[:n])
    return out


def check_fixed_with_matches(chunk_lists):
    lsyms, dcodes = set(), set()
    for chunks in chunk_lists:
        for mode, b, *_ in chunks:
            if mode == 1:
                for t in b["tokens"]:
                    if isinstance(t, tuple):
                        lsyms.add(t[2])
                        dcodes.add(R.dist_sym(t[1])[0])
    assert lsyms & set(range(280, 286)) == set(range(280, 286)), sorted(lsyms)
    assert len(dcodes) >= 10, sorted(dcodes)


def test_writer_fixed_chunks_with_matches(gpu_ctx):
    text = _text(65536, 6)
    res = []
    for tail in periodic_tails():
        res.append(gzip_and_check(gpu_ctx, [tail]))
        res.append(gzip_and_check(gpu_ctx, [text, tail]))
    check_fixed_with_matches(res)


def check_dist_32768(chunks):
    assert any(isinstance(t, tuple) and t[1] == 32768 for mode, b, *_ in chunks if mode for t in b["tokens"])


def test_writer_distance_32768(gpu_ctx):
    r = _rand(32768, 7)
    data = r + r[:20000]
    check_dist_32768(gzip_and_check(gpu_ctx, [data]))
    check_dist_32768(gzip_and_check(gpu_ctx, [data[:32768], data[32768:]]))


def test_writer_chunk_end_truncation(gpu_ctx):
    """a zero run through the end of each piece's first chunk; the last match before the chunk end has `left`
    bytes, 0..258, to take"""
    pat = bytes(np.random.default_rng(10).integers(1, 256, 997, dtype=np.uint8))   # no zero byte: cheap to parse
    pieces = []
    for left in range(259):
        s = 65536 - left - 1 - 258 * 4
        pieces.append((pat * (s // 997 + 1))[:s] + bytes(65536 - s + 300))
    chunks = gzip_and_check(gpu_ctx, pieces)
    ends = set()
    for i in range(259):
        mode, b, clen, _ = chunks[2 * i]
        assert mode and clen == 65536
        last = b["tokens"][-1]
        ends.add(last[0] if isinstance(last, tuple) else 1)
    assert ends >= set(range(3, 259)), sorted(set(range(3, 259)) - ends)


def coverage_input():
    """Planted copies of every length 3..258 (twice) at distances that cycle through all 30 codes.  Each copy's
    source is fresh 7-bit random bytes that no other copy reads, the bytes around the copy differ from those around
    its source, and no copy crosses a chunk boundary, so the longest match is exactly the copy."""
    rng = np.random.default_rng(8)

    def fresh(n):
        return rng.integers(0, 128, n, dtype=np.uint8).tobytes()
    out = bytearray(fresh(64))
    for k, length in enumerate(list(range(3, 259)) * 2):
        code = k % 30
        dist = min(R.DBASE[code] + int(rng.integers(0, 1 << R.DEXT[code])), 32768)
        if length == 3 and dist > 4096:
            dist = 1 + k % 4096
        n = max(dist, 8)
        at = len(out) + n
        if at // 65536 != (at + length + 1) // 65536:
            out += fresh(65536 - at % 65536 + 8)
        out += fresh(n)
        out[-1] = out[-1 - dist] ^ 0x5A              # the byte in front of the copy differs from the source's
        for _ in range(length):
            out.append(out[-dist])
        out.append(out[-dist] ^ 0xA5)                # and so does the byte after it
    return bytes(out)


def check_coverage(chunks):
    lengths, dcodes = set(), set()
    for mode, b, *_ in chunks:
        if mode:
            for t in b["tokens"]:
                if isinstance(t, tuple):
                    lengths.add(t[0])
                    dcodes.add(R.dist_sym(t[1])[0])
    assert lengths >= set(range(3, 259)), sorted(set(range(3, 259)) - lengths)
    assert dcodes == set(range(30)), sorted(set(range(30)) - dcodes)


def test_writer_every_length_and_distance_code(gpu_ctx):
    check_coverage(gzip_and_check(gpu_ctx, [coverage_input()]))
