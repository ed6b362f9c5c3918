"""GPU checks of the seek table: GpuGzipFile / gzip_tarball / strip_tarball with seek_table=True (lb2_gzip_chunk_sizes)
at the default mode and level 9, at 64 MB, 1 MB and odd piece sizes, write the no-table file plus one member; the file
reads back through lb2_inflate_run_table with the bytes and CRC-32 of the search path and no find or count rounds;
tampered tables fall back with the search path's bytes and are refused exactly where the CPU emulator of the same core
refuses them; output is deterministic; extraction gives the tree of the no-table file."""
import ctypes as C
import gzip
import io
import os
import subprocess
import tarfile

import numpy as np
import pytest

import inflate_streams as IS
import seek_streams as SS
from lambdipy_b200 import _native as N
from lambdipy_b200 import seek_table as ST
from lambdipy_b200 import tarball as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ctx():
    c = N.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def payload():
    rnd = np.random.default_rng(3).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    return IS.so_bytes(5 << 20) + IS.text(2 << 20) + rnd + bytes(300000)


def write(ctx, path, data, **kw):
    """path/t.gz: the same gzip header (FNAME, MTIME) for every path"""
    path.mkdir()
    with T.GpuGzipFile(str(path / "t.gz"), mtime=7, ctx=ctx, **kw) as gz:
        gz.write(data)
    return gz.stats


def read(ctx, path):
    """(bytes, summed stats, counts) through inflate_members"""
    d = C.c_void_p()
    ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    outs, stats, counts = [], {}, {}
    try:
        def keep(isize, last, st):
            buf = C.create_string_buffer(max(isize, 1))
            ctx.check(ctx.lib.lb2_inflate_read(d, buf, isize))
            outs.append(buf.raw[:isize])
            for k, v in st.as_dict().items():
                stats[k] = stats.get(k, 0) + v
        T.inflate_members(ctx, d, str(path), keep, counts)
    finally:
        ctx.lib.lb2_inflate_destroy(d)
    return b"".join(outs), stats, counts


def run_table(ctx, body, entries):
    """lb2_inflate_run_table on body -> (rc, bytes | None, in_bytes, crc32, used, refused)"""
    d = C.c_void_p()
    ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    try:
        spans = (N.InflateSpan * max(len(entries), 1))()
        for i, (c, u) in enumerate(entries):
            spans[i].in_len, spans[i].out_len = c, u
        out_n, st, used, refused = C.c_uint64(), N.InflateStats(), C.c_uint32(), C.c_uint32()
        rc = ctx.lib.lb2_inflate_run_table(d, body, len(body), spans, len(entries), C.byref(out_n), C.byref(st),
                                           C.byref(used), C.byref(refused))
        data = None
        if rc == N.LB2_OK:
            buf = C.create_string_buffer(max(out_n.value, 1))
            ctx.check(ctx.lib.lb2_inflate_read(d, buf, out_n.value))
            data = buf.raw[:out_n.value]
        return rc, data, st.in_bytes, st.crc32, used.value, refused.value, st
    finally:
        ctx.lib.lb2_inflate_destroy(d)


@pytest.mark.parametrize("level", [None, 9])
@pytest.mark.parametrize("piece", [64 << 20, 1 << 20, 3 * 65536 + 4097])
def test_writer_and_reader(ctx, tmp_path, payload, level, piece):
    st0 = write(ctx, tmp_path / "a.gz", payload, piece_bytes=piece, compresslevel=level)
    st1 = write(ctx, tmp_path / "b.gz", payload, piece_bytes=piece, compresslevel=level, seek_table=True)
    plain, indexed = (tmp_path / "a.gz" / "t.gz").read_bytes(), (tmp_path / "b.gz" / "t.gz").read_bytes()
    off, entries = ST.gzip_tail(indexed)
    assert indexed[:off] == plain and off == len(plain)
    assert gzip.decompress(indexed) == payload
    assert st1["seek_entries"] == len(entries) and st0["out_bytes"] == st1["out_bytes"]
    body = len(T.gzip_header("t.gz"))
    assert ST.valid(entries, len(plain) - 8 - body, len(payload))
    n_chunks = sum(-(-min(piece, len(payload) - p) // ST.CHUNK) for p in range(0, len(payload), piece))
    assert len(entries) == n_chunks
    got, st, counts = read(ctx, tmp_path / "b.gz" / "t.gz")
    assert got == payload and counts == {"seek_table": 1, "seek_table_refused": 0}
    assert st["n_rounds"] == 0 and st["find_ms"] == 0 and st["count_ms"] == 0 and st["n_spans"] == len(entries)
    want, st_plain, counts_plain = read(ctx, tmp_path / "a.gz" / "t.gz")
    assert want == payload and counts_plain == {} and st["crc32"] == st_plain["crc32"]
    assert st["in_bytes"] == st_plain["in_bytes"] and st_plain["n_rounds"] >= 1
    write(ctx, tmp_path / "c.gz", payload, piece_bytes=piece, compresslevel=level, seek_table=True)
    assert (tmp_path / "c.gz" / "t.gz").read_bytes() == indexed


def test_tampered_tables_on_the_device(ctx):
    from test_seek_table_emulated import Emu
    emu = Emu()
    n = 0
    for name, body, data, entries in SS.matrix():
        padded = body + bytes(8)
        rc, out, ib, crc, used, refused, st = run_table(ctx, padded, entries)
        assert (rc, out, ib, used, refused) == (0, data, len(body), 1, 0), name
        assert st.n_rounds == 0
        for how, t in SS.tampered(entries):
            rc, out, ib, crc2, used, refused, _ = run_table(ctx, padded, t)
            assert (rc, out, ib, crc2) == (0, data, len(body), crc), (name, how)
            assert used == emu.table(padded, t)[3] and refused == 1 - used, (name, how)
            n += t != entries
    assert n > 100


def _tree(root):
    os.makedirs(os.path.join(root, "pkg", "lib"))
    for i, f in enumerate(sorted(x for x in os.listdir(GOLDEN) if x.endswith(".in.bin"))):
        with open(os.path.join(GOLDEN, f), "rb") as s, open(os.path.join(root, "pkg", "lib", "m%d.so" % i), "wb") as d:
            d.write(s.read())
    with open(os.path.join(root, "pkg", "data.txt"), "wb") as d:
        d.write(IS.text(3 << 20))
    return os.path.join(root, "pkg")


def _members(raw):
    with tarfile.open(fileobj=io.BytesIO(gzip.decompress(raw)), mode="r:") as tar:
        return [(m.name, m.size) for m in tar.getmembers()]


@pytest.mark.parametrize("level", [None, 9])
def test_tarball_strip_and_extract(ctx, tmp_path, level):
    src = _tree(str(tmp_path / "t"))
    kw = {} if level is None else {"compresslevel": level}
    pa, pb = tmp_path / "a" / "pkg.tar.gz", tmp_path / "b" / "pkg.tar.gz"
    pa.parent.mkdir()
    pb.parent.mkdir()
    T.gzip_tarball([src], str(pa), ctx=ctx, **kw)
    T.gzip_tarball([src], str(pb), ctx=ctx, seek_table=True, **kw)
    a, b = pa.read_bytes(), pb.read_bytes()
    off, _ = ST.gzip_tail(b)
    assert b[:4] + b[8:off] == a[:4] + a[8:]            # MTIME is the clock's
    subprocess.run(["gzip", "-t", str(pb)], check=True)
    T.extract_tarball(str(pb), str(tmp_path / "xb"), ctx=ctx)
    with tarfile.open(pa, "r:gz") as tar:
        tar.extractall(tmp_path / "xa", filter="fully_trusted")
    for d, _, fs in os.walk(tmp_path / "xa"):
        for f in fs:
            p = os.path.join(d, f)
            q = os.path.join(tmp_path / "xb", os.path.relpath(p, tmp_path / "xa"))
            assert open(p, "rb").read() == open(q, "rb").read(), p
    # strip_tarball: a table source is read from the table; the output with a table is the output without plus one member
    out = {k: tmp_path / k / "out.tar.gz" for k in ("s0", "s1", "s2", "s3")}
    s0 = T.strip_tarball(str(pb), str(out["s0"]), ctx=ctx, **kw)
    s1 = T.strip_tarball(str(pb), str(out["s1"]), ctx=ctx, seek_table=True, piece_bytes=1 << 20, **kw)
    s2 = T.strip_tarball(str(pb), str(out["s2"]), ctx=ctx, piece_bytes=1 << 20, **kw)
    assert s0["inflate"]["seek_table"] == 1 and s0["inflate"]["n_rounds"] == 0 and s0["gpu"] + s0["fallback"] >= 1
    r1, r2 = out["s1"].read_bytes(), out["s2"].read_bytes()
    off, _ = ST.gzip_tail(r1)
    assert r1[:off] == r2 and gzip.decompress(r1) == gzip.decompress(out["s0"].read_bytes())
    assert _members(r1) == _members(r2)
    s3 = T.strip_tarball(str(out["s1"]), str(out["s3"]), ctx=ctx, **kw)
    assert s3["inflate"]["seek_table"] == 1 and s1["deflate"]["seek_entries"] >= 2 and s2["gpu"] == s1["gpu"]


def test_chunk_sizes_abi(ctx):
    g = C.c_void_p()
    ctx.check(ctx.lib.lb2_gzip_create(ctx.h, 0, C.byref(g)))
    try:
        k = C.c_uint32()
        assert ctx.lib.lb2_gzip_chunk_sizes(g, None, 0, C.byref(k)) == N.LB2_E_STATE
        data = IS.text(200000)
        buf = C.create_string_buffer(data, len(data))
        ctx.check(ctx.lib.lb2_gzip_submit(g, buf, len(data)))
        out = C.create_string_buffer(N.gzip_bound(len(data)))
        n = C.c_uint64()
        ctx.check(ctx.lib.lb2_gzip_collect(g, out, len(out), C.byref(n)))
        sizes = (C.c_uint32 * 4)()
        assert ctx.lib.lb2_gzip_chunk_sizes(g, sizes, 2, C.byref(k)) == N.LB2_E_CAPACITY and k.value == 4
        ctx.check(ctx.lib.lb2_gzip_chunk_sizes(g, sizes, 4, C.byref(k)))
        assert k.value == 4 and sum(sizes) == n.value
        before = list(sizes)
        ctx.check(ctx.lib.lb2_gzip_submit(g, buf, len(data)))   # the other slot: the sizes stay readable
        sizes = (C.c_uint32 * 4)()
        ctx.check(ctx.lib.lb2_gzip_chunk_sizes(g, sizes, 4, C.byref(k)))
        assert k.value == 4 and list(sizes) == before
    finally:
        ctx.lib.lb2_gzip_destroy(g)


def _zip_tree_src(root):
    """a tree whose zip mixes stored-size, one-chunk, one-span and many-chunk members"""
    os.makedirs(os.path.join(root, "d", "e"))
    files = {"empty": b"", "tiny": b"x" * 10, "one.txt": IS.text(50000), "two.bin": IS.so_bytes(130000),
             "big.bin": IS.so_bytes(3 << 20), "d/e/text": IS.text(2 << 20),
             "rand": np.random.default_rng(9).integers(0, 256, 700000, dtype=np.uint8).tobytes()}
    for i, f in enumerate(sorted(x for x in os.listdir(GOLDEN) if x.endswith(".in.bin"))):
        with open(os.path.join(GOLDEN, f), "rb") as g:
            files["d/m%d.so" % i] = g.read()
    for name, data in files.items():
        with open(os.path.join(root, name), "wb") as f:
            f.write(data)
    return files


@pytest.mark.parametrize("level", [None, 9])
@pytest.mark.parametrize("piece", [64 << 20, 1 << 20])
def test_zip_tree_extract_testzip_strip(ctx, tmp_path, level, piece):
    import zipfile
    from lambdipy_b200 import zipfile_gpu as Z
    src = str(tmp_path / "src")
    os.makedirs(src)
    files = _zip_tree_src(src)
    kw = {} if level is None else {"compresslevel": level}
    pa, pb = tmp_path / "a" / "t.zip", tmp_path / "b" / "t.zip"
    Z.zip_tree(src, str(pa), ctx=ctx, piece_bytes=piece, **kw)
    Z.zip_tree(src, str(pb), ctx=ctx, piece_bytes=piece, seek_table=True, **kw)
    a, b = pa.read_bytes(), pb.read_bytes()
    with zipfile.ZipFile(pa) as za, zipfile.ZipFile(pb) as zb:
        assert b[:za.start_dir] == a[:za.start_dir] and zb.testzip() is None
        tabled = [zi.filename for zi in zb.infolist() if Z._seek_entries(zi)]
        for zi in zb.infolist():
            if not zi.is_dir():
                assert zb.read(zi) == files[zi.filename]
    assert sorted(tabled) == sorted(k for k, v in files.items() if len(v) > ST.CHUNK)
    with zipfile.ZipFile(pb) as zb:
        expect = sum(1 for zi in zb.infolist() if Z._seek_entries(zi) and zi.compress_size > 128 << 10)
    # reading: the same trees and testzip answers, members larger than a span decoded from their tables
    sa = Z.extract_zip(str(pa), str(tmp_path / "xa"), ctx=ctx)
    sb = Z.extract_zip(str(pb), str(tmp_path / "xb"), ctx=ctx)
    for name, data in files.items():
        assert (tmp_path / "xb" / name).read_bytes() == data == (tmp_path / "xa" / name).read_bytes()
    assert expect >= 2 and sb["seek_table"] == expect and sb["seek_table_refused"] == 0 and "seek_table" not in sa
    assert Z.testzip(str(pb), ctx=ctx) is None
    # strip_zip: kept members keep their tables in the central directory only, rewritten ones get new ones
    s0 = Z.strip_zip(str(pb), str(tmp_path / "s0" / "o.zip"), ctx=ctx, **kw)
    s1 = Z.strip_zip(str(pb), str(tmp_path / "s1" / "o.zip"), ctx=ctx, seek_table=True, **kw)
    with zipfile.ZipFile(pb) as zb:   # a selected member is read from its table when it is larger than one span
        want = sum(1 for zi in zb.infolist() if zi.filename.endswith(".so") and Z._seek_entries(zi) and
                   zi.compress_size > 128 << 10)
    assert s0["unzip"].get("seek_table", 0) == want and s0["unzip"].get("seek_table_refused", 0) == 0
    with zipfile.ZipFile(tmp_path / "s0" / "o.zip") as z0, zipfile.ZipFile(tmp_path / "s1" / "o.zip") as z1:
        r0, r1 = (tmp_path / "s0" / "o.zip").read_bytes(), (tmp_path / "s1" / "o.zip").read_bytes()
        assert r1[:z0.start_dir] == r0[:z0.start_dir]
        assert z0.testzip() is None and z1.testzip() is None
        t0 = {zi.filename for zi in z0.infolist() if Z._seek_entries(zi)}
        t1 = {zi.filename for zi in z1.infolist() if Z._seek_entries(zi)}
        kept = {k for k, v in files.items() if len(v) > ST.CHUNK and not k.endswith(".so")}
        assert t0 == kept and t1 == kept | {zi.filename for zi in z1.infolist()
                                            if zi.filename.endswith(".so") and zi.file_size > ST.CHUNK}
        for zi in z0.infolist():
            assert z0.read(zi) == z1.read(zi.filename)
            assert ST.zip_field_of(_local_extra(r0, zi)) == b""
    assert s1["gpu"] + s1["fallback"] == sum(k.endswith(".so") for k in files)


def test_unzip_tampered_tables_in_one_batch(ctx):
    """table and no-table, stored and one-span members in one batch; a tampered table falls back"""
    from lambdipy_b200 import zipfile_gpu as Z
    streams = SS.matrix()
    members, tables, want, blob = [], [], [], bytearray()
    for i, (name, body, data, entries) in enumerate(streams):
        members.append((len(blob), len(body), len(data), zlib_crc(data), 8))
        blob += body
        tables.append(entries if i % 3 else SS.tampered(entries)[i % 12][1])
        want.append(data)
    members.append((len(blob), 5, 5, zlib_crc(b"abcde"), 0))
    blob += b"abcde"
    tables.append(None)
    want.append(b"abcde")
    with Z.GpuUnzipDecoder(ctx) as dec:
        view = dec.buffer(len(blob))
        view[:] = blob
        got = dec.run(len(blob), members, tables=tables)
        st = dec.stats()
        assert [(s, bytes(d)) for s, d in got] == [(0, w) for w in want]
        plain = dec.run(len(blob), members)
        assert [bytes(d) for _, d in plain] == want
    honest = sum(1 for i in range(len(streams)) if i % 3)
    assert st["seek_table"] == honest and st["seek_table_refused"] == len(streams) - honest


def zlib_crc(b):
    import zlib
    return zlib.crc32(b)


def _local_extra(raw, zi):
    import struct
    import zipfile
    fh = struct.unpack(zipfile.structFileHeader, raw[zi.header_offset:zi.header_offset + zipfile.sizeFileHeader])
    at = zi.header_offset + zipfile.sizeFileHeader + fh[zipfile._FH_FILENAME_LENGTH]
    return raw[at:at + fh[zipfile._FH_EXTRA_FIELD_LENGTH]]
