"""CPU checks of the seek-table format (lambdipy_b200/seek_table.py) and of everything around it that needs no GPU:
the round trip and the choice of k at the field's limit; a gzip file with a table, built from a zlib stream flushed at
64 KB (what the GPU writer writes), is the no-table file plus one member, and gzip, tar, tarfile and gzip.decompress
read it as the same tree; the reader's tail detection (tarball._seek_spans) takes exactly [data member][table member]
and refuses near-misses; the LAMBDIPY_SEEK_TABLE variable and the --seek-table flag."""
import gzip
import io
import os
import shutil
import struct
import subprocess
import tarfile
import zlib

import pytest

import seek_streams as SS
from lambdipy_b200 import seek_table as ST
from lambdipy_b200 import tarball as T


def test_varints_round_trip():
    entries = [(1, 1), (127, 128), (16383, 16384), (2 ** 63, 2 ** 64 - 1), (65541, 65536)]
    assert ST.decode(ST.encode(entries)) == entries
    assert ST.encode([(1, 300)]) == b"\x01\xac\x02"
    assert ST.decode(b"\x01\xac") is None                          # truncated varint
    assert ST.decode(b"\x01") is None                              # odd count
    assert ST.decode(b"\xff" * 9 + b"\x02" + b"\x01") is None      # past 64 bits
    assert ST.decode(b"") == []


def test_runs_and_the_choice_of_k():
    chunks = [(1000 + i, ST.CHUNK) for i in range(10)] + [(500, 100)]
    assert ST.runs(chunks, 1) == chunks
    assert ST.runs(chunks, 4) == [(4006, 4 * ST.CHUNK), (4022, 4 * ST.CHUNK), (2517, 2 * ST.CHUNK + 100)]
    # a short chunk (the end of a piece) ends a run
    pieces = [(10, ST.CHUNK), (10, 5), (10, ST.CHUNK), (10, ST.CHUNK), (10, 7)]
    assert ST.runs(pieces, 3) == [(20, ST.CHUNK + 5), (30, 2 * ST.CHUNK + 7)]
    one = len(ST.encode(chunks))
    assert ST.build(chunks, one) == chunks
    assert ST.build(chunks, one - 1) == ST.runs(chunks, 2)
    assert ST.build([(10, 100)]) is None and ST.build([(10, ST.CHUNK)] * 2, 3) is None
    # torch/lib scale: 23 300 chunks of about 45 % need runs of 3 to fit the gzip field
    big = [(30000, ST.CHUNK)] * 23300
    entries = ST.build(big)
    assert len(ST.encode(entries)) <= ST.GZIP_LIMIT and len(ST.encode(ST.runs(big, 2))) > ST.GZIP_LIMIT
    assert entries == ST.runs(big, 3)


def test_valid():
    e = [(100, ST.CHUNK), (50, 10)]
    assert ST.valid(e, 150, ST.CHUNK + 10)
    assert not ST.valid(e, 151, ST.CHUNK + 10) and not ST.valid(e, 150, ST.CHUNK + 11)
    assert ST.valid(e, 150, (ST.CHUNK + 10) | 1 << 32, 0xFFFFFFFF)
    assert not ST.valid(e[:1], 100, ST.CHUNK)
    assert not ST.valid([(0, 0), (100, ST.CHUNK)], 100, ST.CHUNK)
    assert not ST.valid([(1, 1033), (100, 10)], 101, 1043) and ST.valid([(1, 1032), (100, 10)], 101, 1042)


def _gzip_files(tmp_path, data):
    """(no-table file, table file) around the DEFLATE body zlib writes when flushed every 64 KB, as the GPU writer is"""
    body, chunks = SS.flushed(data, SS.every(len(data), ST.CHUNK))
    head = T.gzip_header("t.tar.gz", mtime=1234)
    plain = head + body + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)
    entries = ST.build(chunks)
    indexed = plain + ST.gzip_member(entries, len(plain))
    (tmp_path / "plain.tar.gz").write_bytes(plain)
    (tmp_path / "indexed.tar.gz").write_bytes(indexed)
    return plain, indexed, entries


def _tar_bytes(root):
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        tar.add(root, arcname="pkg")
    return buf.getvalue()


@pytest.fixture
def tree(tmp_path):
    root = tmp_path / "src"
    (root / "lib").mkdir(parents=True)
    (root / "lib" / "a.txt").write_bytes(SS.IS.text(300000))
    (root / "lib" / "b.bin").write_bytes(SS.IS.so_bytes(200000))
    (root / "c").write_bytes(os.urandom(70000))
    return root


def _snapshot(root):
    return {os.path.relpath(os.path.join(d, f), root): open(os.path.join(d, f), "rb").read()
            for d, _, fs in os.walk(root) for f in fs}


def test_file_is_the_plain_file_plus_one_member_and_tools_read_it(tmp_path, tree):
    data = _tar_bytes(tree)
    plain, indexed, entries = _gzip_files(tmp_path, data)
    off, got = ST.gzip_tail(indexed)
    assert indexed[:off] == plain and got == entries and off == len(plain)
    assert indexed[-22:-20] == b"LO" and indexed[-10:] == b"\x03\x00" + bytes(8)
    assert gzip.decompress(indexed) == data
    with tarfile.open(tmp_path / "indexed.tar.gz", "r:gz") as tar:
        tar.extractall(tmp_path / "x1", filter="fully_trusted")
    assert _snapshot(tmp_path / "x1" / "pkg") == _snapshot(tree)
    if shutil.which("gzip"):
        subprocess.run(["gzip", "-t", str(tmp_path / "indexed.tar.gz")], check=True)
    if shutil.which("tar"):
        listing = subprocess.run(["tar", "-tzf", str(tmp_path / "indexed.tar.gz")], check=True, capture_output=True).stdout
        assert listing == subprocess.run(["tar", "-tzf", str(tmp_path / "plain.tar.gz")], check=True,
                                         capture_output=True).stdout


def test_reader_takes_exactly_data_then_table(tmp_path, tree):
    data = _tar_bytes(tree)
    plain, indexed, entries = _gzip_files(tmp_path, data)

    def spans(raw):
        end, sp = T._seek_spans(bytearray(raw), len(raw))
        return end, None if sp is None else [(s.in_len, s.out_len) for s in sp]
    assert spans(indexed) == (len(plain), entries)
    assert spans(plain) == (len(plain), None)
    head = indexed[:len(plain)]
    member = indexed[len(plain):]
    near = {
        "fname": head + member[:3] + bytes([member[3] | 8]) + member[4:],
        "offset": head + member[:-18] + struct.pack("<Q", len(plain) + 1) + member[-10:],
        "trailing": indexed + b"\0",
        "two-data": head + head + ST.gzip_member(entries, 2 * len(plain)),
        "sums": head + ST.gzip_member(entries[:-1] + [(entries[-1][0] + 1, entries[-1][1])], len(plain)),
        "isize": head[:-4] + struct.pack("<I", len(data) + 1) + member,
        "truncated-varint": head + member[:16] + b"\x80" + member[17:],
        "leading-zero": b"\0" + head + ST.gzip_member(entries, len(plain) + 1),
    }
    for name, raw in near.items():
        assert spans(raw)[1] is None, name
    # a table member with a broken varint is still an empty gzip member: the file reads as before
    assert gzip.decompress(near["truncated-varint"]) == data


def test_patch_variable(monkeypatch):
    from lambdipy_b200 import patch
    monkeypatch.delenv("LAMBDIPY_SEEK_TABLE", raising=False)
    assert patch.seek_table() is False
    monkeypatch.setenv("LAMBDIPY_SEEK_TABLE", "1")
    assert patch.seek_table() is True
    for bad in ("0", "yes", ""):
        monkeypatch.setenv("LAMBDIPY_SEEK_TABLE", bad)
        with pytest.raises(ValueError, match="LAMBDIPY_SEEK_TABLE"):
            patch.seek_table()


class _PackageBuild:
    def __init__(self, build_dir):
        self._b = build_dir

    def git_tag(self):
        return "pkg-1.0-2"

    def build_directory(self):
        return self._b


def test_mirror_passes_the_seek_table(tmp_path, monkeypatch):
    (tmp_path / "build" / "pkg").mkdir(parents=True)
    monkeypatch.setenv("HOME", str(tmp_path))
    calls = []
    monkeypatch.setattr(T, "gzip_tarball", lambda srcs, path, ctx=None, **kw: calls.append(kw) or path)
    pb = _PackageBuild(str(tmp_path / "build"))
    T.tarball_method(None, seek_table=True)(pb)
    T.tarball_method(9, seek_table=True)(pb)
    T.tarball_method(None)(pb)
    assert calls == [{"compresslevel": None, "seek_table": True}, {"compresslevel": 9, "seek_table": True}, {}]


def test_cli_flag(monkeypatch, capsys):
    seen = []

    def fake(src, dst, compresslevel=None, seek_table=False):
        seen.append((src, dst, compresslevel, seek_table))
        return {"src_bytes": 3e6, "dst_bytes": 2e6, "gpu": 3, "fallback": 1, "in_bytes": 5e6, "out_bytes": 1e6}
    monkeypatch.setattr(T, "strip_tarball", fake)
    assert T.main(["strip", "a.tar.gz", "b.tar.gz", "--seek-table"]) == 0
    assert T.main(["strip", "a.tar.gz", "b.tar.gz", "--level", "9", "--seek-table"]) == 0
    assert T.main(["strip", "a.tar.gz", "b.tar.gz"]) == 0
    assert seen == [("a.tar.gz", "b.tar.gz", None, True), ("a.tar.gz", "b.tar.gz", 9, True),
                    ("a.tar.gz", "b.tar.gz", None, False)]


def _zip_bytes(tmp_path, name, data, body, chunks):
    import time
    from lambdipy_b200 import zipfile_gpu as Z
    import zipfile
    zi = zipfile.ZipInfo("pkg/a.txt", time.localtime(1e9)[:6])
    zi.file_size = len(data)
    small = zipfile.ZipInfo("pkg/b.txt", time.localtime(1e9)[:6])
    small.file_size = 5
    sbody = zlib.compressobj(6, zlib.DEFLATED, -15)
    sbody = sbody.compress(b"hello") + sbody.flush()
    path = tmp_path / name
    with open(path, "w+b") as fp:
        w = Z._ContainerWriter(fp, [(None, zi), (None, small)])
        w.part(0, body, zlib.crc32(data), True, len(data), chunks)
        w.part(1, sbody, zlib.crc32(b"hello"), True, 5, [(len(sbody), 5)] if chunks else None)
        w.finish()
    return path.read_bytes()


def test_zip_table_lives_in_the_central_directory(tmp_path):
    import zipfile
    from lambdipy_b200 import zipfile_gpu as Z
    data = SS.IS.text(400000)
    body, chunks = SS.flushed(data, SS.every(len(data), ST.CHUNK))
    plain = _zip_bytes(tmp_path, "plain.zip", data, body, None)
    indexed = _zip_bytes(tmp_path, "indexed.zip", data, body, chunks)
    with zipfile.ZipFile(tmp_path / "plain.zip") as zf:
        cd = zf.start_dir
    assert indexed[:cd] == plain[:cd] and len(indexed) > len(plain)
    with zipfile.ZipFile(tmp_path / "indexed.zip") as zf:
        assert zf.testzip() is None and zf.read("pkg/a.txt") == data
        a, b = zf.getinfo("pkg/a.txt"), zf.getinfo("pkg/b.txt")
        assert Z._seek_entries(a) == ST.build(chunks) and Z._seek_entries(b) is None
        zf.extractall(tmp_path / "x")
    assert (tmp_path / "x" / "pkg" / "a.txt").read_bytes() == data
    # a kept member does not carry its table into the local header
    assert ST.zip_field_of(Z._kept(a).extra) == b"" and ST.zip_field_of(a.extra) != b""
    # near-misses of the field read as no table
    assert ST.zip_entries(struct.pack("<HH", ST.ZIP_ID, 3) + b"\x01\x80") is None
    assert ST.zip_entries(b"") is None


def test_zip_hook_and_cli_pass_the_seek_table(monkeypatch, tmp_path, capsys):
    from lambdipy_b200 import patch
    from lambdipy_b200 import zipfile_gpu as Z
    calls = []
    monkeypatch.setattr(Z, "zip_tree", lambda root, path, ctx=None, **kw: calls.append(kw))
    monkeypatch.setattr("lambdipy_b200.project_build.tree_bytes", lambda d: 0)
    (tmp_path / "b.zip").write_bytes(b"")
    for seek in (False, True):
        patch.zip_after_copy(lambda p, d: None, str(tmp_path / "b.zip"), seek=seek)([], str(tmp_path))
    assert calls == [{}, {"seek_table": True}]
    seen = []

    def fake(src, dst, compresslevel=None, **kw):
        seen.append(kw)
        import zipfile
        with zipfile.ZipFile(dst, "w"):
            pass
        return {"zip_bytes": 1, "gpu": 0, "fallback": 0, "in_bytes": 0, "out_bytes": 0}
    monkeypatch.setattr(Z, "strip_zip", fake)
    Z.main(["strip", "a.zip", str(tmp_path / "o.zip"), "--seek-table"])
    Z.main(["strip", "a.zip", str(tmp_path / "o.zip")])
    assert seen == [{"seek_table": True}, {}]
