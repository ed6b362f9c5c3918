"""CPU checks of zip_tarballs' merge, selection and container logic (lambdipy_b200.layer.zip_with) with stand-ins for
the engines: zlib for the reader and the encoder, a Python index and a fake `strip`, over a fake device memory.

The oracle is the contract run literally: `extractall(tree / prefix, filter="fully_trusted")` of each source in turn,
the fake strip on every `*.so` that `find` lists (each inode once, its mtime kept as `strip -p` keeps it), then
`tree_entries` with os.walk listing every directory sorted and ZipInfo.from_file clamping timestamps.  Names, order,
types, external_attr, date_time, sizes, CRC and bytes must match.  The documented deviations (directories without a
member, directories a later source adds to) are applied to the oracle's tree and asserted on their own."""
import gzip
import io
import os
import stat
import tarfile
import time
import zipfile

import pytest

from lambdipy_b200 import layer as L
from lambdipy_b200 import zipfile_gpu as Z
from test_strip_tarball_host import PyIndex, ZlibReader, gz
from test_strip_zip_host import MARK, DeviceZlibEncoder, FakeMemory, FakeStripper, elf, fake_strip

T0 = 1_700_000_000
EPOCH_1980 = time.mktime((1980, 1, 1, 0, 0, 0, 0, 0, -1))


class ArenaReader(ZlibReader):
    """every source's tar stream in one fake device block, each at a 256-byte-aligned offset, as read_many lays
    them out"""

    def read_many(self, paths):
        buf, spans = bytearray(), []
        for p in paths:
            raw = open(p, "rb").read()
            tar = gzip.decompress(raw)
            self.uploaded += len(raw)
            buf += bytes(-len(buf) % 256)
            spans.append((len(buf), len(tar)))
            buf += tar
        base = self.mem.put(buf)
        return [(base + o, n) for o, n in spans]


def tarb(files, fmt=tarfile.GNU_FORMAT):
    """files: [(name, bytes | ("sym", target) | ("lnk", target) | ("dir",) | ("fifo",), mode, mtime)]; mode and
    mtime may be left out"""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=fmt) as tar:
        for name, what, *rest in files:
            ti = tarfile.TarInfo(name)
            ti.mode, ti.mtime = (rest + [0o644, T0])[:2] if rest else (0o644, T0)
            if isinstance(what, bytes):
                ti.size = len(what)
                tar.addfile(ti, io.BytesIO(what))
                continue
            ti.type = {"sym": tarfile.SYMTYPE, "lnk": tarfile.LNKTYPE, "dir": tarfile.DIRTYPE,
                       "fifo": tarfile.FIFOTYPE}[what[0]]
            if what[0] in ("sym", "lnk"):
                ti.linkname = what[1]
            tar.addfile(ti)
    return buf.getvalue()


def run(srcs, dst, piece_bytes=1 << 20, empty_index=False, **kw):
    mem = FakeMemory()
    enc = DeviceZlibEncoder(mem, piece_bytes)
    st = L.zip_with(srcs, str(dst), ArenaReader(mem), PyIndex(mem, empty_index), FakeStripper(mem), enc, **kw)
    return st, enc


def open_dirs(root):
    """Give the owner search and read permission on every directory under root, so that walking and stripping the
    tree does not depend on who runs them (a directory member may carry mode 0o644: the file under it is extracted,
    since tarfile applies a directory's mode after its source's files, but an ordinary user could not stat it).
    Returns {directory: its mode before}, which sorted_entries reports."""
    modes = {}
    for d, dirs, _ in os.walk(root):
        for name in dirs:
            p = os.path.join(d, name)
            if not os.path.islink(p):
                mode = modes[os.path.realpath(p)] = stat.S_IMODE(os.stat(p).st_mode)
                os.chmod(p, mode | 0o700)
    return modes


def sorted_entries(root, monkeypatch, modes=None):
    """tree_entries(root) with os.walk listing every directory sorted and from_file clamping timestamps; modes
    {directory: mode} (open_dirs) are the modes the directory entries report"""
    real_walk, real_from_file = os.walk, zipfile.ZipInfo.from_file

    def walk(top, *a, **k):
        for d, dirs, files in real_walk(top, *a, **k):
            dirs.sort()
            files.sort()
            yield d, dirs, files
    with monkeypatch.context() as m:
        m.setattr(os, "walk", walk)
        m.setattr(zipfile.ZipInfo, "from_file",
                  classmethod(lambda cls, f, a=None, **k: real_from_file.__func__(cls, f, a, strict_timestamps=False)))
        entries = Z.tree_entries(root)
    for path, zi in entries:
        if zi.is_dir() and os.path.realpath(path) in (modes or {}):
            zi.external_attr = (stat.S_IFDIR | modes[os.path.realpath(path)]) << 16 | 0x10
    return entries


def oracle(tars, tmp_path, prefix="", monkeypatch=None):
    """the literal passes, with the documented deviations applied: (entries, {dir: "implicit" | "member"})"""
    root = str(tmp_path / "tree")
    os.makedirs(root)
    dir_mtime = {}
    for tar in tars:
        with tarfile.open(fileobj=io.BytesIO(tar)) as t:
            t.extractall(os.path.join(root, prefix), filter="fully_trusted")
            for m in t.getmembers():
                if m.isdir():
                    dir_mtime[os.path.normpath(os.path.join(root, prefix, m.name))] = m.mtime
    modes = open_dirs(root)
    done = set()
    for d, dirs, files in os.walk(root):
        for name in dirs + files:
            p = os.path.join(d, name)
            if not name.endswith(".so") or not os.path.isfile(p) or os.stat(p).st_ino in done:
                continue
            done.add(os.stat(p).st_ino)
            st = os.stat(p)
            new = fake_strip(open(p, "rb").read())
            if new is None:                                                 # tolerate_non_elf keeps it
                continue
            with open(p, "r+b") as f:
                f.write(new)
                f.truncate()
            os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns))          # strip -p
    kinds = {}
    for d, dirs, _ in os.walk(root, topdown=False):
        for name in dirs:
            p = os.path.join(d, name)
            if os.path.islink(p):
                continue
            rel = os.path.relpath(p, root)
            if os.path.normpath(p) in dir_mtime:
                kinds[rel] = "member"
                os.utime(p, (dir_mtime[os.path.normpath(p)],) * 2)
            else:
                kinds[rel] = "implicit"
                os.utime(p, (EPOCH_1980, EPOCH_1980))
    return sorted_entries(root, monkeypatch, modes), kinds


def compare(dst, want):
    with zipfile.ZipFile(dst) as zf:
        assert zf.testzip() is None
        got = zf.infolist()
        assert [z.filename for z in got] == [zi.filename for _, zi in want]
        for z, (path, w) in zip(got, want):
            for attr in ("external_attr", "file_size", "create_system", "flag_bits"):
                assert getattr(z, attr) == getattr(w, attr), (z.filename, attr)
            assert z.date_time == w.date_time[:5] + (w.date_time[5] // 2 * 2,), z.filename   # DOS time: 2 s steps
            if w.is_dir():
                assert z.compress_type == zipfile.ZIP_STORED
            else:
                data = open(path, "rb").read()
                assert z.compress_type == zipfile.ZIP_DEFLATED and zf.read(z) == data
                assert z.CRC == zipfile.crc32(data)


def case(tmp_path, monkeypatch, tars, prefix="", members=1, **kw):
    srcs = [gz(tmp_path / ("s%d.tar.gz" % i), t, members) for i, t in enumerate(tars)]
    dst = tmp_path / "out" / "layer.zip"
    st, enc = run(srcs, dst, prefix=prefix, **kw)
    want, kinds = oracle(tars, tmp_path, prefix, monkeypatch)
    compare(str(dst), want)
    assert os.listdir(tmp_path / "out") == ["layer.zip"]
    assert st["entries"] == len(want) and st["zip_bytes"] == os.path.getsize(dst)
    return st, dst, kinds


def package(tag=b""):
    return [("pkg/", ("dir",), 0o755, T0 - 50), ("pkg/__init__.py", b"import this\n" * 40 + tag, 0o644, T0 + 1),
            ("pkg/core.so", elf(b"core " * 300 + tag), 0o755, T0 + 2), ("pkg/bin/", ("dir",), 0o700, T0 - 10),
            ("pkg/bin/tool", b"#!/bin/sh\n" + tag, 0o4755, T0 + 3), ("pkg/empty.txt", b"", 0o600, T0 + 4),
            ("pkg/libz.so.1", elf(b"versioned"), 0o755, T0 + 5)]


@pytest.mark.parametrize("fmt", ["gnu", "pax", "ustar", "v7"])
def test_formats(tmp_path, monkeypatch, fmt):
    if fmt == "v7":
        import tar_archives as A
        tar = A.crafted()["v7_aregtype"]
    else:
        long = "pkg/" + "/".join("segment%02d" % i for i in range(12)) + ".so"      # a GNU longname, pax path, ustar prefix
        tar = tarb(package() + [(long, elf(b"long name"))],
                   {"gnu": tarfile.GNU_FORMAT, "pax": tarfile.PAX_FORMAT, "ustar": tarfile.USTAR_FORMAT}[fmt])
    st, dst, _ = case(tmp_path, monkeypatch, [tar], tolerate_non_elf=True)
    assert st["sources"] == 1 and st["skipped_entries"] == 0
    if fmt == "v7":   # a directory without search permission lists its file, whoever runs the call
        with zipfile.ZipFile(dst) as zf:
            assert zf.namelist() == ["v7dir/", "v7dir/f.so"] and zf.getinfo("v7dir/").external_attr >> 16 == 0o40644


def test_pax_size_record(tmp_path, monkeypatch):
    import tar_archives as A
    tar = A.crafted()["pax_size_record"]
    tar = tar.replace(b"\x7fELF" + b"p" * 3000, b"\x7fELF" + b"p" * 1000 + MARK + b"p" * (2000 - len(MARK)))
    st, _, _ = case(tmp_path, monkeypatch, [tar])
    assert (st["gpu"], st["out_bytes"]) == (1, 1004)


def test_links(tmp_path, monkeypatch):
    files = [("pkg/", ("dir",), 0o755, T0), ("pkg/libx.so.1", elf(b"x" * 500), 0o755, T0 + 1),
             ("pkg/libx.so", ("sym", "libx.so.1")), ("pkg/again.so", ("sym", "./libx.so")),      # a chain
             ("pkg/hard.so", ("lnk", "pkg/libx.so.1"), 0o700, T0 + 9),                           # mode, mtime win
             ("pkg/dangling.so", ("sym", "nowhere.so")), ("pkg/out.so", ("sym", "../../../nonexistent/x.so")),
             ("pkg/sub/", ("dir",), 0o750, T0 + 3), ("pkg/sub/up.so", ("sym", "../libx.so.1")),
             ("pkg/libdir", ("sym", "sub")), ("pkg/via.so", ("sym", "libdir/up.so")),
             ("pkg/loop", ("sym", "loop")), ("pkg/pipe", ("fifo",)), ("pkg/dir.so", ("dir",)),
             ("pkg/text.txt", b"plain text " * 99)]
    st, dst, _ = case(tmp_path, monkeypatch, [tarb(files)])
    assert (st["selected"], st["gpu"]) == (1, 1)                         # libx.so.1, through every name
    assert st["skipped"] == 3                                             # dangling, out, dir.so
    assert st["skipped_entries"] == 4                                     # dangling, out, loop, pipe
    with zipfile.ZipFile(dst) as zf:
        names = zf.namelist()
        assert "pkg/libdir/" in names and "pkg/libdir/up.so" not in names   # not descended into
        stripped = fake_strip(elf(b"x" * 500))
        assert all(zf.read(n) == stripped for n in ("pkg/libx.so", "pkg/again.so", "pkg/hard.so", "pkg/via.so"))
        assert zf.getinfo("pkg/libx.so.1").external_attr >> 16 == 0o100700


def test_sparse_member_raises(tmp_path):
    import tar_archives as A
    raw = bytearray(tarb([("a.so", elf(b"a")), ("b.txt", b"b")]))
    h = bytearray(raw[:512])
    h[156:157] = tarfile.GNUTYPE_SPARSE
    h[483:495] = tarfile.itn(len(elf(b"a")), 12, tarfile.GNU_FORMAT)
    raw[:512] = A.seal(h)
    src = gz(tmp_path / "s.tar.gz", bytes(raw))
    with pytest.raises(ValueError, match="sparse"):
        run([src], tmp_path / "o.zip")
    assert sorted(os.listdir(tmp_path)) == ["s.tar.gz"]


@pytest.mark.parametrize("prefix", ["", "python/", "opt/python/"])
def test_implicit_directories_and_prefix(tmp_path, monkeypatch, prefix):
    tar = tarb([("a/b/c.so", elf(b"deep")), ("a/b/d.txt", b"d" * 70_000), ("./", ("dir",), 0o751, T0 + 7),
                ("top.py", b"print()\n")])
    st, dst, kinds = case(tmp_path, monkeypatch, [tar], prefix=prefix)
    umask = Z._umask()
    with zipfile.ZipFile(dst) as zf:
        for rel, kind in kinds.items():
            zi = zf.getinfo(rel + "/")
            if kind == "implicit":                                          # the documented deviation
                assert zi.date_time == (1980, 1, 1, 0, 0, 0) and zi.external_attr >> 16 == 0o40777 & ~umask
        if prefix:
            assert zf.namelist()[0] == prefix.split("/")[0] + "/"
            assert zf.getinfo(prefix).external_attr >> 16 == 0o40751        # the "./" member is the prefix
    assert set(kinds.values()) == {"implicit"} | ({"member"} if prefix else set())


def test_mtime_zero_and_far_future_are_clamped(tmp_path, monkeypatch):
    tar = tarb([("old/", ("dir",), 0o755, 0), ("old/a.so", elf(b"a"), 0o755, 0), ("old/b.txt", b"b", 0o644, 0),
                ("new.txt", b"n", 0o644, 4_500_000_000)])
    _, dst, _ = case(tmp_path, monkeypatch, [tar])
    with zipfile.ZipFile(dst) as zf:
        assert zf.getinfo("old/a.so").date_time == (1980, 1, 1, 0, 0, 0)
        assert zf.getinfo("new.txt").date_time == (2107, 12, 31, 23, 59, 58)     # 59 s in DOS time's 2 s steps


def test_two_and_three_sources_with_overrides(tmp_path, monkeypatch):
    a = tarb(package(b"A") + [("pkg/only_a.so", elf(b"only a"))])
    b = tarb([("pkg/", ("dir",), 0o711, T0 + 100), ("pkg/core.so", elf(b"core from b " * 50), 0o700, T0 + 101),
              ("pkg/__init__.py", b"# b\n", 0o600, T0 + 102), ("other/x.so", elf(b"x")),
              ("pkg/new/", ("dir",))], tarfile.PAX_FORMAT)
    c = tarb([("pkg/bin/", ("dir",), 0o755, T0 + 200), ("pkg/bin/more.so", elf(b"more")),
              ("other/x.so", elf(b"x again " * 9)), ("pkg/link.so", ("sym", "core.so"))])
    st, dst, _ = case(tmp_path, monkeypatch, [a, b])
    assert (st["sources"], st["selected"]) == (2, 3)
    (tmp_path / "three").mkdir()
    st, dst, _ = case(tmp_path / "three", monkeypatch, [a, b, c], members=2)
    assert st["selected"] == 4 and st["members"] == sum(len(tarfile.open(fileobj=io.BytesIO(t)).getmembers())
                                                         for t in (a, b, c))
    with zipfile.ZipFile(dst) as zf:
        assert zf.read("pkg/link.so") == zf.read("pkg/core.so") == fake_strip(elf(b"core from b " * 50))
        assert zf.getinfo("pkg/bin/").date_time == time.localtime(T0 + 200)[:6]
        assert zf.getinfo("pkg/").date_time == time.localtime(T0 + 100)[:6]  # a later source adds to it: kept


@pytest.mark.parametrize("first,second", [
    (("x", b"file"), ("x", ("dir",))), (("x", ("dir",)), ("x", b"file")),
    (("x", ("sym", "y")), ("x", b"file")), (("x", b"file"), ("x", ("sym", "y"))),
    (("x", b"file"), ("x", ("lnk", "y"))), (("d/f", b"f"), ("d", b"file onto an implicit directory")),
    (("x", b"file"), ("x/y", b"below a file")), (("l", ("sym", "d")), ("l/f", b"below a symlink")),
    (("x", ("fifo",)), ("x", b"file"))])
@pytest.mark.parametrize("same_source", [False, True])
def test_refused_collisions(tmp_path, first, second, same_source):
    base = [("y", b"y"), ("d/", ("dir",))]
    tars = [tarb(base + [first, second])] if same_source else [tarb(base + [first]), tarb([second])]
    srcs = [gz(tmp_path / ("s%d.tar.gz" % i), t) for i, t in enumerate(tars)]
    with pytest.raises(ValueError):
        run(srcs, tmp_path / "o.zip")
    assert sorted(os.listdir(tmp_path)) == sorted(os.path.basename(s) for s in srcs)


def test_replacing_a_file_a_hard_link_shares_is_refused(tmp_path):
    a = tarb([("f.so", elf(b"f")), ("h.so", ("lnk", "f.so"))])
    for tars in ([a, tarb([("f.so", elf(b"new"))])], [a, tarb([("h.so", elf(b"new"))])]):
        srcs = [gz(tmp_path / ("s%d.tar.gz" % i), t) for i, t in enumerate(tars)]
        with pytest.raises(ValueError, match="hard link shares"):
            run(srcs, tmp_path / "o.zip")
    assert not os.path.exists(tmp_path / "o.zip")


def test_duplicate_within_a_source_and_empty_source(tmp_path, monkeypatch):
    a = tarb([("p/dup.so", elf(b"first " * 10), 0o700, T0), ("p/dup.so", elf(b"second"), 0o755, T0 + 5),
              ("p/dir/", ("dir",), 0o700, T0), ("p/dir/", ("dir",), 0o755, T0 + 6)])
    st, dst, _ = case(tmp_path, monkeypatch, [tarb([]), a, tarb([])])
    assert st["selected"] == 1                                   # the shadowed member is not stripped
    with zipfile.ZipFile(dst) as zf:
        assert zf.read("p/dup.so") == fake_strip(elf(b"second"))


def test_more_than_65535_entries(tmp_path):
    tar = tarb([("m/%05d" % i, b"") for i in range(65_600)] + [("m/last.so", elf(b"the only object"))])
    st, _ = run([gz(tmp_path / "s.tar.gz", tar)], tmp_path / "o.zip")
    assert st["entries"] == 65_602 and st["gpu"] == 1
    assert zipfile.stringEndArchive64 in (tmp_path / "o.zip").read_bytes()[-200:]
    with zipfile.ZipFile(tmp_path / "o.zip") as zf:
        names = zf.namelist()
        assert names[:2] == ["m/", "m/00000"] and names[-1] == "m/last.so" and len(names) == 65_602
        assert zf.read("m/last.so") == fake_strip(elf(b"the only object"))


@pytest.mark.parametrize("members", [1, 3])
def test_pieces_bus_bytes_and_the_index(tmp_path, monkeypatch, members):
    files = [("p/%d.so" % i, elf(b"%d" % i * (i * 997 % 50_000))) for i in range(30)] + [("p/big", os.urandom(300_000))]
    tars = [tarb(files[:15], tarfile.PAX_FORMAT), tarb(files[15:])]
    st, dst, _ = case(tmp_path, monkeypatch, tars, members=members, piece_bytes=96 << 10)
    assert st["index"]["misses"] == 0 and st["gpu"] == 30
    assert st["uploaded_bytes"] == st["src_bytes"]
    with zipfile.ZipFile(dst) as zf:
        assert st["deflated_bytes"] == sum(z.compress_size for z in zf.infolist())
        assert st["file_bytes"] == sum(z.file_size for z in zf.infolist())
    assert st["downloaded_bytes"] == 16 * st["index"]["ranges"] + st["index"]["bytes"] + st["deflated_bytes"]
    srcs = [str(tmp_path / ("s%d.tar.gz" % i)) for i in range(2)]
    st2, _ = run(srcs, tmp_path / "again.zip", empty_index=True, piece_bytes=96 << 10)
    assert st2["index"]["misses"] > 0 and (tmp_path / "again.zip").read_bytes() == dst.read_bytes()


def test_failures_leave_nothing(tmp_path):
    src = gz(tmp_path / "s.tar.gz", tarb([("a.so", elf(b"a")), ("t.so", b"not an elf\n" * 10),
                                         ("r.so", elf(b"r", refused=True))]))
    with pytest.raises(Z.StripFailed, match="t.so"):
        run([src], tmp_path / "o.zip")
    st, _ = run([src], tmp_path / "o.zip", tolerate_non_elf=True)
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    assert st["uploaded_bytes"] == os.path.getsize(src) + len(fake_strip(elf(b"r", refused=True)))
    with zipfile.ZipFile(tmp_path / "o.zip") as zf:
        assert zf.read("t.so") == b"not an elf\n" * 10 and zf.read("r.so") == fake_strip(elf(b"r", refused=True))
    os.unlink(tmp_path / "o.zip")
    with pytest.raises(Z.StripFailed, match="r.so"):
        run([src], tmp_path / "o.zip", tolerate_non_elf=True, fallback_host_strip=False)
    raw = open(src, "rb").read()
    (tmp_path / "bad.tar.gz").write_bytes(raw[:len(raw) // 2])
    with pytest.raises((EOFError, gzip.BadGzipFile)):
        run([src, str(tmp_path / "bad.tar.gz")], tmp_path / "o.zip")
    gz(tmp_path / "junk.tar.gz", b"this is not a tar stream" * 100)
    with pytest.raises(tarfile.ReadError):
        run([str(tmp_path / "junk.tar.gz")], tmp_path / "o.zip")
    assert sorted(os.listdir(tmp_path)) == ["bad.tar.gz", "junk.tar.gz", "s.tar.gz"]
    for dst in (src, str(tmp_path / "." / "s.tar.gz")):
        with pytest.raises(ValueError, match="source being read"):
            run([str(tmp_path / "junk.tar.gz"), src], dst)
    for prefix in ("python", "/python/", "a/../b/", "a//", "./"):
        with pytest.raises(ValueError, match="prefix"):
            run([src], tmp_path / "o.zip", prefix=prefix)
    assert open(src, "rb").read() == raw and sorted(os.listdir(tmp_path)) == ["bad.tar.gz", "junk.tar.gz", "s.tar.gz"]


def test_member_leaving_the_tree_is_refused(tmp_path):
    for name in ("../evil.so", "/abs/evil.so"):
        src = gz(tmp_path / "s.tar.gz", tarb([(name, elf(b"e"))]))
        with pytest.raises(ValueError, match="leaves"):
            run([src], tmp_path / "o.zip")


def test_cli_and_export(monkeypatch, capsys):
    seen = {}

    def fake(srcs, dst, prefix="", compresslevel=None, seek_table=False):
        seen.update(srcs=srcs, dst=dst, prefix=prefix, level=compresslevel, seek=seek_table)
        return {"zip_bytes": 4e6, "src_bytes": 5e6, "entries": 12, "gpu": 3, "fallback": 1, "in_bytes": 5e6,
                "out_bytes": 1e6}
    monkeypatch.setattr(L, "zip_tarballs", fake)
    assert L.main(["l.zip", "a.tar.gz", "b.tar.gz", "--prefix", "python/", "--level", "9", "--seek-table"]) == 0
    assert seen == {"srcs": ["a.tar.gz", "b.tar.gz"], "dst": "l.zip", "prefix": "python/", "level": 9, "seek": True}
    out = capsys.readouterr().out.strip().splitlines()
    assert len(out) == 1 and "l.zip" in out[0] and "4 shared objects stripped (1 via host strip)" in out[0]
    for bad in (["l.zip"], ["l.zip", "a.tar.gz", "--level", "6"], []):
        with pytest.raises(SystemExit):
            L.main(bad)
    import lambdipy_b200
    assert lambdipy_b200.zip_tarballs is fake
