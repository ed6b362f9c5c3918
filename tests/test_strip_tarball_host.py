"""CPU checks of strip_tarball's tar logic (lambdipy_b200.tarball.strip_with) with stand-ins for the four engines:
zlib for the reader and the writer, a Python index (the ranges tarfile itself reads) and a fake `strip` that cuts a
file at a marker, all over a fake device memory in which a reference used after its buffer is gone fails the test.

* header rewriting: the size field and checksum of a stripped member, and a pax `size` record with its header;
* the end-of-archive blocks and record padding; a source with nothing to strip keeps its tar stream;
* the link, hard-link, duplicate-name, directory and sparse rules against `extractall(filter="fully_trusted")` and
  the fake strip run as the reference's `find -name "*.so" | xargs strip` runs;
* multi-member sources, an index that returns nothing (every read a counted miss, the same output);
* StripFailed / tolerate_non_elf, no file left behind on any failure, dst == src, and the new entry points."""
import gzip
import io
import os
import re
import tarfile
import zlib

import pytest

import tar_archives as A
from lambdipy_b200 import _native as N
from lambdipy_b200 import tarball as T
from lambdipy_b200 import zipfile_gpu as Z
from test_strip_zip_host import MARK, FakeMemory, FakeStripper, elf, fake_strip


class ZlibReader:
    def __init__(self, mem):
        self.mem, self.uploaded, self.downloaded = mem, 0, 0

    def read(self, path):
        raw = open(path, "rb").read()
        tar = gzip.decompress(raw)
        self.uploaded += len(raw)
        return (self.mem.put(tar), len(tar)), int.from_bytes(raw[4:8], "little")

    def fetch(self, addr, n):
        self.downloaded += n
        return self.mem.get((addr, n))

    def upload(self, data):
        self.uploaded += len(data)
        return self.mem.put(data)

    def zeros(self, n):
        return self.mem.put(bytes(n))

    def stats(self):
        return {"kernel_ms": 0.0}


class PyIndex:
    """the ranges tarfile reads to list the members, found by letting it read them; empty=True returns none"""

    def __init__(self, mem, empty=False):
        self.mem, self.empty = mem, empty

    def index(self, ref):
        addr, n = ref
        tar = self.mem.get(ref)
        if self.empty:
            return [], b"", {"kernel_ms": 0.0}
        from test_tar_walk_emulated import tarfile_listing
        reads, _, _ = tarfile_listing(tar)
        ranges = []
        for pos, k in sorted(reads):
            if ranges and pos <= ranges[-1][0] + ranges[-1][1]:
                ranges[-1] = (ranges[-1][0], max(ranges[-1][1], pos + k - ranges[-1][0]))
            else:
                ranges.append((pos, k))
        return ranges, b"".join(tar[o:o + k] for o, k in ranges), {"kernel_ms": 0.0}


class ZlibWriter:
    """GpuGzipFile's device-fed side with zlib underneath; records the pieces it was given"""

    def __init__(self, mem, fileobj, name, mtime):
        self.mem, self.pieces, self.stats = mem, [], None
        self.gz = gzip.GzipFile(filename=os.path.basename(name)[:-3], fileobj=fileobj, mode="wb", mtime=mtime)

    def submit_device(self, refs):
        data = b"".join(self.mem.get(r) for r in refs)
        self.pieces.append(len(data))
        self.gz.write(data)

    def close(self):
        self.gz.close()
        self.stats = {"out_bytes": 2}


def run(src, dst, empty_index=False, piece_bytes=1 << 16, **kw):
    mem = FakeMemory()
    writers = []

    def open_writer(fileobj, name, mtime):
        writers.append(ZlibWriter(mem, fileobj, name, mtime))
        return writers[-1]
    st = T.strip_with(str(src), str(dst), ZlibReader(mem), PyIndex(mem, empty_index), FakeStripper(mem), open_writer,
                      piece_bytes, **kw)
    return st, writers[0].pieces


def gz(path, tar, members=1):
    with open(path, "wb") as f:
        cut = [len(tar) * k // members for k in range(members + 1)]
        for a, b in zip(cut, cut[1:]):
            f.write(gzip.compress(tar[a:b], mtime=1234567))
    return str(path)


def tar_of(files, fmt=tarfile.GNU_FORMAT, **kw):
    """files: [(name, bytes | ("sym", target) | ("lnk", target) | ("dir",))] in order"""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=fmt, **kw) as tar:
        for name, what in files:
            ti = tarfile.TarInfo(name)
            ti.mtime, ti.mode = 1700000000, 0o755
            if isinstance(what, bytes):
                ti.size = len(what)
                tar.addfile(ti, io.BytesIO(what))
            else:
                ti.type = {"sym": tarfile.SYMTYPE, "lnk": tarfile.LNKTYPE, "dir": tarfile.DIRTYPE}[what[0]]
                if what[0] != "dir":
                    ti.linkname = what[1]
                tar.addfile(ti)
    return buf.getvalue()


def reference(tar, root):
    """extractall, then the fake strip over `find -name "*.so"` (symlinks followed by strip, each inode once)"""
    with tarfile.open(fileobj=io.BytesIO(tar)) as t:
        t.extractall(root, filter="fully_trusted")
    done = set()
    for d, dirs, files in os.walk(root):
        for name in dirs + files:
            p = os.path.join(d, name)
            if not name.endswith(".so") or not os.path.isfile(p):
                continue
            st = os.stat(p)
            if (st.st_dev, st.st_ino) in done:
                continue
            done.add((st.st_dev, st.st_ino))
            with open(p, "r+b") as f:
                new = fake_strip(f.read())
                assert new is not None, p
                f.seek(0)
                f.write(new)
                f.truncate()
    return root


def snapshot(root):
    out = {}
    for d, dirs, files in os.walk(root):
        for name in dirs + files:
            p = os.path.join(d, name)
            rel = os.path.relpath(p, root)
            if os.path.islink(p):
                out[rel] = ("sym", os.readlink(p))
            elif os.path.isdir(p):
                out[rel] = ("dir",)
            else:
                out[rel] = open(p, "rb").read()
    return out


def check_tree(tar_src, dst, tmp_path):
    want = snapshot(reference(tar_src, str(tmp_path / "want")))
    with tarfile.open(dst) as t:
        t.extractall(str(tmp_path / "got"), filter="fully_trusted")
    assert snapshot(str(tmp_path / "got")) == want


def members_equal_but_sizes(a, b, stripped):
    ma, mb = tarfile.open(fileobj=io.BytesIO(a)).getmembers(), tarfile.open(fileobj=io.BytesIO(b)).getmembers()
    assert len(ma) == len(mb)
    for x, y in zip(ma, mb):
        fx, fy = x.get_info(), y.get_info()
        if x.name in stripped:
            for k in ("size", "chksum"):
                fx.pop(k), fy.pop(k)
        assert fx == fy, x.name


def test_links_duplicates_and_rules(tmp_path):
    files = [("pkg/", ("dir",)), ("pkg/libx.so.1", elf(b"x")), ("pkg/libx.so", ("sym", "libx.so.1")),
             ("pkg/again.so", ("sym", "./libx.so")),                       # a link to a link: stripped once
             ("pkg/hard.so", ("lnk", "pkg/libx.so.1")), ("pkg/plain.so", elf(b"plain")),
             ("pkg/dup.so", elf(b"first")), ("pkg/dup.so", elf(b"second")),
             ("pkg/dangling.so", ("sym", "nowhere.so")), ("pkg/out.so", ("sym", "../../etc/x.so")),
             ("pkg/dir.so", ("dir",)), ("pkg/dir.so/inner.so", elf(b"inner")), ("pkg/readme.txt", b"text\n" * 100),
             ("pkg/sub/", ("dir",)), ("pkg/sub/up.so", ("sym", "../libx.so.1")),
             ("pkg/libdir", ("sym", "sub")), ("pkg/via.so", ("sym", "libdir/up.so"))]
    tar = tar_of(files)
    src = gz(tmp_path / "s.tar.gz", tar)
    dst = tmp_path / "d.tar.gz"
    st, _ = run(src, dst)
    assert st["selected"] == 5 and st["gpu"] == 5          # libx.so.1, plain, dup x2, inner
    assert st["skipped"] == 3                               # dangling, out, dir.so
    check_tree(tar, str(dst), tmp_path)
    new = gzip.decompress(dst.read_bytes())
    members_equal_but_sizes(tar, new, {"pkg/libx.so.1", "pkg/plain.so", "pkg/dup.so", "pkg/dir.so/inner.so"})
    for m in tarfile.open(fileobj=io.BytesIO(new)).getmembers():
        h = new[m.offset:m.offset + 512]
        assert re.fullmatch(rb"[0-7]{11}\0", h[124:136]) and re.fullmatch(rb"[0-7]{6}\0 ", h[148:156])
    assert len(new) % tarfile.RECORDSIZE == 0 and st["tar_bytes_out"] == len(new)


def test_sparse_member_is_left_alone(tmp_path):
    raw = bytearray(tar_of([("a.so", elf(b"a")), ("b.txt", b"b")]))
    h = bytearray(raw[:512])
    h[156:157] = tarfile.GNUTYPE_SPARSE
    h[483:495] = tarfile.itn(len(elf(b"a")), 12, tarfile.GNU_FORMAT)
    raw[:512] = A.seal(h)
    src = gz(tmp_path / "s.tar.gz", bytes(raw))
    st, _ = run(src, tmp_path / "d.tar.gz")
    assert (st["selected"], st["skipped"]) == (0, 1)
    assert gzip.decompress((tmp_path / "d.tar.gz").read_bytes()) == bytes(raw)


def test_pax_size_record_is_rewritten(tmp_path):
    tar = A.crafted()["pax_size_record"]
    tar = tar.replace(b"\x7fELF" + b"p" * 3000, b"\x7fELF" + b"p" * 1000 + MARK + b"p" * (2000 - len(MARK)))
    src = gz(tmp_path / "s.tar.gz", tar)
    st, _ = run(src, tmp_path / "d.tar.gz")
    assert st["gpu"] == 1 and st["out_bytes"] == 1004
    new = gzip.decompress((tmp_path / "d.tar.gz").read_bytes())
    t = tarfile.open(fileobj=io.BytesIO(new))
    m = t.getmember("pax/size_record.so")
    assert m.size == 1004 and m.pax_headers["size"] == "1004" and t.extractfile(m).read() == b"\x7fELF" + b"p" * 1000
    assert b"13 size=1004\n" in new[:1024] and tarfile.nti(new[124:136]) == 13 + len(b"") + \
        sum(len(r) for r, _ in T._pax_records(new[512:1024]) if _ != b"size")
    assert [x.name for x in t.getmembers()] == ["pax/size_record.so", "pax/after.txt"]


def test_pax_record_length_prefix():
    for k, v in ((b"size", b"1"), (b"size", b"12345"), (b"path", b"x" * 90), (b"path", b"y" * 994)):
        rec = T._pax_record(k, v)
        assert int(rec.split(b" ")[0]) == len(rec)
        ti = tarfile.TarInfo()
        want = ti._create_pax_generic_header({k.decode(): v.decode()}, tarfile.XHDTYPE, "utf-8")[512:]
        assert want.rstrip(b"\0") == rec


@pytest.mark.parametrize("fmt", sorted(A.crafted()) + ["tarfile_gnu", "tarfile_pax", "gnu_posix", "gnu_gnu"])
def test_nothing_selected_keeps_the_stream_and_trees_match(tmp_path, fmt):
    if fmt.startswith("tarfile_"):
        tar = A.tarfile_bytes(A.sample_tree(str(tmp_path / "pkg")), tarfile.GNU_FORMAT if fmt == "tarfile_gnu" else tarfile.PAX_FORMAT)
    elif fmt.startswith("gnu_"):
        tar = A.gnu_tar_bytes(A.sample_tree(str(tmp_path / "pkg")), fmt[4:], str(tmp_path))
        if tar is None:
            pytest.skip("GNU tar is not installed")
    else:
        tar = A.crafted()[fmt]
    src = gz(tmp_path / "s.tar.gz", tar)   # the fake strip refuses these payloads: tolerated, nothing changes
    st, _ = run(src, tmp_path / "d.tar.gz", tolerate_non_elf=True)
    new = gzip.decompress((tmp_path / "d.tar.gz").read_bytes())
    if st["gpu"] + st["fallback"] == 0:
        end = tarfile.open(fileobj=io.BytesIO(tar))
        end.getmembers()
        want = tar[:end.offset] + bytes(1024)
        want += bytes(-len(want) % tarfile.RECORDSIZE)
        assert new == want
        if fmt.startswith("tarfile_"):
            assert new == tar                                  # tarfile's own output comes out unchanged


def test_trailing_garbage_is_dropped(tmp_path):
    tar = tar_of([("a.so", elf(b"a")), ("b.txt", b"b" * 700)])
    src = gz(tmp_path / "s.tar.gz", tar + bytes(range(256)) * 50)
    st, _ = run(src, tmp_path / "d.tar.gz")
    new = gzip.decompress((tmp_path / "d.tar.gz").read_bytes())
    assert len(new) == st["tar_bytes_out"] and len(new) % tarfile.RECORDSIZE == 0
    assert new.rstrip(b"\0").endswith(b"b" * 700)


@pytest.mark.parametrize("members", [1, 2, 5])
def test_multi_member_sources_and_empty_index(tmp_path, members):
    files = [("p/%d.so" % i, elf(b"%d" % i * (i * 997 % 5000))) for i in range(40)] + [("p/t.txt", b"t" * 9000)]
    tar = tar_of(files, tarfile.PAX_FORMAT)
    src = gz(tmp_path / "s.tar.gz", tar, members)
    (tmp_path / "b").mkdir()
    a, pieces = run(src, tmp_path / "a.tar.gz", piece_bytes=4096)
    b, _ = run(src, tmp_path / "b" / "a.tar.gz", empty_index=True, piece_bytes=4096)
    assert (tmp_path / "a.tar.gz").read_bytes() == (tmp_path / "b" / "a.tar.gz").read_bytes()
    assert a["index"]["misses"] == 0 and b["index"]["misses"] > 0 and b["downloaded_bytes"] > a["downloaded_bytes"]
    assert a["gpu"] == 40 and all(p == 4096 for p in pieces[:-1]) and 0 < pieces[-1] <= 4096
    check_tree(tar, str(tmp_path / "a.tar.gz"), tmp_path)
    assert gzip.open(tmp_path / "a.tar.gz").read()[:10]   # one readable gzip member, MTIME from the source
    assert int.from_bytes((tmp_path / "a.tar.gz").read_bytes()[4:8], "little") == 1234567


def test_failures_leave_nothing(tmp_path):
    good = tar_of([("a.so", elf(b"a")), ("t.so", b"not an elf at all\n" * 10), ("r.so", elf(b"r", refused=True))])
    src = gz(tmp_path / "s.tar.gz", good)
    with pytest.raises(Z.StripFailed, match="t.so"):
        run(src, tmp_path / "o.tar.gz")
    assert sorted(os.listdir(tmp_path)) == ["s.tar.gz"]
    st, _ = run(src, tmp_path / "o.tar.gz", tolerate_non_elf=True)
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    os.unlink(tmp_path / "o.tar.gz")
    with pytest.raises(Z.StripFailed, match="r.so"):
        run(src, tmp_path / "o.tar.gz", tolerate_non_elf=True, fallback_host_strip=False)
    # framing, data and header errors
    raw = (tmp_path / "s.tar.gz").read_bytes()
    (tmp_path / "bad.tar.gz").write_bytes(raw[:len(raw) // 2])
    with pytest.raises((EOFError, zlib.error, gzip.BadGzipFile)):
        run(tmp_path / "bad.tar.gz", tmp_path / "o.tar.gz")
    gz(tmp_path / "junk.tar.gz", b"this is not a tar stream" * 100)
    with pytest.raises(tarfile.ReadError):
        run(tmp_path / "junk.tar.gz", tmp_path / "o.tar.gz")
    assert sorted(os.listdir(tmp_path)) == ["bad.tar.gz", "junk.tar.gz", "s.tar.gz"]
    with pytest.raises(ValueError):
        run(src, src)


def test_cli_and_entry_points(monkeypatch, tmp_path, capsys):
    seen = {}

    def fake(src, dst, compresslevel=None):
        seen.update(src=src, dst=dst, level=compresslevel)
        return {"src_bytes": 3e6, "dst_bytes": 2e6, "gpu": 3, "fallback": 1, "in_bytes": 5e6, "out_bytes": 1e6}
    monkeypatch.setattr(T, "strip_tarball", fake)
    assert T.main(["strip", "a.tar.gz", "b.tar.gz", "--level", "9"]) == 0
    assert seen == {"src": "a.tar.gz", "dst": "b.tar.gz", "level": 9}
    assert "4 shared objects stripped (1 via host strip)" in capsys.readouterr().out
    import lambdipy_b200
    assert lambdipy_b200.strip_tarball is fake
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "lambdipy_b200.h")).read()
    for sym in ("lb2_inflate_device_output", "lb2_memcpy_d2d", "lb2_gzip_submit_device", "lb2_tar_index"):
        assert sym in N.EXPORTS and sym + "(" in header
