"""CPU checks of strip_zip's container logic (lambdipy_b200.zipfile_gpu.strip_with) with stand-ins for the three
engines: zlib for the decoder and the encoder, and a fake `strip` that cuts a file at a marker.  The stand-ins keep a
fake device memory, so a reference used after the engine that made it has moved on fails the test.

* unselected members keep body bytes and metadata, lose the data-descriptor bit, and have their sizes in the local
  header; order, archive comment, `*.so` directory entries and symlink-mode entries are left alone;
* selected members, stored ones included, come out deflated with the stripped bytes; a member larger than a piece is
  cut at chunk multiples; a repeated name keeps both entries;
* zip64: force_zip64 local headers on the way in, more than 65 535 members on the way out, no doubled zip64 field;
* dst == src is refused, a failure leaves neither dst nor a temporary file, the tolerate_non_elf / failure split,
  the fallback, the command line, and the two new entry points in the header and the export list.
"""
import io
import os
import re
import struct
import zipfile
import zlib

import pytest

from lambdipy_b200 import _native as N
from lambdipy_b200 import zipfile_gpu as Z
from test_zip_host import ZlibEncoder

MARK = b"\0.symtab"


def elf(payload, debug=b"debug " * 50, refused=False):
    return b"\x7fELF" + (b"!" if refused else b".") + payload + MARK + debug


def fake_strip(data):
    """the stand-in for `strip`: an "ELF" loses everything from the marker on; anything else is refused"""
    return data[:data.index(MARK)] if data[:4] == b"\x7fELF" and MARK in data else None


class FakeMemory:
    """device memory: blocks at addresses 2^40 apart; reading outside a live block fails"""

    def __init__(self):
        self.blocks, self.n = {}, 0

    def put(self, data):
        self.n += 1
        self.blocks[self.n << 40] = bytes(data)
        return self.n << 40

    def get(self, ref):
        addr, n = ref
        block = self.blocks[addr >> 40 << 40]
        off = addr & ((1 << 40) - 1)
        assert off + n <= len(block)
        return block[off:off + n]


def _pack(mem, datas, align):
    off, buf = [], bytearray()
    for d in datas:
        buf += bytes(-len(buf) % align)
        off.append(len(buf))
        buf += d
    base = mem.put(buf)
    return [(base + o, len(d)) for o, d in zip(off, datas)]


class ZlibDecoder:
    def __init__(self, mem):
        self.mem, self.buf, self.block, self.runs = mem, None, None, 0

    def buffer(self, n):
        self.buf = memoryview(bytearray(n))
        return self.buf

    def run_device(self, n, members):
        if self.block is not None:
            del self.mem.blocks[self.block]
        self.runs += 1
        datas, status = [], []
        for off, blen, size, crc, method in members:
            body = bytes(self.buf[off:off + blen])
            try:
                d = zlib.decompressobj(-15).decompress(body) if method == 8 else body
                st = Z.UNZIP_WRONG_SIZE if len(d) != size else Z.UNZIP_BAD_CRC if zlib.crc32(d) != crc else Z.UNZIP_OK
            except zlib.error:
                d, st = b"", Z.UNZIP_BAD_DATA
            datas.append(d if st == Z.UNZIP_OK else bytes(size))
            status.append(st)
        refs = _pack(self.mem, datas, 16)
        self.block = refs[0][0] >> 40 << 40 if refs else None
        return list(zip(status, refs))

    def stats(self):
        return {"kernel_ms": 0.0}


class FakeStripper:
    host_strip = staticmethod(fake_strip)

    def __init__(self, mem):
        self.mem, self.mine, self.uploaded, self.downloaded = mem, [], 0, 0

    def strip(self, refs):
        for b in self.mine:
            del self.mem.blocks[b]
        self.mine = []
        assert all(a % 16 == 0 for a, _ in refs) and len({a >> 40 for a, _ in refs}) <= 1
        outs, status = [], []
        for ref in refs:
            d = self.mem.get(ref)
            refused = d[:5] == b"\x7fELF!"
            out = None if refused else fake_strip(d)
            status.append(N.ST_PLANNER_LIMIT if refused else N.ST_NOT_ELF if out is None else N.ST_OK)
            outs.append(out or b"")
        new = _pack(self.mem, outs, 256)
        if new:
            self.mine.append(new[0][0] >> 40 << 40)
        return list(zip(status, new))

    def fetch(self, ref):
        self.downloaded += ref[1]
        return self.mem.get(ref)

    def upload(self, data):
        self.uploaded += len(data)
        self.mine.append(self.mem.put(data))
        return self.mine[-1], len(data)

    def stats(self):
        return {"plan_ms": 0.0, "compact_ms": 0.0}


class DeviceZlibEncoder(ZlibEncoder):
    """ZlibEncoder fed from the fake device memory, at the offsets lb2_zip_submit_device lays segments out at"""

    def __init__(self, mem, piece_bytes=1 << 20, max_segs=Z.MAX_SEGS):
        super().__init__(piece_bytes, max_segs)
        self.mem, self.piece_bytes, self.k, self.flags = mem, piece_bytes, 0, []

    def submit_device(self, refs, flags):
        off, fill = [], 0
        for ref in refs:
            fill = -(-fill // 16) * 16
            off.append(fill)
            self.buffers[self.k][fill:fill + ref[1]] = self.mem.get(ref)
            fill += ref[1]
        assert fill <= self.piece_bytes
        self.flags.append(([n for _, n in refs], flags))
        self.submit(self.k, fill, off, [n for _, n in refs], flags)
        self.k ^= 1


def engines(piece_bytes=1 << 20, max_segs=Z.MAX_SEGS):
    mem = FakeMemory()
    return ZlibDecoder(mem), FakeStripper(mem), DeviceZlibEncoder(mem, piece_bytes, max_segs)


def symlink_info(name):
    zi = zipfile.ZipInfo(name, (2023, 1, 2, 3, 4, 6))
    zi.create_system, zi.external_attr = 3, (0o120777 << 16)
    return zi


def sample(path):
    """a bundle with every kind of entry; {name: what the member must read back as}"""
    want = {}
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        zf.comment = b"built elsewhere"
        zf.writestr("pkg/__init__.py", b"import this\n" * 40)
        want["pkg/__init__.py"] = b"import this\n" * 40
        zf.writestr("pkg/a.so", elf(b"alpha " * 3000))
        want["pkg/a.so"] = fake_strip(elf(b"alpha " * 3000))
        zf.writestr(zipfile.ZipInfo("pkg/stored.so", (2020, 2, 3, 4, 5, 6)), elf(os.urandom(5000)), zipfile.ZIP_STORED)
        zi = zipfile.ZipInfo("pkg/mode.so", (2021, 2, 3, 4, 5, 6))
        zi.external_attr, zi.comment, zi.extra = 0o100755 << 16, b"a member comment", struct.pack("<HH4s", 0x9999, 4, b"abcd")
        zf.writestr(zi, elf(b"mode " * 100), zipfile.ZIP_DEFLATED)
        want["pkg/mode.so"] = fake_strip(elf(b"mode " * 100))
        zf.writestr("pkg/libz.so.1", elf(b"versioned"))                      # basename does not end in .so
        want["pkg/libz.so.1"] = elf(b"versioned")
        zf.writestr(zipfile.ZipInfo("pkg/dir.so/"), b"")
        zf.writestr(symlink_info("pkg/link.so"), b"a.so")
        want["pkg/link.so"] = b"a.so"
        zf.writestr("pkg/données_名前.txt", "non-ASCII name".encode())
        want["pkg/données_名前.txt"] = "non-ASCII name".encode()
        with zf.open(zipfile.ZipInfo("pkg/streamed.txt", (2022, 1, 1, 1, 1, 2)), "w", force_zip64=True) as f:
            f.write(b"zip64 local header\n" * 10)
        want["pkg/streamed.txt"] = b"zip64 local header\n" * 10
        with zf.open(zipfile.ZipInfo("pkg/z64.so", (2022, 1, 1, 1, 1, 2)), "w", force_zip64=True) as f:
            f.write(elf(b"zip64 so"))
        want["pkg/z64.so"] = fake_strip(elf(b"zip64 so"))
        zf.writestr("pkg/refused.so", elf(b"too many sections", refused=True))
        want["pkg/refused.so"] = fake_strip(elf(b"too many sections", refused=True))
        zf.writestr("empty.txt", b"")
        want["empty.txt"] = b""
    with zipfile.ZipFile(path) as zf:
        want["pkg/stored.so"] = fake_strip(zf.read("pkg/stored.so"))
    return want


def with_descriptor(path, name, data):
    """append a member written to an unseekable stream: flag bit 3, sizes only in the data descriptor"""
    class Unseekable:
        def __init__(self, f):
            self.f = f

        def write(self, b):
            return self.f.write(b)

        def flush(self):
            self.f.flush()

    whole = open(path, "rb").read()
    with open(path, "wb") as f:
        with zipfile.ZipFile(Unseekable(f), "w", zipfile.ZIP_DEFLATED) as zf:
            with zipfile.ZipFile(io.BytesIO(whole)) as old:
                zf.comment = old.comment
                for zi in old.infolist():
                    zf.writestr(zi, old.read(zi), zi.compress_type)
            zf.writestr(name, data)


def local_header(path, zi):
    with open(path, "rb") as f:
        f.seek(zi.header_offset)
        fh = struct.unpack(zipfile.structFileHeader, f.read(zipfile.sizeFileHeader))
        f.seek(fh[zipfile._FH_FILENAME_LENGTH] + fh[zipfile._FH_EXTRA_FIELD_LENGTH], 1)
        return fh, f.read(zi.compress_size)


def test_members_metadata_and_bodies(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "out" / "dst.zip")
    want = sample(src)
    dec, stripper, enc = engines()
    before = open(src, "rb").read()
    st = Z.strip_with(src, dst, dec, stripper, enc)
    assert open(src, "rb").read() == before
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        assert b.testzip() is None and b.comment == b"built elsewhere"
        assert [z.filename for z in b.filelist] == [z.filename for z in a.filelist]
        for za, zb in zip(a.filelist, b.filelist):
            for attr in ("date_time", "external_attr", "create_system", "comment", "internal_attr"):
                assert getattr(za, attr) == getattr(zb, attr), (za.filename, attr)
            assert zb.extra == zipfile._strip_extra(za.extra, (1,))
            fh, body = local_header(dst, zb)
            assert not fh[zipfile._FH_GENERAL_PURPOSE_FLAG_BITS] & 0x08
            if za.filename not in ("pkg/streamed.txt", "pkg/z64.so"):
                assert (fh[zipfile._FH_CRC], fh[zipfile._FH_COMPRESSED_SIZE], fh[zipfile._FH_UNCOMPRESSED_SIZE]) == \
                    (zb.CRC, zb.compress_size, zb.file_size)
            if Z.selected_for_strip(za):
                assert zb.compress_type == zipfile.ZIP_DEFLATED
                assert zlib.decompressobj(-15).decompress(body) == want[za.filename]
            else:                                                      # the body is the source's, byte for byte
                assert (zb.compress_type, zb.CRC, zb.file_size, zb.compress_size) == \
                    (za.compress_type, za.CRC, za.file_size, za.compress_size)
                assert body == local_header(src, za)[1]
            if not zb.is_dir():
                assert b.read(zb) == want[zb.filename]
        assert b.getinfo("pkg/mode.so").extra == struct.pack("<HH4s", 0x9999, 4, b"abcd")
    sel = ["pkg/a.so", "pkg/stored.so", "pkg/mode.so", "pkg/z64.so", "pkg/refused.so"]
    assert (st["members"], st["selected"], st["gpu"], st["fallback"], st["skipped"]) == (12, 5, 4, 1, 2)
    assert st["out_bytes"] == sum(len(want[k]) for k in sel) and st["zip_bytes"] == os.path.getsize(dst)
    assert st["src_zip_bytes"] == len(before) and st["in_bytes"] > st["out_bytes"]
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        refused = len(a.read("pkg/refused.so"))
        assert st["uploaded_bytes"] == sum(a.getinfo(k).compress_size for k in sel) + len(want["pkg/refused.so"])
        assert st["downloaded_bytes"] == sum(b.getinfo(k).compress_size for k in sel) + refused
    assert os.listdir(tmp_path / "out") == ["dst.zip"]


def test_data_descriptors_are_resolved(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    sample(src)
    with_descriptor(src, "late/b.so", elf(b"behind a descriptor " * 20))
    with zipfile.ZipFile(src) as a:
        assert all(z.flag_bits & 0x08 for z in a.filelist if not z.is_dir())
    Z.strip_with(src, dst, *engines())
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        assert b.testzip() is None
        for za, zb in zip(a.filelist, b.filelist):
            fh, _ = local_header(dst, zb)
            assert not zb.flag_bits & 0x08 and not fh[zipfile._FH_GENERAL_PURPOSE_FLAG_BITS] & 0x08
            assert fh[zipfile._FH_CRC] == zb.CRC and fh[zipfile._FH_UNCOMPRESSED_SIZE] == zb.file_size
        assert b.read("late/b.so") == fake_strip(elf(b"behind a descriptor " * 20))
        assert b.read("pkg/__init__.py") == a.read("pkg/__init__.py")


def test_member_larger_than_a_piece_and_batches(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    big = elf(os.urandom(300_001 - 5))
    with zipfile.ZipFile(src, "w", zipfile.ZIP_DEFLATED) as zf:
        zf.writestr("a/pad.so", elf(b"padding " * 6250))
        zf.writestr("a/readme.txt", b"between the two\n")
        zf.writestr("b/big.so", big)
        for i in range(5):
            zf.writestr("c/%d.so" % i, elf(b"small %d " % i * 10))
    for batch_bytes, runs in ((2_000_000, 1), (400_000, 3)):   # the big member behind another in its piece; alone
        dec, stripper, enc = engines(piece_bytes=96 << 10, max_segs=3)
        Z.strip_with(src, dst, dec, stripper, enc, batch_bytes=batch_bytes)
        assert dec.runs == runs
        with zipfile.ZipFile(dst) as b:
            assert b.testzip() is None
            assert b.read("b/big.so") == fake_strip(big) and b.read("a/readme.txt") == b"between the two\n"
            assert [b.read("c/%d.so" % i) for i in range(5)] == [fake_strip(elf(b"small %d " % i * 10)) for i in range(5)]
        parts = [lens[0] if flags & N.ZIP_CONTINUES else lens[-1] for lens, flags in enc.flags
                 if flags & (N.ZIP_CONTINUES | N.ZIP_MORE)]
        assert sum(parts) == len(fake_strip(big)) and len(parts) >= 4 and all(n % Z.CHUNK == 0 for n in parts[:-1])
        assert all(len(lens) <= 3 for lens, _ in enc.flags)


def test_repeated_name_keeps_both_entries(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    with zipfile.ZipFile(src, "w", zipfile.ZIP_DEFLATED) as zf:
        zf.writestr("x.so", elf(b"first"))
        with pytest.warns(UserWarning):
            zf.writestr("x.so", elf(b"second, longer"))
    st = Z.strip_with(src, dst, *engines())
    with zipfile.ZipFile(dst) as b:
        assert [z.filename for z in b.filelist] == ["x.so", "x.so"]
        assert [b.read(z) for z in b.filelist] == [fake_strip(elf(b"first")), fake_strip(elf(b"second, longer"))]
    assert st["gpu"] == 2


def test_more_than_65535_members_zip64_end_records(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    with zipfile.ZipFile(src, "w", zipfile.ZIP_STORED) as zf:
        for i in range(65_600):
            zf.writestr("m/%05d" % i, b"")
        zf.writestr("m/last.so", elf(b"the only object"))
    st = Z.strip_with(src, dst, *engines())
    assert st["members"] == 65_601 and st["gpu"] == 1
    assert zipfile.stringEndArchive64 in open(dst, "rb").read()[-200:]
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        assert b.namelist() == a.namelist() and b.read("m/last.so") == fake_strip(elf(b"the only object"))


def test_zip64_field_is_regenerated_not_doubled():
    zi = zipfile.ZipInfo("big.bin", (2024, 5, 6, 7, 8, 10))
    zi.file_size, zi.compress_size, zi.header_offset, zi.flag_bits, zi.CRC = 5 << 30, 5 << 30, 6 << 30, 0x08, 7
    zi.extra = struct.pack("<HHQQQ", 1, 24, 5 << 30, 5 << 30, 6 << 30) + struct.pack("<HH2s", 0x9999, 2, b"hi")
    out = Z._kept(zi)
    assert out.extra == struct.pack("<HH2s", 0x9999, 2, b"hi") and not out.flag_bits & 0x08 and zi.flag_bits == 0x08
    header = out.FileHeader()
    assert header.count(struct.pack("<HH", 1, 16)) == 1 and header.endswith(struct.pack("<HHQQ", 1, 16, 5 << 30, 5 << 30))
    cd = Z.central_directory([out], 7 << 30, b"note")
    assert cd.count(struct.pack("<HHQQQ", 1, 24, 5 << 30, 5 << 30, 6 << 30)) == 1
    assert zipfile.stringEndArchive64 in cd and cd.endswith(struct.pack("<H", 4) + b"note")


def test_same_file_refused(tmp_path):
    src = str(tmp_path / "src.zip")
    sample(src)
    os.symlink(src, tmp_path / "alias.zip")
    before = open(src, "rb").read()
    for dst in (src, str(tmp_path / "alias.zip"), str(tmp_path / "." / "src.zip")):
        with pytest.raises(ValueError, match="archive being read"):
            Z.strip_with(src, dst, *engines())
    assert open(src, "rb").read() == before and sorted(os.listdir(tmp_path)) == ["alias.zip", "src.zip"]


def test_non_elf_fails_or_is_tolerated_and_nothing_is_left(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    with zipfile.ZipFile(src, "w", zipfile.ZIP_DEFLATED) as zf:
        zf.writestr("ok.so", elf(b"fine"))
        zf.writestr("text.so", b"this is not an ELF file\n" * 10)
        zf.writestr("refused.so", elf(b"planner limit", refused=True))
    with pytest.raises(Z.StripFailed, match="text.so") as e:
        Z.strip_with(src, dst, *engines())
    assert e.value.member == "text.so" and os.listdir(tmp_path) == ["src.zip"]
    with pytest.raises(Z.StripFailed, match="refused.so"):    # reported, not handed to the host strip
        Z.strip_with(src, dst, *engines(), fallback_host_strip=False, tolerate_non_elf=True)
    assert os.listdir(tmp_path) == ["src.zip"]
    st = Z.strip_with(src, dst, *engines(), tolerate_non_elf=True)
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        assert b.read("text.so") == b"this is not an ELF file\n" * 10
        assert local_header(dst, b.getinfo("text.so"))[1] == local_header(src, a.getinfo("text.so"))[1]
        assert b.read("refused.so") == fake_strip(elf(b"planner limit", refused=True))


def test_bad_member_raises_and_nothing_is_left(tmp_path):
    from test_unzip_host import corrupt
    good, dst = tmp_path / "good.zip", str(tmp_path / "dst.zip")
    with zipfile.ZipFile(good, "w", zipfile.ZIP_DEFLATED) as zf:
        zf.writestr("m/0.so", elf(b"zero " * 400))
        zf.writestr("m/3.txt", b"text " * 400)
        zf.writestr("m/3.so", elf(b"three " * 4000))
    for what in ("crc", "size", "body"):
        bad = corrupt(good, tmp_path / "bad.zip", "m/3.so", what)
        with pytest.raises(Z.BadZipMember, match="m/3.so"):
            Z.strip_with(str(bad), dst, *engines())
        os.unlink(bad)
        assert os.listdir(tmp_path) == ["good.zip"]
    bad = corrupt(good, tmp_path / "bad.zip", "m/3.txt", "body")   # an unselected member is not read: copied as it is
    Z.strip_with(str(bad), dst, *engines())


def test_member_the_reader_does_not_take_is_stripped_on_the_host(tmp_path):
    src, dst = str(tmp_path / "src.zip"), str(tmp_path / "dst.zip")
    with zipfile.ZipFile(src, "w") as zf:
        zf.writestr("b/bz.so", elf(b"bzip2 member " * 50), zipfile.ZIP_BZIP2)
        zf.writestr("b/bz.txt", b"stays bzip2 " * 50, zipfile.ZIP_BZIP2)
    dec, stripper, enc = engines()
    st = Z.strip_with(src, dst, dec, stripper, enc)
    assert (st["gpu"], st["fallback"], dec.runs) == (0, 1, 0)
    with zipfile.ZipFile(dst) as b:
        assert b.getinfo("b/bz.so").compress_type == zipfile.ZIP_DEFLATED
        assert b.getinfo("b/bz.txt").compress_type == zipfile.ZIP_BZIP2
        assert b.read("b/bz.so") == fake_strip(elf(b"bzip2 member " * 50)) and b.read("b/bz.txt") == b"stays bzip2 " * 50
    with pytest.raises(Z.StripFailed, match="bz.so"):
        Z.strip_with(src, dst, *engines(), fallback_host_strip=False)


def test_selection():
    def zi(name, mode=0o100644):
        z = zipfile.ZipInfo(name)
        z.create_system, z.external_attr = 3, mode << 16
        return z
    assert Z.selected_for_strip(zi("a/b.so")) is True and Z.selected_for_strip(zi(".so")) is True
    assert Z.selected_for_strip(zipfile.ZipInfo("plain.so")) is True            # no Unix mode at all
    assert Z.selected_for_strip(zi("a/b.so.1")) is None and Z.selected_for_strip(zi("x.so/y.py")) is None
    assert Z.selected_for_strip(zi("d.so/", 0o40755)) is False and Z.selected_for_strip(zi("l.so", 0o120777)) is False


def test_main_arguments(monkeypatch, tmp_path, capsys):
    calls = []

    def fake(src, dst, compresslevel=None):
        calls.append((src, dst, compresslevel))
        with zipfile.ZipFile(dst, "w") as zf:
            zf.writestr("a.so", b"x" * 1000)
        return {"zip_bytes": os.path.getsize(dst), "gpu": 3, "fallback": 1, "in_bytes": 5_000_000, "out_bytes": 2_000_000}

    monkeypatch.setattr(Z, "strip_zip", fake)
    dst = str(tmp_path / "o.zip")
    assert Z.main(["strip", "in.zip", dst]) == 0
    assert Z.main(["strip", "in.zip", dst, "--level", "9"]) == 0
    assert calls == [("in.zip", dst, None), ("in.zip", dst, 9)]
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == 2 and "50 MB" in lines[0] and "250 MB" in lines[0] and "o.zip" in lines[0]
    assert "4 shared objects stripped (1 via host strip), 5.0 MB -> 2.0 MB" in lines[0]
    for bad in (["strip", "in.zip"], ["strip", "a", "b", "--level", "6"], ["unstrip", "a", "b"], []):
        with pytest.raises(SystemExit):
            Z.main(bad)
    assert len(calls) == 2


def test_new_entry_points_declared_and_exported():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "lambdipy_b200.h")).read()
    for name in ("lb2_zip_submit_device", "lb2_unzip_device_output"):
        assert re.search(r"\bint %s\(" % name, header) and name in N.EXPORTS
    assert "typedef struct lb2_zip_source" in header
    assert [f for f, _ in N.ZipSource._fields_] == ["d_ptr", "len"]
