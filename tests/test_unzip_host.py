"""CPU checks of the zip reader's container logic (lambdipy_b200/zipfile_gpu.py: extract_with / testzip_with) with a
zlib stand-in for the GPU decoder: the extracted tree must equal ZipFile.extractall's on crafted archives, members the
GPU does not take must go to the stdlib's own code, and LAMBDIPY_BUNDLE_VERIFY must be checked and passed through."""
import io
import os
import struct
import sys
import warnings
import zipfile
import zlib

import pytest

from lambdipy_b200 import zipfile_gpu as Z


class ZlibDecoder:
    """Stand-in for GpuUnzipDecoder: the same buffer / run / stats, with each member decoded by zlib and given the
    status the CUDA reader gives it."""

    def __init__(self, capacity=None):
        self.buf, self.runs, self.members, self.capacity = bytearray(), 0, 0, capacity

    def buffer(self, n):
        self.buf = bytearray(n)
        return memoryview(self.buf)

    def run(self, n, members):
        if self.capacity is not None and sum(m[1] + 3 * m[2] for m in members) > self.capacity:
            raise Z.DeviceTooSmall("stand-in capacity")
        self.runs += 1
        self.members += len(members)
        out = []
        for off, blen, size, crc, method in members:
            assert 0 <= off and off + blen <= n
            body = bytes(self.buf[off:off + blen])
            if method == 0:
                data, status = body, (Z.UNZIP_OK if blen == size else Z.UNZIP_WRONG_SIZE)
            else:
                d = zlib.decompressobj(-15)
                try:
                    data = d.decompress(body)
                    status = Z.UNZIP_OK if d.eof else Z.UNZIP_BAD_DATA
                except zlib.error:
                    data, status = b"", Z.UNZIP_BAD_DATA
                if status == Z.UNZIP_OK and len(data) != size:
                    status = Z.UNZIP_WRONG_SIZE
            if status == Z.UNZIP_OK and zlib.crc32(data) != crc:
                status = Z.UNZIP_BAD_CRC
            out.append((status, memoryview(data)))
        return out

    def stats(self):
        return {"runs": self.runs}


def tree(root):
    out = {}
    for dirpath, dirnames, filenames in os.walk(root):
        for d in dirnames:
            out[os.path.relpath(os.path.join(dirpath, d), root)] = None
        for f in filenames:
            p = os.path.join(dirpath, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


def same_as_extractall(tmp_path, zip_path, **kw):
    want, got = tmp_path / "want", tmp_path / "got"
    with zipfile.ZipFile(zip_path) as zf:
        zf.extractall(want)
    dec = ZlibDecoder()
    st = Z.extract_with(zip_path, got, dec, **kw)
    assert tree(got) == tree(want)
    assert Z.testzip_with(zip_path, ZlibDecoder(), **kw)[0] is None
    return st, dec


def write_zip(path, entries, compression=zipfile.ZIP_DEFLATED):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # duplicate names
        with zipfile.ZipFile(path, "w", compression) as zf:
            for name, data in entries:
                zf.writestr(zipfile.ZipInfo(name) if not name.endswith("/") else name, data)
    return path


def test_hostile_names(tmp_path):
    entries = [("../evil.txt", b"a" * 100), ("/abs/root.txt", b"b"), ("a/../../c.txt", b"c" * 5000),
               ("C:/drive/d.txt", b"d"), ("./dot/./e.txt", b"e"), ("x//y///f.txt", b"f"), ("sub/", b""),
               ("sub/g.bin", os.urandom(3000)), ("..\\back\\h.txt", b"h")]
    st, _ = same_as_extractall(tmp_path, write_zip(tmp_path / "h.zip", entries))
    assert st["gpu_members"] == len(entries) - 1 and st["stdlib_members"] == 0


def test_duplicate_names(tmp_path):
    entries = [("dup.txt", b"first" * 100), ("other.txt", b"o"), ("dup.txt", b"second" * 50), ("d/", b""), ("d/", b"")]
    same_as_extractall(tmp_path, write_zip(tmp_path / "d.zip", entries))


def test_directories_only(tmp_path):
    st, dec = same_as_extractall(tmp_path, write_zip(tmp_path / "dirs.zip", [("a/", b""), ("a/b/", b""), ("c/", b"")]))
    assert st["gpu_members"] == 0 and dec.runs == 0


def test_zip64_many_entries_and_batches(tmp_path):
    n = 65_600
    path = tmp_path / "many.zip"
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for i in range(n):
            zf.writestr("f/%05d" % i, b"%d" % i * (i % 7))
    with open(path, "rb") as fh:
        assert zipfile.structEndArchive64Locator and b"PK\x06\x06" in fh.read()[-200:]  # the zip64 end record
    st, dec = same_as_extractall(tmp_path, path, batch_bytes=4 << 20)
    assert st["gpu_members"] == n and st["batches"] > 1 and dec.runs == st["batches"]


def test_data_descriptors(tmp_path):
    raw = io.BytesIO()

    class Unseekable:
        def write(self, b):
            return raw.write(b)

        def flush(self):
            pass

    with zipfile.ZipFile(Unseekable(), "w", zipfile.ZIP_DEFLATED) as zf:
        for i in range(20):
            with zf.open("dd/%d.txt" % i, "w") as f:
                f.write(b"descriptor %d " % i * (i * 50))
    path = tmp_path / "dd.zip"
    path.write_bytes(raw.getvalue())
    with zipfile.ZipFile(path) as zf:
        assert all(zi.flag_bits & 0x08 for zi in zf.infolist())
    st, _ = same_as_extractall(tmp_path, path)
    assert st["gpu_members"] == 20


def test_prepended_bytes(tmp_path):
    inner = write_zip(tmp_path / "inner.zip", [("p/a.txt", b"prepended " * 300), ("p/b.txt", b"")])
    path = tmp_path / "sfx.zip"
    path.write_bytes(b"#!/bin/sh\necho self-extracting\nexit 0\n" * 40 + inner.read_bytes())
    st, _ = same_as_extractall(tmp_path, path)
    assert st["gpu_members"] == 2


def test_stored_bzip2_lzma_members(tmp_path):
    path = tmp_path / "mixed.zip"
    with zipfile.ZipFile(path, "w") as zf:
        zf.writestr("s.txt", b"stored " * 99, compress_type=zipfile.ZIP_STORED)
        zf.writestr("z.txt", b"deflated " * 99, compress_type=zipfile.ZIP_DEFLATED)
        zf.writestr("b.txt", b"bzip2 " * 99, compress_type=zipfile.ZIP_BZIP2)
        zf.writestr("l.txt", b"lzma " * 99, compress_type=zipfile.ZIP_LZMA)
    st, _ = same_as_extractall(tmp_path, path)
    assert st["gpu_members"] == 2 and st["stdlib_members"] == 2


def test_member_too_large_for_the_device_goes_to_the_stdlib(tmp_path):
    path = write_zip(tmp_path / "big.zip", [("small.txt", b"s" * 10), ("big.bin", os.urandom(200_000)),
                                            ("small2.txt", b"t" * 10)])
    want, got = tmp_path / "want", tmp_path / "got"
    with zipfile.ZipFile(path) as zf:
        zf.extractall(want)
    st = Z.extract_with(path, got, ZlibDecoder(capacity=100_000))
    assert tree(got) == tree(want)
    assert st["gpu_members"] == 2 and st["stdlib_members"] == 1


def set_flag(data, bit):
    """set general-purpose flag `bit` in every local and central header"""
    b = bytearray(data)
    for sig, at in ((b"PK\x03\x04", 6), (b"PK\x01\x02", 8)):
        i = b.find(sig)
        while i >= 0:
            b[i + at] |= bit
            i = b.find(sig, i + 4)
    return bytes(b)


def test_encrypted_member_raises_what_the_stdlib_raises(tmp_path):
    plain = write_zip(tmp_path / "plain.zip", [("secret.txt", b"hidden " * 40)], zipfile.ZIP_STORED)
    path = tmp_path / "enc.zip"
    path.write_bytes(set_flag(plain.read_bytes(), 0x01))
    with zipfile.ZipFile(path) as zf, pytest.raises(RuntimeError) as want:
        zf.extractall(tmp_path / "want")
    with pytest.raises(RuntimeError) as got:
        Z.extract_with(path, tmp_path / "got", ZlibDecoder())
    assert str(got.value) == str(want.value)


def corrupt(path, out, name, what):
    """a copy of `path` with member `name`'s CRC, body or size changed in its central directory entry or body"""
    data = bytearray(path.read_bytes())
    with zipfile.ZipFile(path) as zf:
        zi = zf.getinfo(name)
        cd = data.find(zi.filename.encode(), zf.start_dir) - 46
        assert data[cd:cd + 4] == b"PK\x01\x02"
        if what == "crc":
            data[cd + 16] ^= 0x01
        elif what == "size":  # one byte fewer: the stdlib's CRC check then fails too
            data[cd + 24:cd + 28] = struct.pack("<I", zi.file_size - 1)
        elif what == "body":
            body = zi.header_offset + 30 + len(zi.filename.encode()) + len(zi.extra)
            for k in range(8):
                data[body + k] ^= 0xFF
    out.write_bytes(bytes(data))
    return out


def test_testzip_names_the_first_bad_member_and_crc_raises(tmp_path):
    entries = [("m/%d.txt" % i, (b"member %d " % i) * 400) for i in range(6)]
    good = write_zip(tmp_path / "good.zip", entries)
    for what in ("crc", "size", "body"):
        bad = corrupt(good, tmp_path / ("bad_%s.zip" % what), "m/3.txt", what)
        try:
            with zipfile.ZipFile(bad) as zf:
                want = zf.testzip()
        except (zlib.error, EOFError):
            want = "m/3.txt"
        assert Z.testzip_with(bad, ZlibDecoder())[0] == want == "m/3.txt", what
    bad = tmp_path / "bad_crc.zip"
    with pytest.raises(zipfile.BadZipFile, match=r"Bad CRC-32 for file 'm/3.txt'"):
        Z.extract_with(bad, tmp_path / "x", ZlibDecoder())
    with pytest.raises(Z.BadZipMember, match="m/3.txt"):
        Z.extract_with(tmp_path / "bad_size.zip", tmp_path / "y", ZlibDecoder())
    assert not os.path.exists(tmp_path / "x" / "m" / "0.txt")  # the batch is checked before any file is written


# ---- LAMBDIPY_BUNDLE_VERIFY ----------------------------------------------------------------------------------------
@pytest.fixture
def standin(tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lambdipy"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "project_build.py").write_text(
        "def install_non_resolved_requirements(*a, **k):\n    pass\n"
        "def copy_include_paths(include_paths, build_directory='./build'):\n    COPIED.append(build_directory)\n"
        "COPIED = []\n")
    (pkg / "cli.py").write_text("from .project_build import install_non_resolved_requirements, copy_include_paths\n")
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    monkeypatch.setenv("LAMBDIPY_B200_EAGER_WARMUP", "0")
    for v in ("LAMBDIPY_TARBALL_BACKEND", "LAMBDIPY_UNTAR_BACKEND", "LAMBDIPY_BUNDLE_ZIP", "LAMBDIPY_DEFLATE_LEVEL",
              "LAMBDIPY_BUNDLE_VERIFY"):
        monkeypatch.delenv(v, raising=False)
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


@pytest.mark.parametrize("bad", ["", "0", "true", "yes", " 1", "2"])
def test_verify_refused_before_rebinding(standin, monkeypatch, tmp_path, bad):
    monkeypatch.setenv("LAMBDIPY_BUNDLE_VERIFY", bad)
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", str(tmp_path / "b.zip"))
    import lambdipy.cli as cli
    import lambdipy.project_build as ref
    from lambdipy_b200 import patch
    before = (ref.install_non_resolved_requirements, cli.copy_include_paths)
    with pytest.raises(ValueError, match="LAMBDIPY_BUNDLE_VERIFY"):
        patch.apply()
    assert (ref.install_non_resolved_requirements, cli.copy_include_paths) == before


def test_verify_hook(standin, monkeypatch, tmp_path, capsys):
    import lambdipy.cli as cli
    from lambdipy_b200 import patch
    checked = []

    def fake_zip_tree(root, path, ctx=None, **kw):
        write_zip(path, [("a.txt", b"a"), ("b/", b""), ("b/c.txt", b"c")])
        return {}

    monkeypatch.setattr(Z, "zip_tree", fake_zip_tree)
    monkeypatch.setattr(Z, "testzip", lambda path, ctx=None: checked.append(path) or None)
    (tmp_path / "build").mkdir()
    monkeypatch.chdir(tmp_path)
    zip_path = str(tmp_path / "bundle.zip")
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", zip_path)
    patch.apply()  # unset: no check, the line as before
    cli.copy_include_paths(())
    assert checked == [] and "members checked" not in capsys.readouterr().out
    monkeypatch.setenv("LAMBDIPY_BUNDLE_VERIFY", "1")
    patch.apply()
    cli.copy_include_paths(())
    assert checked == [zip_path] and "; 3 members checked" in capsys.readouterr().out
    monkeypatch.setattr(Z, "testzip", lambda path, ctx=None: "b/c.txt")
    with pytest.raises(RuntimeError, match="b/c.txt"):
        cli.copy_include_paths(())
