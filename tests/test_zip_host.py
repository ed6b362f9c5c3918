"""CPU checks of the zip writer's container (lambdipy_b200.zipfile_gpu) and of its build-flow hook.

* with the member bodies from zlib level 6 (what zipfile itself writes), zip_tree's container is
  `shutil.make_archive`'s output byte for byte: nested and empty directories, empty / 1-byte / 64 KB +- 1 files, a file
  spanning three pieces, an executable mode, symlinks to a file and to a directory, a non-ASCII name, and a tree of
  65 600 empty files (zip64 end records);
* zip64 headers of members over 4 GiB equal ZipInfo.FileHeader's and ZipFile's central-directory record;
* LAMBDIPY_BUNDLE_ZIP: a bad value is refused before anything is rebound; the hook is installed only when it is set.
"""
import os
import shutil
import struct
import sys
import zipfile
import zlib

import pytest

from lambdipy_b200 import _native as N
from lambdipy_b200 import zipfile_gpu as Z


class ZlibEncoder:
    """GpuZipEncoder's interface with zlib's raw DEFLATE at level 6 (compressobj(-1, DEFLATED, -15), as zipfile)."""

    def __init__(self, piece_bytes, max_segs=Z.MAX_SEGS):
        self.buffers = [memoryview(bytearray(piece_bytes)) for _ in range(2)]
        self.max_segs = max_segs
        self.done, self.z, self.crc, self.open, self.pieces = [], None, 0, False, 0

    def submit(self, k, n, seg_off, seg_len, flags):
        assert len(self.done) < 2 and 0 < len(seg_off) <= self.max_segs
        assert bool(flags & N.ZIP_CONTINUES) == self.open and (not self.open or seg_off[0] == 0)
        out, res, end = bytearray(), [], 0
        for i, (o, n_i) in enumerate(zip(seg_off, seg_len)):
            assert o % Z.ALIGN == 0 and o >= end and o + n_i <= n
            end = o + n_i
            if not (i == 0 and flags & N.ZIP_CONTINUES):
                self.z, self.crc = zlib.compressobj(-1, zlib.DEFLATED, -15), 0
            data = bytes(self.buffers[k][o:o + n_i])
            start = len(out)
            out += self.z.compress(data)
            self.crc = zlib.crc32(data, self.crc)
            ended = i + 1 < len(seg_off) or not flags & N.ZIP_MORE
            if ended:
                out += self.z.flush()
            res.append((start, len(out) - start, self.crc, ended))
        self.open = bool(flags & N.ZIP_MORE)
        self.done.append((memoryview(bytes(out)), res))
        self.pieces += 1

    def collect(self):
        return self.done.pop(0)

    def stats(self):
        return {"pieces": self.pieces}


def edge_tree(root):
    """the edge cases of the container, as files under root"""
    os.makedirs(os.path.join(root, "pkg", "sub", "deeper"))
    os.makedirs(os.path.join(root, "empty_dir"))
    os.makedirs(os.path.join(root, "pkg", "empty_nested"))
    sizes = {"empty.txt": 0, "one.bin": 1, "k64m1.bin": 65535, "k64.bin": 65536, "k64p1.bin": 65537}
    for i, (name, n) in enumerate(sizes.items()):
        with open(os.path.join(root, "pkg", name), "wb") as f:
            f.write(bytes((j * 7 + i) & 0xFF for j in range(n // 3)) + os.urandom(n - n // 3))
    with open(os.path.join(root, "pkg", "sub", "big.txt"), "wb") as f:      # three 96 KB pieces and a bit
        f.write(b"".join(b"line %d of a file spanning pieces\n" % i for i in range(9000)))
    with open(os.path.join(root, "pkg", "sub", "deeper", "run.sh"), "w") as f:
        f.write("#!/bin/sh\necho hi\n")
    os.chmod(os.path.join(root, "pkg", "sub", "deeper", "run.sh"), 0o755)
    with open(os.path.join(root, "données_ünïcödé_名前.py"), "w", encoding="utf-8") as f:
        f.write("# non-ASCII name\n")
    os.symlink("pkg/one.bin", os.path.join(root, "link_to_file"))
    os.symlink("pkg/sub", os.path.join(root, "link_to_dir"))
    os.symlink("missing", os.path.join(root, "dangling"))
    return root


def make_archive_bytes(root, tmp):
    return open(shutil.make_archive(os.path.join(tmp, "ref"), "zip", root), "rb").read()


@pytest.mark.parametrize("piece_bytes", [96 << 10, 1 << 20])
def test_container_equals_make_archive(tmp_path, piece_bytes):
    root = edge_tree(str(tmp_path / "tree"))
    assert os.path.getsize(os.path.join(root, "pkg", "sub", "big.txt")) > 2 * (96 << 10)
    enc = ZlibEncoder(piece_bytes)
    out = str(tmp_path / "out" / "gpu.zip")
    st = Z.write_zip(root, out, enc)
    ref = make_archive_bytes(root, str(tmp_path))
    assert open(out, "rb").read() == ref
    assert st["zip_bytes"] == len(ref) and st["files"] == sum(1 for i in zipfile.ZipFile(out).infolist() if not i.is_dir())
    if piece_bytes == 96 << 10:
        assert enc.pieces >= 3


def test_container_many_files_zip64_end_records(tmp_path):
    root = tmp_path / "many"
    for d in range(41):
        (root / ("d%02d" % d)).mkdir(parents=True)
        for i in range(1600):
            (root / ("d%02d" % d) / ("f%04d" % i)).touch()
    out = str(tmp_path / "many.zip")
    enc = ZlibEncoder(1 << 20, max_segs=4096)
    st = Z.write_zip(str(root), out, enc)
    ref = make_archive_bytes(str(root), str(tmp_path))
    data = open(out, "rb").read()
    assert st["entries"] == 41 + 41 * 1600 > zipfile.ZIP_FILECOUNT_LIMIT
    assert zipfile.stringEndArchive64 in data[-200:]
    assert data == ref
    assert enc.pieces >= 16


def _central_record_by_zipfile(zi):
    """ZipFile.close()'s central directory and end records for one entry, starting at offset 0"""
    import io
    buf = io.BytesIO()
    zf = zipfile.ZipFile(buf, "w")
    zf.filelist.append(zi)
    zf._didModify = True
    zf.close()
    return buf.getvalue()


@pytest.mark.parametrize("size,offset", [(5 << 30, 100), (100, 5 << 30), (5 << 30, 6 << 30), (100, 100)])
def test_zip64_headers(size, offset):
    zi = zipfile.ZipInfo("big.bin", (2024, 5, 6, 7, 8, 10))
    zi.external_attr = 0o644 << 16
    zi.file_size = size
    # the container writer's header for this member: zip64 from ZipFile's size guess, then the final values
    w = Z._ContainerWriter(_Sink(offset), [("big.bin", zi)])
    w.part(0, b"\x03\x00", 0x1234, False, 0)
    w.part(0, b"", 0x1234, True, size)
    first, final = w.fp.writes[0], w.fp.writes[-1]
    ref = zipfile.ZipInfo("big.bin", (2024, 5, 6, 7, 8, 10))
    ref.external_attr, ref.file_size, ref.compress_type = 0o644 << 16, size, zipfile.ZIP_DEFLATED
    ref.CRC = ref.compress_size = 0
    zip64 = size * 1.05 > zipfile.ZIP64_LIMIT
    assert first == ref.FileHeader(zip64)
    ref.CRC, ref.compress_size = 0x1234, 2
    assert final == ref.FileHeader(zip64)
    assert (struct.unpack("<I", final[22:26])[0] == 0xFFFFFFFF) == zip64
    ref.header_offset = offset
    assert zi.header_offset == offset
    assert Z.central_directory([zi], 0) == _central_record_by_zipfile(ref)


class _Sink:
    """a write-only file at `offset` that records every write"""

    def __init__(self, offset):
        self.pos, self.writes = offset, []

    def tell(self):
        return self.pos

    def seek(self, p):
        self.pos = p

    def write(self, b):
        self.writes.append(bytes(b))
        self.pos += len(b)


# ---------------------------------------------------------------------------------------------- build-flow hook
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
    for v in ("LAMBDIPY_TARBALL_BACKEND", "LAMBDIPY_UNTAR_BACKEND", "LAMBDIPY_BUNDLE_ZIP"):
        monkeypatch.delenv(v, raising=False)
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


@pytest.mark.parametrize("bad", ["", "bundle.tar.gz", "bundle", ".zip"])
def test_bundle_zip_bad_value_refused_before_rebinding(standin, monkeypatch, bad):
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", bad)
    import lambdipy.cli as cli
    import lambdipy.project_build as ref
    from lambdipy_b200 import patch
    before = (ref.install_non_resolved_requirements, cli.copy_include_paths)
    with pytest.raises(ValueError, match="LAMBDIPY_BUNDLE_ZIP"):
        patch.apply()
    assert (ref.install_non_resolved_requirements, cli.copy_include_paths) == before


def test_bundle_zip_directory_refused(standin, monkeypatch, tmp_path):
    (tmp_path / "d.zip").mkdir()
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", str(tmp_path / "d.zip"))
    from lambdipy_b200 import patch
    with pytest.raises(ValueError, match="LAMBDIPY_BUNDLE_ZIP"):
        patch.apply()


def test_bundle_zip_hook_only_when_set(standin, monkeypatch, tmp_path, capsys):
    import lambdipy.cli as cli
    import lambdipy.project_build as ref
    from lambdipy_b200 import patch
    original = cli.copy_include_paths
    patch.apply()
    assert cli.copy_include_paths is original          # unset: the reference's own function

    calls = []
    monkeypatch.setattr(Z, "zip_tree", lambda root, path, ctx=None: calls.append((root, path)) or
                        open(path, "wb").write(b"x" * 1000) and {"zip_bytes": 1000})
    target = str(tmp_path / "bundle.zip")
    monkeypatch.setenv("LAMBDIPY_BUNDLE_ZIP", target)
    build = tmp_path / "build"
    build.mkdir()
    (build / "a.py").write_bytes(b"y" * 5000)
    monkeypatch.chdir(tmp_path)
    patch.apply()
    assert cli.copy_include_paths is not original
    cli.copy_include_paths(())
    assert ref.COPIED == ["./build"] and calls == [("./build", target)]
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert "50 MB" in line and "250 MB" in line and "bundle.zip" in line


class _RecordingEncoder(ZlibEncoder):
    """ZlibEncoder that records the (entry bytes, flags) of every piece"""

    def __init__(self, piece_bytes):
        super().__init__(piece_bytes)
        self.parts = []

    def submit(self, k, n, seg_off, seg_len, flags):
        self.parts.append((list(seg_len), flags))
        super().submit(k, n, seg_off, seg_len, flags)


def test_continued_files_are_cut_at_chunk_multiples(tmp_path):
    """a file that goes on in the next piece leaves a multiple of 64 KB of its bytes in each earlier piece, so the
    encoder cuts it into the chunks it would cut it into whole (no extra chunk or framing per piece boundary)"""
    root = tmp_path / "tree"
    (root / "a").mkdir(parents=True)                    # os.walk visits a/ before b/
    (root / "b").mkdir()
    (root / "a" / "pad.txt").write_bytes(b"padding " * 6250)       # 50 000 bytes in front of the big file
    (root / "b" / "big.bin").write_bytes(os.urandom(300_001))
    enc = _RecordingEncoder(96 << 10)
    out = str(tmp_path / "x.zip")
    Z.write_zip(str(root), out, enc)
    assert open(out, "rb").read() == make_archive_bytes(str(root), str(tmp_path))
    big = []                                            # the big file's part in each piece, in order
    for lens, flags in enc.parts:
        if flags & N.ZIP_CONTINUES or flags & N.ZIP_MORE:
            big.append(lens[0] if flags & N.ZIP_CONTINUES else lens[-1])
    assert sum(big) == 300_001 and len(big) == 5
    assert all(n % Z.CHUNK == 0 for n in big[:-1])


def test_piece_smaller_than_a_chunk_refused(tmp_path):
    (tmp_path / "t").mkdir()
    with pytest.raises(ValueError, match="at least"):
        Z.write_zip(str(tmp_path / "t"), str(tmp_path / "x.zip"), ZlibEncoder(Z.CHUNK - 16))
