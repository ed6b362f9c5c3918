"""CPU-side checks of the tarball reading path: the gzip framing parser against gzip.decompress, patch.apply()'s
LAMBDIPY_UNTAR_BACKEND switch, and the prepare_tarfile mirror (download call, extraction target, and the hand-over to
the reference's own tarfile lines when the GPU reader refuses the data)."""
import ctypes
import gzip
import io
import os
import struct
import sys
import tarfile
import zlib

import pytest

from lambdipy_b200 import _native as N
from lambdipy_b200 import tarball


def _member(data, flags=0, extra=b"xy", name=b"n.tar", comment=b"c", level=6):
    head = struct.pack("<BBBBIBB", 0x1F, 0x8B, 8, flags, 0, 0, 255)
    if flags & tarball.FEXTRA:
        head += struct.pack("<H", len(extra)) + extra
    if flags & tarball.FNAME:
        head += name + b"\0"
    if flags & tarball.FCOMMENT:
        head += comment + b"\0"
    if flags & tarball.FHCRC:
        head += struct.pack("<H", zlib.crc32(head) & 0xFFFF)
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    return head + c.compress(data) + c.flush() + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def _split(buf):
    """(body offset, body length) per member, found by the framing parser with zlib standing in for the GPU"""
    out, gen = [], tarball.gzip_members(memoryview(buf))
    body = next(gen, None)
    while body is not None:
        d = zlib.decompressobj(-15)
        d.decompress(buf[body:])
        used = len(buf) - body - len(d.unused_data)
        out.append((body, used))
        try:
            body = gen.send(used)
        except StopIteration:
            body = None
    return out


@pytest.mark.parametrize("flags", range(32))
def test_framing_every_flag_combination(flags):
    data = b"payload %d " % flags * 50
    gz = _member(data, flags)
    (body, used), = _split(gz)
    assert zlib.decompress(gz[body:body + used], -15) == data == gzip.decompress(gz)


def test_framing_members_and_zero_padding():
    parts = [b"a" * 1000, b"", b"bc" * 7000]
    gz = _member(parts[0], tarball.FNAME) + b"\0" * 5 + _member(parts[1]) + _member(parts[2], tarball.FEXTRA) + b"\0" * 3
    got = [zlib.decompress(gz[b:b + u], -15) for b, u in _split(gz)]
    assert got == parts and b"".join(got) == gzip.decompress(gz)


@pytest.mark.parametrize("mutate", ["magic", "method"])
def test_framing_errors_match_stdlib(mutate):
    gz = bytearray(_member(b"x" * 100))
    gz[0 if mutate == "magic" else 2] ^= 0x40
    with pytest.raises(gzip.BadGzipFile) as want:
        gzip.decompress(bytes(gz))
    with pytest.raises(type(want.value)):
        _split(bytes(gz))


def test_framing_refuses_reserved_flags():
    gz = bytearray(_member(b"x" * 100))
    gz[3] |= 0x20
    with pytest.raises(zlib.error):       # zlib refuses them; gzip.GzipFile ignores them
        zlib.decompress(bytes(gz), 31)
    with pytest.raises(gzip.BadGzipFile):
        _split(bytes(gz))


@pytest.fixture
def standin_lambdipy(tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lambdipy"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "project_build.py").write_text("def install_non_resolved_requirements(*a, **k):\n    raise AssertionError\n"
                                          "def prepare_tarfile(url, download_filename, package_directory):\n    return 'ref'\n")
    (pkg / "cli.py").write_text("from .project_build import install_non_resolved_requirements\n")
    (pkg / "package_build.py").write_text("class PackageBuild:\n    def create_compressed_tarball(self):\n        return 'ref'\n")
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    monkeypatch.setenv("LAMBDIPY_B200_EAGER_WARMUP", "0")
    monkeypatch.delenv("LAMBDIPY_TARBALL_BACKEND", raising=False)
    yield
    for k in [k for k in sys.modules if k == "lambdipy" or k.startswith("lambdipy.")]:
        del sys.modules[k]


def test_patch_leaves_prepare_tarfile_alone_by_default(standin_lambdipy, monkeypatch):
    import lambdipy_b200.patch as patch
    import lambdipy.project_build as ref
    before = ref.prepare_tarfile
    monkeypatch.delenv("LAMBDIPY_UNTAR_BACKEND", raising=False)
    patch.apply()
    assert ref.prepare_tarfile is before
    monkeypatch.setenv("LAMBDIPY_UNTAR_BACKEND", "python")
    patch.apply()
    assert ref.prepare_tarfile is before


def test_patch_installs_gpu_prepare_tarfile_when_asked(standin_lambdipy, monkeypatch):
    import lambdipy_b200.patch as patch
    import lambdipy.project_build as ref
    monkeypatch.setenv("LAMBDIPY_UNTAR_BACKEND", "b200")
    patch.apply()
    assert ref.prepare_tarfile is tarball.prepare_tarfile
    assert "lambdipy.package_build" not in sys.modules   # the writer's switch is separate


@pytest.mark.parametrize("var", ["LAMBDIPY_UNTAR_BACKEND", "LAMBDIPY_TARBALL_BACKEND"])
def test_patch_rejects_unknown_untar_backend_before_patching(standin_lambdipy, monkeypatch, var):
    import lambdipy_b200.patch as patch
    import lambdipy.project_build as ref
    import lambdipy.cli as cli
    before = (ref.install_non_resolved_requirements, ref.prepare_tarfile, cli.install_non_resolved_requirements)
    monkeypatch.setenv("LAMBDIPY_UNTAR_BACKEND", "b200")
    monkeypatch.setenv(var, "pigz")
    with pytest.raises(ValueError):
        patch.apply()
    assert (ref.install_non_resolved_requirements, ref.prepare_tarfile, cli.install_non_resolved_requirements) == before


def test_gunzip_is_public():
    import lambdipy_b200
    assert lambdipy_b200.gunzip is tarball.gunzip


def _tarball(tmp_path):
    src = tmp_path / "src" / "pkg"
    src.mkdir(parents=True)
    (src / "a.py").write_text("a = 1\n")
    (src / "lib.so").write_bytes(os.urandom(5000))
    path = tmp_path / "pkg.tar.gz"
    with tarfile.open(path, "w:gz") as tar:
        tar.add(src, arcname="pkg")
    return str(path)


def test_mirror_downloads_once_and_extracts_into_package_directory(tmp_path, monkeypatch):
    src = _tarball(tmp_path)
    calls, extracted = [], []
    monkeypatch.setattr(tarball.urllib.request, "urlretrieve", lambda url, fn: calls.append((url, fn)) or
                        open(fn, "wb").write(open(src, "rb").read()))
    monkeypatch.setattr(tarball, "extract_tarball", lambda p, d, ctx=None: extracted.append((p, d)))
    dl, dest = str(tmp_path / "dl.tar.gz"), str(tmp_path / "pkgdir")
    tarball.prepare_tarfile("https://example.invalid/pkg.tar.gz", dl, dest)
    assert calls == [("https://example.invalid/pkg.tar.gz", dl)]
    assert extracted == [(dl, dest)]


class _FakeLib:
    """lb2_inflate_* whose run reports LB2_E_DATA"""
    def lb2_inflate_create(self, h, flags, out):
        return 0

    def lb2_inflate_run(self, d, h_in, n, out_n, st):
        return N.LB2_E_DATA

    def lb2_inflate_destroy(self, d):
        pass

    def lb2_last_error(self, h):
        return b"invalid DEFLATE stream"


class _FakeCtx:
    def __init__(self):
        self.lib, self.h, self._bufs = _FakeLib(), None, {}

    def pinned_alloc(self, n):
        b = ctypes.create_string_buffer(n)
        self._bufs[ctypes.addressof(b)] = b
        return ctypes.addressof(b)

    def pinned_free(self, p):
        del self._bufs[p]

    def check(self, rc):
        assert rc == 0

    def close(self):
        pass


def test_mirror_hands_refused_data_to_the_reference_lines(tmp_path, monkeypatch, capsys):
    src = _tarball(tmp_path)
    monkeypatch.setattr(tarball.urllib.request, "urlretrieve", lambda url, fn: open(fn, "wb").write(open(src, "rb").read()))
    monkeypatch.setattr(tarball, "_default_context", lambda: (_FakeCtx(), True))
    opened = []
    real_open = tarfile.open
    monkeypatch.setattr(tarball.tarfile, "open", lambda *a, **k: opened.append((a, k)) or real_open(*a, **k))
    dl, dest = str(tmp_path / "dl.tar.gz"), tmp_path / "pkgdir"
    tarball.prepare_tarfile("https://example.invalid/pkg.tar.gz", dl, str(dest))
    assert opened == [((dl, "r:gz"), {})]
    assert (dest / "pkg" / "a.py").read_text() == "a = 1\n"
    assert "extracting with tarfile" in capsys.readouterr().out
