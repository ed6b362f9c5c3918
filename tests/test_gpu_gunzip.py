"""GPU checks of the gzip reader (lb2_inflate_*, tarball.gunzip / extract_tarball / prepare_tarfile): every stream
decodes to zlib's bytes at the default span size and at tiny spans, false candidates are rejected, corrupt input is
refused, and extracted trees equal the reference's."""
import ctypes as C
import gzip
import io
import os
import random
import tarfile
import urllib.request
import zipfile
import zlib

import numpy as np
import pytest

import inflate_streams as IS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from lambdipy_b200 import _native as N
    with N.Context(0) as c:
        yield c


def run(ctx, body):
    """raw DEFLATE body through lb2_inflate_run / read -> (bytes, stats)"""
    from lambdipy_b200 import _native as N
    d = C.c_void_p()
    ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    try:
        n, st = C.c_uint64(), N.InflateStats()
        buf = C.create_string_buffer(body, max(len(body), 1))
        ctx.check(ctx.lib.lb2_inflate_run(d, buf, len(body), C.byref(n), C.byref(st)))
        out = C.create_string_buffer(max(n.value, 1))
        ctx.check(ctx.lib.lb2_inflate_read(d, out, n.value))
        return out.raw[:n.value], st.as_dict()
    finally:
        ctx.lib.lb2_inflate_destroy(d)


def gz_file(tmp_path, data, name="t.gz", **kw):
    p = tmp_path / name
    p.write_bytes(gzip.compress(data, **kw))
    return str(p)


@pytest.mark.parametrize("span_kb", [None, "1", "8"])
def test_stream_matrix(ctx, monkeypatch, span_kb):
    if span_kb:
        monkeypatch.setenv("LB2_INFLATE_SPAN_KB", span_kb)
    else:
        monkeypatch.delenv("LB2_INFLATE_SPAN_KB", raising=False)
    for name, body, data in IS.matrix(1 << 20):
        got, st = run(ctx, body)
        assert got == data, name
        assert st["in_bytes"] == len(body) and st["crc32"] == zlib.crc32(data), (name, st)


@pytest.mark.parametrize("span_kb", [None, "2"])
def test_own_writer_output_and_zeros(ctx, tmp_path, monkeypatch, span_kb):
    from lambdipy_b200.tarball import GpuGzipFile, gunzip
    if span_kb:
        monkeypatch.setenv("LB2_INFLATE_SPAN_KB", span_kb)
    data = IS.so_bytes(6 << 20) + IS.text(1 << 20)
    p = str(tmp_path / "own.gz")
    with GpuGzipFile(p, ctx=ctx, piece_bytes=4 << 20) as g:
        g.write(data)
    assert gunzip(p, ctx) == data
    zeros = bytes(256 << 20)
    body = zlib.compress(zeros, 9)[2:-4]
    got, st = run(ctx, body)
    assert got == zeros and st["out_bytes"] == len(zeros)


@pytest.mark.parametrize("n", [0, 1, 2, 131071, 131072, 131073])
def test_sizes(ctx, tmp_path, n):
    from lambdipy_b200.tarball import gunzip
    data = IS.text(n, seed=n)
    assert gunzip(gz_file(tmp_path, data), ctx) == data


def _inner_archive(tmp_path):
    """a tar holding .gz and zip-deflated .whl members of several MB"""
    so = IS.so_bytes(12 << 20)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for k in range(3):
            inner = gzip.compress(so[k * (4 << 20):(k + 1) * (4 << 20)], 6)
            ti = tarfile.TarInfo("pkg/part%d.gz" % k)
            ti.size = len(inner)
            tar.addfile(ti, io.BytesIO(inner))
            zb = io.BytesIO()
            with zipfile.ZipFile(zb, "w", zipfile.ZIP_DEFLATED) as z:
                z.writestr("lib%d.so" % k, so[k * (3 << 20):(k + 1) * (3 << 20)])
            ti = tarfile.TarInfo("pkg/w%d.whl" % k)
            ti.size = len(zb.getvalue())
            tar.addfile(ti, io.BytesIO(zb.getvalue()))
    return buf.getvalue()


@pytest.mark.parametrize("level", [0, 9])
def test_speculation_under_attack(ctx, tmp_path, level):
    from lambdipy_b200.tarball import gunzip
    data = _inner_archive(tmp_path)
    body = IS.deflate(data, level)
    got, st = run(ctx, body)
    assert got == data
    if level == 0:
        assert st["n_rejected"] > 0, st
    assert gunzip(gz_file(tmp_path, data, compresslevel=level), ctx) == data


def test_framing_on_gpu_path(ctx, tmp_path):
    from lambdipy_b200.tarball import gunzip
    import test_untar_host as H
    parts = [IS.text(300 << 10), b"", IS.so_bytes(500 << 10)]
    raw = H._member(parts[0], 0x1F & ~0x01) + H._member(parts[1]) + b"\0" * 4 + \
        H._member(parts[2], H.tarball.FEXTRA | H.tarball.FCOMMENT | H.tarball.FHCRC, level=9) + b"\0" * 16
    p = tmp_path / "multi.gz"
    p.write_bytes(raw)
    assert gunzip(str(p), ctx) == b"".join(parts) == gzip.decompress(raw)


def test_corrupt_input(ctx, tmp_path):
    from lambdipy_b200.tarball import gunzip
    data = IS.so_bytes(2 << 20)
    good = gzip.compress(data, 9)
    cases = {"truncated": good[:len(good) // 2], "trailer_cut": good[:-3]}
    bad = bytearray(good); bad[-8] ^= 1; cases["crc"] = bytes(bad)
    bad = bytearray(good); bad[-1] ^= 1; cases["isize"] = bytes(bad)
    rng = random.Random(3)
    for k in range(6):
        bad = bytearray(good)
        bad[rng.randrange(20, len(good) - 8)] ^= 1 << rng.randrange(8)
        cases["flip%d" % k] = bytes(bad)
    for name, raw in cases.items():
        p = tmp_path / (name + ".gz")
        p.write_bytes(raw)
        try:
            got = gunzip(str(p), ctx)
        except (gzip.BadGzipFile, EOFError):
            continue
        assert got == gzip.decompress(raw), name   # never success with other bytes


def _tree(root, dir_mtime=True):
    """name -> (mode, mtime, link target or contents); dir_mtime=False leaves out directory mtimes, which are the
    time of extraction when extractall stops before it sets them"""
    out = {}
    for dp, dns, fns in os.walk(root):
        for n in dns + fns:
            p = os.path.join(dp, n)
            st = os.lstat(p)
            rec = (oct(st.st_mode), int(st.st_mtime) if dir_mtime or not os.path.isdir(p) else None)
            if os.path.islink(p):
                rec += (os.readlink(p),)
            elif os.path.isfile(p):
                with open(p, "rb") as f:
                    rec += (f.read(),)
            out[os.path.relpath(p, root)] = rec
    return out


def _reference_prepare(url, download_filename, package_directory):
    """the reference's prepare_tarfile (lambdipy/project_build.py:98-102)"""
    urllib.request.urlretrieve(url, download_filename)
    tar = tarfile.open(download_filename, "r:gz")
    tar.extractall(package_directory)
    tar.close()


def test_prepare_tarfile_corrupt_matches_reference(ctx, tmp_path, monkeypatch):
    from lambdipy_b200 import tarball
    site = os.path.dirname(os.path.dirname(np.__file__))
    src = tmp_path / "t.tar.gz"
    with tarfile.open(src, "w:gz") as tar:
        tar.add(os.path.join(site, "numpy", "_core"), arcname="_core")
    raw = src.read_bytes()
    bad = tmp_path / "bad.tar.gz"
    monkeypatch.setattr(tarball.urllib.request, "urlretrieve", lambda url, fn: open(fn, "wb").write(bad.read_bytes()))
    monkeypatch.setattr(tarball, "_default_context", lambda: (ctx, False))
    for at in (len(raw) // 3, len(raw) * 2 // 3, len(raw) - 6):
        raw = bytearray(src.read_bytes())
        raw[at] ^= 0x10
        bad.write_bytes(bytes(raw))
        errs = []
        for fn, d in ((tarball.prepare_tarfile, "mine"), (_reference_prepare, "ref")):
            try:   # tarfile stops at the end-of-archive blocks, so a flip may go unnoticed by both
                fn("https://example.invalid/t.tar.gz", str(tmp_path / ("dl_" + d)), str(tmp_path / ("%s%d" % (d, at))))
                errs.append(None)
            except Exception as e:
                errs.append(type(e))
        assert errs[0] is errs[1], (at, errs)
        assert _tree(tmp_path / ("mine%d" % at), False) == _tree(tmp_path / ("ref%d" % at), False), at


@pytest.mark.parametrize("writer", ["tarfile", "gzip_tarball"])
def test_tarball_parity_and_parallelism(ctx, tmp_path, monkeypatch, writer):
    from lambdipy_b200 import tarball
    monkeypatch.delenv("LB2_INFLATE_SPAN_KB", raising=False)
    site = os.path.dirname(os.path.dirname(np.__file__))
    srcs = [os.path.join(site, d) for d in ("numpy", "numpy.libs", "scipy", "scipy.libs") if os.path.exists(os.path.join(site, d))]
    path = str(tmp_path / "ns.tar.gz")
    if writer == "tarfile":
        with tarfile.open(path, "w:gz") as tar:
            for p in srcs:
                tar.add(p, arcname=os.path.basename(p))
    else:
        tarball.gzip_tarball(srcs, path, ctx=ctx)
    tarball.extract_tarball(path, str(tmp_path / "mine"), ctx)
    monkeypatch.setattr(tarball.urllib.request, "urlretrieve", lambda url, fn: None)
    monkeypatch.setattr(tarball, "_default_context", lambda: (ctx, False))
    tarball.prepare_tarfile("https://example.invalid/ns.tar.gz", path, str(tmp_path / "mirror"))
    _reference_prepare(None, path, str(tmp_path / "ref"))
    ref = _tree(tmp_path / "ref")
    assert _tree(tmp_path / "mine") == ref and _tree(tmp_path / "mirror") == ref
    if writer == "tarfile":   # zlib level 9, no flush points: the spans still decode in parallel
        raw = open(path, "rb").read()
        body = raw[raw.index(b"\0", 10) + 1:]
        _, st = run(ctx, body)
        _, st2 = run(ctx, body)
        assert st["n_spans"] == st2["n_spans"] and st["n_rejected"] == st2["n_rejected"]
        nominal = (len(body) + (128 << 10) - 1) // (128 << 10)
        assert (nominal - st["n_absorbed"] - st["n_rejected"]) >= 0.9 * nominal, st
