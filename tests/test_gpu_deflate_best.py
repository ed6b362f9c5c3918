"""GPU tests of the thorough DEFLATE mode (LB2_DEFLATE_BEST: the optimal parse after the greedy one, csrc/deflate.cu
and csrc/deflate_parse.cuh) in the gzip and the zip writer.

* Every best-mode gzip stream and zip member inflates with zlib to its input and ends where it should, with the right
  CRC-32; deflate_ref parses it with complete codes within 15 / 7 bits, BFINAL only in the closing block, and every
  chunk in the block type that is cheapest by the kernel's byte formula, with the kernel's code for its tokens.
* Chunk by chunk (gzip) and member by member (zip), best mode is never larger than the default mode.
* On numpy + scipy: best is strictly smaller than the default with n_opt_chunks > 0, the tar stream's body is no
  larger than zlib level 9's, and the tree's zip is no larger than make_archive's.
* Edge cases: empty files (03 00), 10 MB of random bytes (stored, within the bound), 256 MB of zeros, a stream and a
  file continued across pieces, a match at distance exactly 32 768; two runs give the same bytes; unknown flags are
  refused.
"""
import ctypes as C
import os
import shutil
import tarfile
import zipfile
import zlib

import numpy as np
import pytest

from test_gpu_deflate_edges import analyse, check_pricing_and_optimality, check_dist_32768, _text, _rand
from test_gpu_zip import check_zip, raw_bodies
from test_zip_host import edge_tree

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))
BEST = 1


def gzip_pieces(ctx, pieces, flags):
    """Raw API: DEFLATE the concatenation of `pieces` with the writer's `flags`, one submission each (two in flight).
    Returns (gzip file bytes, crc32, isize, stats)."""
    from lambdipy_b200 import _native as N
    from lambdipy_b200.tarball import gzip_header
    lib = ctx.lib
    g = C.c_void_p()
    ctx.check(lib.lb2_gzip_create(ctx.h, flags, C.byref(g)))
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


def best_and_default(ctx, pieces, parse=True):
    """Both modes on the same pieces; checks each stream, and best <= default chunk by chunk.  Returns
    (best chunks, default chunks, best stats, default stats), chunks as analyse() gives them (None without parse)."""
    whole = b"".join(pieces)
    out = []
    for flags in (BEST, 0):
        gz, crc, isize, st = gzip_pieces(ctx, pieces, flags)
        assert crc == zlib.crc32(whole) and isize == len(whole)
        assert zlib.decompress(gz, wbits=31) == whole
        assert (st["n_opt_chunks"] > 0) <= (flags == BEST)
        chunks = None
        if parse:
            chunks = analyse(gz, pieces, st)
            check_pricing_and_optimality(chunks)
        out.append((gz, chunks, st))
    (gz_b, ch_b, st_b), (gz_d, ch_d, st_d) = out
    assert len(gz_b) <= len(gz_d)
    if parse:
        assert len(ch_b) == len(ch_d)
        assert all(b[3] <= d[3] for b, d in zip(ch_b, ch_d)), [(b[3], d[3]) for b, d in zip(ch_b, ch_d)]
    return ch_b, ch_d, st_b, st_d, gz_b, gz_d


def test_structured_inputs(gpu_ctx):
    text = _text(300_000, 1)
    periodic = bytes((i * 37) & 0xFF for i in range(13)) * 20_000
    mixed = _rand(50_000, 2) + text[:100_000] + b"\0" * 70_000 + _rand(50_000, 2)
    for pieces in ([text], [periodic], [mixed], [text[:100_003], text[100_003:]], [b"abc"], [text[:65536 * 2]]):
        ch_b, ch_d, st_b, _, _, _ = best_and_default(gpu_ctx, pieces)
        assert st_b["n_opt_chunks"] == sum(b[3] < d[3] for b, d in zip(ch_b, ch_d))
    _, _, st_b, st_d, gz_b, gz_d = best_and_default(gpu_ctx, [text])
    assert st_b["n_opt_chunks"] > 0 and len(gz_b) < len(gz_d)


def test_real_shared_objects(gpu_ctx):
    files = sorted(os.path.join(dp, f) for dp, _, fs in os.walk(os.path.join(SITE, "numpy")) for f in fs if f.endswith(".so"))
    data = b"".join(open(f, "rb").read() for f in files)[:12 << 20]
    _, _, st_b, st_d, gz_b, gz_d = best_and_default(gpu_ctx, [data[:5 << 20], data[5 << 20:]])
    assert st_b["n_opt_chunks"] > 0 and len(gz_b) < len(gz_d)


def test_incompressible_stays_stored(gpu_ctx):
    from lambdipy_b200 import _native as N
    data = _rand(10 << 20, 3)
    ch_b, _, st_b, _, gz_b, _ = best_and_default(gpu_ctx, [data], parse=False)
    assert st_b["n_stored_chunks"] == st_b["n_chunks"] == 160 and st_b["n_opt_chunks"] == 0
    assert len(gz_b) - 20 <= N.gzip_bound(len(data)) + 2


def test_zeros_256mb(gpu_ctx):
    data = bytes(256 << 20)
    _, _, st_b, st_d, gz_b, gz_d = best_and_default(gpu_ctx, [data[i:i + (64 << 20)] for i in range(0, len(data), 64 << 20)],
                                                    parse=False)
    assert len(gz_b) <= len(gz_d)


def test_distance_32768(gpu_ctx):
    r = _rand(32768, 7)
    data = r + r[:20000]
    for pieces in ([data], [data[:32768], data[32768:]]):
        ch_b, _, _, _, _, _ = best_and_default(gpu_ctx, pieces)
        check_dist_32768(ch_b)


def test_deterministic(gpu_ctx):
    data = _text(200_000, 4) + _rand(30_000, 4) + _text(150_000, 5)
    a = gzip_pieces(gpu_ctx, [data], BEST)[0]
    b = gzip_pieces(gpu_ctx, [data], BEST)[0]
    assert a == b


def test_unknown_flags_refused(gpu_ctx):
    from lambdipy_b200 import _native as N
    lib = gpu_ctx.lib
    h = C.c_void_p()
    assert lib.lb2_gzip_create(gpu_ctx.h, 2, C.byref(h)) == N.LB2_E_ARG
    assert lib.lb2_zip_create(gpu_ctx.h, 3, C.byref(h)) == N.LB2_E_ARG


# ---------------------------------------------------------------------------------------------- zip
def zip_both(ctx, root, tmp, **kw):
    from lambdipy_b200 import zipfile_gpu
    res = []
    for level in (9, None):
        path = os.path.join(tmp, "best.zip" if level else "default.zip")
        st = zipfile_gpu.zip_tree(root, path, ctx=ctx, compresslevel=level, **kw)
        res.append((path, st))
    (pb, sb), (pd, sd) = res
    sizes_b = {zi.filename: zi.compress_size for zi in zipfile.ZipFile(pb).infolist()}
    sizes_d = {zi.filename: zi.compress_size for zi in zipfile.ZipFile(pd).infolist()}
    assert sizes_b.keys() == sizes_d.keys()
    assert all(sizes_b[k] <= sizes_d[k] for k in sizes_b)
    return pb, sb, pd, sd


@pytest.mark.parametrize("piece_bytes", [96 << 10, 64 << 20])
def test_zip_edge_tree(gpu_ctx, tmp_path, piece_bytes):
    root = edge_tree(str(tmp_path / "tree"))
    (tmp_path / "tree" / "pkg" / "text.txt").write_bytes(_text(200_000, 9))     # continued across 96 KB pieces
    (tmp_path / "tree" / "pkg" / "rnd.bin").write_bytes(_rand(10 << 20, 5))
    pb, sb, pd, sd = zip_both(gpu_ctx, root, str(tmp_path), piece_bytes=piece_bytes)
    check_zip(pb, root, str(tmp_path), parse=True)
    assert sb["n_opt_chunks"] > 0
    for zi, body in raw_bodies(pb):
        if not zi.is_dir() and zi.file_size == 0:
            assert body == b"\x03\x00"
    a = open(pb, "rb").read()
    zip_both(gpu_ctx, root, str(tmp_path), piece_bytes=piece_bytes)
    assert open(pb, "rb").read() == a


def _numpy_scipy_tree(root):
    for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
        p = os.path.join(SITE, d)
        if os.path.exists(p):
            shutil.copytree(p, os.path.join(root, d), symlinks=True)


def test_numpy_scipy_zip(gpu_ctx, tmp_path):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    root = str(tmp_path / "tree")
    _numpy_scipy_tree(root)
    pb, sb, pd, sd = zip_both(gpu_ctx, root, str(tmp_path))
    check_zip(pb, root, str(tmp_path))
    ref = shutil.make_archive(str(tmp_path / "ref"), "zip", root)
    print("numpy+scipy zip: best %d, default %d, make_archive %d bytes; %d opt chunks"
          % (os.path.getsize(pb), os.path.getsize(pd), os.path.getsize(ref), sb["n_opt_chunks"]))
    assert sb["n_opt_chunks"] > 0 and sb["out_bytes"] < sd["out_bytes"]
    assert os.path.getsize(pb) <= os.path.getsize(ref)


def test_numpy_scipy_tar_against_zlib9(gpu_ctx):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    import io
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
            p = os.path.join(SITE, d)
            if os.path.exists(p):
                tar.add(p, arcname=d)
    data = buf.getvalue()
    piece = 64 << 20
    _, _, st_b, st_d, gz_b, gz_d = best_and_default(gpu_ctx, [data[i:i + piece] for i in range(0, len(data), piece)],
                                                    parse=False)
    z = zlib.compressobj(9, zlib.DEFLATED, -15)
    z9 = len(z.compress(data) + z.flush())
    body_b = len(gz_b) - 20  # the 12-byte header of gzip_header("t.gz") and the 8-byte trailer
    print("numpy+scipy tar %d bytes: best body %d, default %d, zlib-9 %d; %d of %d chunks from the optimal parse"
          % (len(data), body_b, len(gz_d) - 20, z9, st_b["n_opt_chunks"], st_b["n_chunks"]))
    assert st_b["n_opt_chunks"] > 0 and len(gz_b) < len(gz_d)
    assert body_b <= z9
