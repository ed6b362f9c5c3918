"""GPU tests of the zip writer (lb2_zip_*, csrc/deflate.cu) behind zipfile_gpu.zip_tree.

Each member body of the GPU-written zip inflates on its own (zlib.decompressobj(-15)) to exactly the file and ends
at compress_size (no window leaks across files), has the CRC-32 zlib computes, and parses with deflate_ref with BFINAL
only in its closing block.  The archive passes testzip() and its infolist equals make_archive's in everything but
compress_size and header_offset, on the edge trees of test_zip_host.py, a file repeating its predecessor, an
incompressible 10 MB file (stored blocks within LB2_GZIP_BOUND), 20 000 tiny files and the numpy + scipy tree; two
runs give the same bytes; on numpy + scipy the zip is no larger than make_archive's at compresslevel 1.
"""
import ctypes as C
import os
import shutil
import struct
import zipfile
import zlib

import numpy as np
import pytest

import deflate_ref as R
from test_zip_host import edge_tree

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))
ATTRS = ("filename", "date_time", "compress_type", "comment", "extra", "create_system", "create_version",
         "extract_version", "reserved", "flag_bits", "volume", "internal_attr", "external_attr", "CRC", "file_size")


def raw_bodies(path):
    """(ZipInfo, raw member body) of every entry, read through the local headers"""
    data = open(path, "rb").read()
    out = []
    for zi in zipfile.ZipFile(path).infolist():
        h = zi.header_offset
        assert data[h:h + 4] == zipfile.stringFileHeader
        n, m = struct.unpack_from("<HH", data, h + 26)
        start = h + 30 + n + m
        out.append((zi, data[start:start + zi.compress_size]))
    return out


def check_zip(path, root, tmp, parse=False):
    from lambdipy_b200 import _native as N
    with zipfile.ZipFile(path) as zf:
        assert zf.testzip() is None
        mine = zf.infolist()
    ref_path = shutil.make_archive(os.path.join(tmp, "ref"), "zip", root)
    with zipfile.ZipFile(ref_path) as zf:
        ref = zf.infolist()
    assert [[getattr(a, k) for k in ATTRS] for a in mine] == [[getattr(b, k) for k in ATTRS] for b in ref]
    for zi, body in raw_bodies(path):
        if zi.is_dir():
            assert zi.compress_type == zipfile.ZIP_STORED and body == b""
            continue
        want = open(os.path.join(root, zi.filename), "rb").read()
        d = zlib.decompressobj(-15)
        assert d.decompress(body) == want and d.eof and d.unused_data == b"", zi.filename
        assert zi.CRC == zlib.crc32(want)
        assert len(body) <= N.gzip_bound(len(want)) + 2
        if not want:
            assert body == b"\x03\x00"
        if parse:
            out, blocks, end = R.parse(body, keep_tokens=False)
            assert out == want and (end + 7) // 8 == len(body)
            assert [b["final"] for b in blocks] == [0] * (len(blocks) - 1) + [1]
    os.remove(ref_path)


def zip_it(ctx, root, path, **kw):
    from lambdipy_b200 import zipfile_gpu
    return zipfile_gpu.zip_tree(root, path, ctx=ctx, **kw)


@pytest.mark.parametrize("piece_bytes", [96 << 10, 64 << 20])
def test_edge_tree(gpu_ctx, tmp_path, piece_bytes):
    root = edge_tree(str(tmp_path / "tree"))
    rng = np.random.default_rng(11)
    block = rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes()
    (tmp_path / "tree" / "pkg" / "rep_a.bin").write_bytes(block)       # its successor repeats it: a match across
    (tmp_path / "tree" / "pkg" / "rep_b.bin").write_bytes(block)       # files would be cheap, and is not allowed
    out = str(tmp_path / "gpu.zip")
    st = zip_it(gpu_ctx, root, out, piece_bytes=piece_bytes)
    check_zip(out, root, str(tmp_path), parse=True)
    bodies = dict((zi.filename, b) for zi, b in raw_bodies(out))
    assert len(bodies["pkg/rep_b.bin"]) >= len(block)                  # stored again: no look-back into rep_a.bin
    assert st["files"] == sum(1 for zi, _ in raw_bodies(out) if not zi.is_dir())


def test_incompressible_is_stored(gpu_ctx, tmp_path):
    from lambdipy_b200 import _native as N
    root = tmp_path / "tree"
    root.mkdir()
    data = np.random.default_rng(5).integers(0, 256, 10 << 20, dtype=np.uint8).tobytes()
    (root / "noise.bin").write_bytes(data)
    (root / "small.txt").write_bytes(b"hello " * 100)
    out = str(tmp_path / "n.zip")
    st = zip_it(gpu_ctx, str(root), out, piece_bytes=4 << 20)
    check_zip(out, str(root), str(tmp_path))
    body = dict((zi.filename, b) for zi, b in raw_bodies(out))["noise.bin"]
    assert len(body) <= N.gzip_bound(len(data)) + 2
    assert st["n_stored_chunks"] == 160


def test_many_tiny_files(gpu_ctx, tmp_path):
    root = tmp_path / "tiny"
    for d in range(20):
        (root / ("d%02d" % d)).mkdir(parents=True)
        for i in range(1000):
            (root / ("d%02d" % d) / ("m%04d.py" % i)).write_bytes(b"x = %d\n" % (i * d) * (i % 7))
    out = str(tmp_path / "t.zip")
    st = zip_it(gpu_ctx, str(root), out)
    assert st["files"] == 20_000
    check_zip(out, str(root), str(tmp_path))


def test_deterministic(gpu_ctx, tmp_path):
    root = edge_tree(str(tmp_path / "tree"))
    a, b = str(tmp_path / "a.zip"), str(tmp_path / "b.zip")
    zip_it(gpu_ctx, root, a, piece_bytes=96 << 10)
    zip_it(gpu_ctx, root, b, piece_bytes=96 << 10)
    assert open(a, "rb").read() == open(b, "rb").read()


def _numpy_scipy(tmp_path):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    root = tmp_path / "bundle"
    for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
        if os.path.exists(os.path.join(SITE, d)):
            shutil.copytree(os.path.join(SITE, d), root / d, symlinks=True)
    return str(root)


def test_numpy_scipy_and_ratio(gpu_ctx, tmp_path):
    root = _numpy_scipy(tmp_path)
    out = str(tmp_path / "ns.zip")
    st = zip_it(gpu_ctx, root, out)
    check_zip(out, root, str(tmp_path))
    a = open(out, "rb").read()
    zip_it(gpu_ctx, root, out)
    assert open(out, "rb").read() == a                                  # deterministic on the large tree too
    ref1 = str(tmp_path / "z1.zip")
    with zipfile.ZipFile(ref1, "w", compression=zipfile.ZIP_DEFLATED, compresslevel=1) as zf:
        for path, zi in __import__("lambdipy_b200.zipfile_gpu", fromlist=["x"]).tree_entries(root):
            zf.write(path, zi.filename)
    print("numpy+scipy: %d files, %d bytes -> GPU zip %d, zlib-1 zip %d" % (st["files"], st["in_bytes"], len(a),
                                                                            os.path.getsize(ref1)))
    assert len(a) <= os.path.getsize(ref1)


def test_raw_api_errors(gpu_ctx):
    """LB2_E_ARG / LB2_E_STATE / LB2_E_CAPACITY as in the gzip writer"""
    from lambdipy_b200 import _native as N
    ctx, lib = gpu_ctx, gpu_ctx.lib
    z = C.c_void_p()
    ctx.check(lib.lb2_zip_create(ctx.h, 0, C.byref(z)))
    buf = ctx.pinned_alloc(1 << 16)
    out = ctx.pinned_alloc(1 << 17)
    try:
        C.memmove(buf, b"abc" * 1000, 3000)
        u64 = lambda *v: (C.c_uint64 * len(v))(*v)
        n, segs = C.c_uint64(), (N.ZipSegment * 4)()
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0, 8), u64(100, 100), 2, 0) == N.LB2_E_ARG      # unaligned
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0, 16), u64(100, 100), 2, 0) == N.LB2_E_ARG     # overlap
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0), u64(3001), 1, 0) == N.LB2_E_ARG             # past the piece
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0), u64(3000), 0, 0) == N.LB2_E_ARG             # no segment
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0), u64(3000), 1, 4) == N.LB2_E_ARG             # unknown flag
        assert lib.lb2_zip_submit(z, buf, 3000, u64(0), u64(3000), 1, N.ZIP_CONTINUES) == N.LB2_E_STATE
        assert lib.lb2_zip_collect(z, out, 1 << 17, C.byref(n), segs, None) == N.LB2_E_STATE
        ctx.check(lib.lb2_zip_submit(z, buf, 3000, u64(0, 1024), u64(1000, 1976), 2, N.ZIP_MORE))
        assert lib.lb2_zip_submit(z, buf, 1000, u64(0), u64(1000), 1, 0) == N.LB2_E_STATE            # open file not continued
        ctx.check(lib.lb2_zip_submit(z, buf, 1000, u64(0), u64(1000), 1, N.ZIP_CONTINUES))
        assert lib.lb2_zip_submit(z, buf, 1000, u64(0), u64(1000), 1, 0) == N.LB2_E_STATE            # two in flight
        assert lib.lb2_zip_collect(z, out, 1, C.byref(n), segs, None) == N.LB2_E_CAPACITY
        need = n.value
        ctx.check(lib.lb2_zip_collect(z, out, 1 << 17, C.byref(n), segs, None))
        assert n.value == need
        first = C.string_at(out, n.value)
        s0, s1 = segs[0], segs[1]
        data = b"abc" * 1000
        assert s0.ended and not s1.ended and s0.crc32 == zlib.crc32(data[:1000]) and s1.crc32 == zlib.crc32(data[1024:3000])
        body0 = first[s0.out_off:s0.out_off + s0.out_len]
        assert zlib.decompressobj(-15).decompress(body0) == data[:1000]
        ctx.check(lib.lb2_zip_collect(z, out, 1 << 17, C.byref(n), segs, None))
        tail = segs[0]
        assert tail.ended and tail.crc32 == zlib.crc32(data[:1000], zlib.crc32(data[1024:3000]))
        body1 = first[s1.out_off:s1.out_off + s1.out_len] + C.string_at(out + tail.out_off, tail.out_len)
        d = zlib.decompressobj(-15)
        assert d.decompress(body1) == data[1024:3000] + data[:1000] and d.eof
    finally:
        lib.lb2_zip_destroy(z)
        ctx.pinned_free(buf)
        ctx.pinned_free(out)


def test_incompressible_file_across_pieces_within_bound(gpu_ctx, tmp_path):
    """an incompressible file that starts mid-piece and goes on over several pieces: stored blocks within
    LB2_GZIP_BOUND of its size, as if it had been deflated whole"""
    from lambdipy_b200 import _native as N
    root = tmp_path / "tree"
    (root / "a").mkdir(parents=True)                    # os.walk visits a/ before b/
    (root / "b").mkdir()
    (root / "a" / "pad.txt").write_bytes(b"padding " * 6250)
    data = np.random.default_rng(9).integers(0, 256, 300_001, dtype=np.uint8).tobytes()
    (root / "b" / "noise.bin").write_bytes(data)
    out = str(tmp_path / "x.zip")
    st = zip_it(gpu_ctx, str(root), out, piece_bytes=96 << 10)
    check_zip(out, str(root), str(tmp_path))
    body = dict((zi.filename, b) for zi, b in raw_bodies(out))["b/noise.bin"]
    assert len(body) <= N.gzip_bound(len(data)) + 2
    assert st["n_stored_chunks"] == (len(data) + 65535) // 65536
