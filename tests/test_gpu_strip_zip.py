"""GPU checks of strip_zip (zipfile_gpu.py) and of the two entry points under it (lb2_zip_submit_device,
lb2_unzip_device_output in csrc/api.cu, the gather kernel in csrc/deflate.cu).

Parity: `extractall(src)` followed by the reference's `find -name "*.so" | xargs strip` gives the tree
`extractall(strip_zip(src))` gives, file by file, on gcc-built variants, the numpy + scipy tree and the golden files
(whose outputs also equal the recorded GNU strip results); every rewritten body is a raw DEFLATE stream of its own that
zlib and the bit-level reference accept; a planner-refused object takes the host strip; members larger than a piece and
members on the span pipeline round-trip; level 9 is never larger; runs are deterministic; only compressed bytes cross
the bus; the device submit gives the bytes of the host submit, odd source addresses included, and refuses what it
refuses."""
import ctypes as C
import glob
import os
import shutil
import subprocess
import zipfile
import zlib

import numpy as np
import pytest

import deflate_ref
from test_strip_zip_host import local_header
from test_unzip_host import tree

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LIMIT_CLASS = "c_many_sections"   # more sections than the planner holds: LB2_ST_PLANNER_LIMIT


def reference_line(root):
    """the reference's strip line on an extracted tree; its exit status"""
    return subprocess.run('find %s/ -name "*.so" | xargs strip' % root, shell=True, capture_output=True).returncode


def zip_of(path, files, compression=zipfile.ZIP_DEFLATED):
    """files: {member name: path or bytes}"""
    with zipfile.ZipFile(path, "w", compression) as zf:
        for name, src in files.items():
            if isinstance(src, bytes):
                zf.writestr(name, src)
            else:
                zf.write(src, name)
    return path


def check_parity(ctx, src, tmp, rc=0, **kw):
    from lambdipy_b200 import zipfile_gpu as Z
    want, got, dst = os.path.join(tmp, "want"), os.path.join(tmp, "got"), os.path.join(tmp, "stripped.zip")
    for d in (want, got):
        shutil.rmtree(d, ignore_errors=True)
    with zipfile.ZipFile(src) as zf:
        zf.extractall(want)
    assert reference_line(want) == rc
    st = Z.strip_zip(src, dst, ctx=ctx, **kw)
    with zipfile.ZipFile(dst) as zf:
        assert zf.testzip() is None
        zf.extractall(got)
    assert Z.testzip(dst, ctx=ctx) is None
    assert tree(got) == tree(want)
    for d in (want, got):
        shutil.rmtree(d)
    return st, dst


def check_bodies(src, dst, parse_below=0):
    """every rewritten member is a raw DEFLATE stream of its own, ending at compress_size"""
    from lambdipy_b200 import zipfile_gpu as Z
    n = 0
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        for za, zb in zip(a.filelist, b.filelist):
            assert za.filename == zb.filename
            body = local_header(dst, zb)[1]
            if not Z.selected_for_strip(za):
                assert body == local_header(src, za)[1] and zb.CRC == za.CRC
                continue
            d = zlib.decompressobj(-15)
            data = d.decompress(body)
            assert d.eof and not d.unused_data and zb.compress_type == zipfile.ZIP_DEFLATED
            assert len(data) == zb.file_size and zlib.crc32(data) == zb.CRC
            if len(body) < parse_below:
                out, blocks, end = deflate_ref.parse(body, keep_tokens=False)
                assert bytes(out) == data and (end + 7) // 8 == len(body) and blocks[-1]["final"]
            n += 1
    return n


def residency(st, src, dst, fallback_in=0, fallback_out=0):
    """only compressed bodies cross the bus, plus what the host strip of the fallback members takes and returns"""
    from lambdipy_b200 import zipfile_gpu as Z
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        up = sum(z.compress_size for z in a.filelist if Z.selected_for_strip(z))
        down = sum(zb.compress_size for za, zb in zip(a.filelist, b.filelist) if Z.selected_for_strip(za))
    assert st["uploaded_bytes"] == up + fallback_out and st["downloaded_bytes"] == down + fallback_in


def test_variants_and_text_files(gpu_ctx, variants, tmp_path):
    files = {"README.txt": b"a bundle built elsewhere\n" * 100, "pkg/__init__.py": b""}
    for k in sorted(variants):
        if k != LIMIT_CLASS:
            files["pkg/%s.so" % k] = variants[k]
    files["pkg/libcopy.so.1"] = variants["c_g"]            # `find -name "*.so"` does not match it
    src = zip_of(str(tmp_path / "v.zip"), files)
    st, dst = check_parity(gpu_ctx, src, str(tmp_path))
    assert st["gpu"] == st["selected"] == len(variants) - 1 and st["fallback"] == 0 and st["skipped"] == 0
    assert st["out_bytes"] < st["in_bytes"] and st["strip"]["plan_ms"] > 0 and st["deflate"]["kernel_ms"] > 0
    assert check_bodies(src, dst, parse_below=1 << 16) == st["selected"]
    residency(st, src, dst)
    with zipfile.ZipFile(src) as a, zipfile.ZipFile(dst) as b:
        assert b.read("pkg/libcopy.so.1") == a.read("pkg/libcopy.so.1")
    # stored members and the thorough encoder: never larger, the same files
    stored = zip_of(str(tmp_path / "stored.zip"), files, zipfile.ZIP_STORED)
    st9, dst9 = check_parity(gpu_ctx, stored, str(tmp_path / "nine"), compresslevel=9)
    with zipfile.ZipFile(dst) as a, zipfile.ZipFile(dst9) as b:
        for name in files:
            if name.endswith(".so"):
                assert b.getinfo(name).compress_size <= a.getinfo(name).compress_size, name
                assert b.getinfo(name).compress_type == zipfile.ZIP_DEFLATED
    assert st9["deflate"]["n_opt_chunks"] > 0
    first = open(dst9, "rb").read()
    from lambdipy_b200 import zipfile_gpu as Z
    Z.strip_zip(stored, dst9, ctx=gpu_ctx, compresslevel=9)
    assert open(dst9, "rb").read() == first
    first = open(dst, "rb").read()
    Z.strip_zip(src, dst, ctx=gpu_ctx)
    assert open(dst, "rb").read() == first


def test_numpy_scipy(gpu_ctx, tmp_path):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    root = tmp_path / "bundle"
    for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
        if os.path.exists(os.path.join(SITE, d)):
            shutil.copytree(os.path.join(SITE, d), root / d, symlinks=True)
    src = shutil.make_archive(str(tmp_path / "ns"), "zip", str(root))
    shutil.rmtree(root)
    st, dst = check_parity(gpu_ctx, src, str(tmp_path))
    assert st["gpu"] + st["fallback"] == st["selected"] > 50 and st["gpu"] > 0.9 * st["selected"]
    assert st["unzip"]["n_large"] > 0                     # members of more than one span take the span pipeline
    assert check_bodies(src, dst) == st["selected"]
    if not st["fallback"]:
        residency(st, src, dst)
    print("numpy+scipy strip_zip:", {k: st[k] for k in ("members", "selected", "gpu", "fallback", "in_bytes", "out_bytes",
                                                        "src_zip_bytes", "zip_bytes", "kernel_ms")})


def test_golden_files(gpu_ctx, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    ins = sorted(glob.glob(os.path.join(GOLDEN, "*.in.bin")))
    assert ins
    src = zip_of(str(tmp_path / "g.zip"), {"golden/%s.so" % os.path.basename(p)[:-7]: p for p in ins})
    st, dst = check_parity(gpu_ctx, src, str(tmp_path))
    assert st["gpu"] == len(ins)
    with zipfile.ZipFile(dst) as zf:
        for p in ins:
            gnu = p[:-7] + ".gnu.bin"
            assert zf.read("golden/%s.so" % os.path.basename(p)[:-7]) == open(gnu, "rb").read(), p


def test_planner_refused_member_takes_the_host_strip(gpu_ctx, variants, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    src = zip_of(str(tmp_path / "f.zip"), {"a/g.so": variants["c_g"], "a/many.so": variants[LIMIT_CLASS],
                                           "a/notes.txt": b"text\n"})
    st, dst = check_parity(gpu_ctx, src, str(tmp_path))
    assert (st["selected"], st["gpu"], st["fallback"]) == (2, 1, 1)
    with zipfile.ZipFile(dst) as zf:
        residency(st, src, dst, fallback_in=os.path.getsize(variants[LIMIT_CLASS]), fallback_out=len(zf.read("a/many.so")))
    with pytest.raises(Z.StripFailed, match="a/many.so"):
        Z.strip_zip(src, str(tmp_path / "no.zip"), ctx=gpu_ctx, fallback_host_strip=False)
    assert not os.path.exists(tmp_path / "no.zip")
    # a file strip refuses: the reference's line exits 123 and strips the rest; here the call fails, or keeps the member
    bad = zip_of(str(tmp_path / "t.zip"), {"a/g.so": variants["c_g"], "a/text.so": b"this is not an ELF file\n" * 10})
    with pytest.raises(Z.StripFailed, match="a/text.so"):
        Z.strip_zip(bad, str(tmp_path / "no.zip"), ctx=gpu_ctx)
    assert sorted(os.listdir(tmp_path)) == ["f.zip", "stripped.zip", "t.zip"]
    st, _ = check_parity(gpu_ctx, bad, str(tmp_path), rc=123, tolerate_non_elf=True)
    assert (st["gpu"], st["skipped"]) == (1, 1)


def test_members_larger_than_a_piece(gpu_ctx, tmp_path):
    """small pieces: a shared object cut over several pieces, with LB2_ZIP_MORE / LB2_ZIP_CONTINUES between them"""
    libs = sorted(glob.glob(os.path.join(SITE, "numpy", "**", "*.so"), recursive=True) +
                  glob.glob(os.path.join(SITE, "numpy.libs", "*.so*")), key=os.path.getsize)
    big = [p for p in libs if os.path.getsize(p) > (2 << 20)]
    assert big
    files = {"n/%d_%s.so" % (i, os.path.basename(p).split(".")[0]): p for i, p in enumerate(libs[:3] + big[:2])}
    src = zip_of(str(tmp_path / "p.zip"), files)
    assert max(z.compress_size for z in zipfile.ZipFile(src).filelist) > (128 << 10)
    st, dst = check_parity(gpu_ctx, src, str(tmp_path), piece_bytes=256 << 10)
    assert st["gpu"] + st["fallback"] == len(files) and st["unzip"]["n_large"] > 0
    check_bodies(src, dst)
    whole, _ = check_parity(gpu_ctx, src, str(tmp_path / "whole"))
    assert whole["zip_bytes"] == st["zip_bytes"]          # cut at chunk multiples: the bytes of the file deflated whole


def test_bad_member_raises(gpu_ctx, variants, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    from test_unzip_host import corrupt
    good = tmp_path / "good.zip"
    zip_of(str(good), {"m/a.so": variants["c_g"], "m/b.so": variants["cxx_g"]})
    for what in ("crc", "body"):
        bad = corrupt(good, tmp_path / ("bad_%s.zip" % what), "m/b.so", what)
        with pytest.raises(Z.BadZipMember, match="m/b.so"):
            Z.strip_zip(str(bad), str(tmp_path / "out.zip"), ctx=gpu_ctx)
        assert not os.path.exists(tmp_path / "out.zip")


def _collect(ctx, z, cap, ns):
    from lambdipy_b200 import _native as N
    out, n, segs = C.create_string_buffer(cap), C.c_uint64(), (N.ZipSegment * ns)()
    ctx.check(ctx.lib.lb2_zip_collect(z, out, cap, C.byref(n), segs, None))
    return out.raw[:n.value], [(s.out_off, s.out_len, s.crc32, s.ended) for s in segs]


@pytest.mark.parametrize("level", [None, 9])
def test_device_submit_equals_host_submit(gpu_ctx, level):
    from lambdipy_b200 import _native as N
    lib, rng = gpu_ctx.lib, np.random.default_rng(0x51DE)
    lens = [0, 1, 15, 16, 17, 4097, 65536, 65537, 200_001, 16384, 16385, 3]
    datas = [bytes(rng.integers(0, 24, n, dtype=np.uint8)) for n in lens]
    big = bytes(rng.integers(0, 12, 300_000, dtype=np.uint8))       # continued over two pieces, cut at 128 KB
    def host_piece(ds):                                             # segments at multiples of 16 of one buffer
        off, buf = [], bytearray()
        for d in ds:
            buf += bytes(-len(buf) % 16)
            off.append(len(buf))
            buf += d
        return bytes(buf), off
    # on the device: the same bytes back to back with one byte between them, so most addresses are odd
    arena = b"\xEE" * 3 + b"\xEE".join(datas + [big]) + b"\xEE" * 64
    d_arena = gpu_ctx.dev_alloc(len(arena))
    gpu_ctx.h2d(d_arena, arena, len(arena))
    addr, pos = [], 3
    for d in datas + [big]:
        addr.append(d_arena + pos)
        pos += len(d) + 1
    assert any(a % 16 for a in addr) and len({a % 16 for a in addr}) > 4
    pieces = [(datas + [big[:131072]], N.ZIP_MORE), ([big[131072:]] + datas[:4], N.ZIP_CONTINUES)]
    results, keep = [], []   # keep: the host pieces stay alive until they are collected
    try:
        for device in (False, True):
            z = C.c_void_p()
            gpu_ctx.check(lib.lb2_zip_create(gpu_ctx.h, N.deflate_flags(level), C.byref(z)))
            try:
                got = []
                for k, (ds, flags) in enumerate(pieces):
                    if device:
                        src = (N.ZipSource * len(ds))()
                        starts = addr[:len(datas)] + [addr[-1]] if k == 0 else [addr[-1] + 131072] + addr[:4]
                        for i, d in enumerate(ds):
                            src[i].d_ptr, src[i].len = starts[i], len(d)
                        gpu_ctx.check(lib.lb2_zip_submit_device(z, src, len(ds), flags))
                    else:
                        buf, off = host_piece(ds)
                        keep.append(buf)
                        gpu_ctx.check(lib.lb2_zip_submit(z, buf, len(buf), (C.c_uint64 * len(ds))(*off),
                                                         (C.c_uint64 * len(ds))(*[len(d) for d in ds]), len(ds), flags))
                for ds, _ in pieces:
                    got.append(_collect(gpu_ctx, z, N.zip_bound(1 << 20, 32), len(ds)))
                results.append(got)
            finally:
                lib.lb2_zip_destroy(z)
    finally:
        gpu_ctx.dev_free(d_arena)
    assert results[0] == results[1]
    body, segs = results[1][0]
    for d, (off, n, crc, ended) in list(zip(datas, segs)):
        assert ended and crc == zlib.crc32(d) and zlib.decompressobj(-15).decompress(body[off:off + n]) == d
    body2, segs2 = results[1][1]
    assert not segs[-1][3] and segs2[0][3] and segs2[0][2] == zlib.crc32(big)
    whole = body[segs[-1][0]:segs[-1][0] + segs[-1][1]] + body2[segs2[0][0]:segs2[0][0] + segs2[0][1]]
    assert zlib.decompressobj(-15).decompress(whole) == big


def test_raw_api_errors(gpu_ctx):
    from lambdipy_b200 import _native as N
    lib = gpu_ctx.lib
    u, d_out, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
    gpu_ctx.check(lib.lb2_unzip_create(gpu_ctx.h, 0, C.byref(u)))
    try:
        assert lib.lb2_unzip_device_output(u, C.byref(d_out), C.byref(n)) == N.LB2_E_STATE   # before any run
        assert lib.lb2_unzip_device_output(u, None, C.byref(n)) == N.LB2_E_ARG
        body = zlib.compress(b"hello, device", 6)[2:-4]
        buf = (C.c_uint8 * 64)(*body)
        m, res, out_n = (N.UnzipMember * 1)(), (N.UnzipResult * 1)(), C.c_uint64()
        m[0].body_off, m[0].body_len, m[0].size, m[0].crc32, m[0].method = 0, len(body), 13, zlib.crc32(b"hello, device"), 8
        gpu_ctx.check(lib.lb2_unzip_run(u, buf, 64, m, 1, C.byref(out_n), res, None))
        assert res[0].status == 0
        gpu_ctx.check(lib.lb2_unzip_device_output(u, C.byref(d_out), C.byref(n)))
        assert n.value == out_n.value == 16 and d_out.value % 256 == 0
        back = C.create_string_buffer(13)
        gpu_ctx.d2h(back, d_out.value + res[0].out_off, 13)
        assert back.raw == b"hello, device"
        m[0].method = 12
        assert lib.lb2_unzip_run(u, buf, 64, m, 1, C.byref(out_n), res, None) == N.LB2_E_ARG
        assert lib.lb2_unzip_device_output(u, C.byref(d_out), C.byref(n)) == N.LB2_E_STATE   # the failed run left nothing
    finally:
        lib.lb2_unzip_destroy(u)
    z = C.c_void_p()
    gpu_ctx.check(lib.lb2_zip_create(gpu_ctx.h, 0, C.byref(z)))
    d = gpu_ctx.dev_alloc(1 << 17)
    try:
        gpu_ctx.check(lib.lb2_memset_d(gpu_ctx.h, d, 7, 1 << 17))
        src = (N.ZipSource * 1)()
        src[0].d_ptr, src[0].len = d, 1 << 17
        assert lib.lb2_zip_submit_device(z, None, 1, 0) == N.LB2_E_ARG
        assert lib.lb2_zip_submit_device(z, src, 0, 0) == N.LB2_E_ARG
        assert lib.lb2_zip_submit_device(z, src, 1, 4) == N.LB2_E_ARG
        assert lib.lb2_zip_submit_device(z, src, 1, N.ZIP_CONTINUES) == N.LB2_E_STATE       # no file is open
        src[0].d_ptr = None
        assert lib.lb2_zip_submit_device(z, src, 1, 0) == N.LB2_E_ARG                       # bytes without a source
        src[0].d_ptr = d
        gpu_ctx.check(lib.lb2_zip_submit_device(z, src, 1, N.ZIP_MORE))
        assert lib.lb2_zip_submit_device(z, src, 1, 0) == N.LB2_E_STATE                     # the open file not continued
        gpu_ctx.check(lib.lb2_zip_submit_device(z, src, 1, N.ZIP_CONTINUES))
        assert lib.lb2_zip_submit_device(z, src, 1, 0) == N.LB2_E_STATE                     # two pieces in flight
        a, _ = _collect(gpu_ctx, z, N.zip_bound(1 << 17, 1), 1)
        b, segs = _collect(gpu_ctx, z, N.zip_bound(1 << 17, 1), 1)
        assert zlib.decompressobj(-15).decompress(a + b) == b"\x07" * (1 << 18) and segs[0][2] == zlib.crc32(b"\x07" * (1 << 18))
    finally:
        gpu_ctx.dev_free(d)
        lib.lb2_zip_destroy(z)
