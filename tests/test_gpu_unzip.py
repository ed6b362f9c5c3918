"""GPU checks of the zip reader (lb2_unzip_* in csrc/api.cu and csrc/inflate.cu, extract_zip / testzip in
zipfile_gpu.py): the extracted tree equals ZipFile.extractall's on zip_tree output in both modes, make_archive output,
the numpy + scipy tree, 20 000 tiny files and a member of over 64 MB at the default span and at 1 KB spans; testzip
names the first bad member of corrupted archives as the stdlib does; results are deterministic; the C ABI refuses bad
tables before any launch."""
import ctypes as C
import os
import shutil
import zipfile
import zlib

import numpy as np
import pytest

from test_unzip_host import corrupt, tree
from test_zip_host import edge_tree

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))


def same_as_extractall(ctx, zip_path, tmp):
    from lambdipy_b200 import zipfile_gpu as Z
    want, got = os.path.join(tmp, "want"), os.path.join(tmp, "got")
    shutil.rmtree(want, ignore_errors=True)
    shutil.rmtree(got, ignore_errors=True)
    with zipfile.ZipFile(zip_path) as zf:
        zf.extractall(want)
    st = Z.extract_zip(zip_path, got, ctx=ctx)
    assert tree(got) == tree(want)
    assert Z.testzip(zip_path, ctx=ctx) is None
    shutil.rmtree(want)
    shutil.rmtree(got)
    return st


def test_zip_tree_both_modes_and_make_archive(gpu_ctx, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    root = edge_tree(str(tmp_path / "tree"))
    (tmp_path / "tree" / "pkg" / "big.bin").write_bytes(np.random.default_rng(3).integers(0, 40, 3 << 20, dtype=np.uint8).tobytes())
    for level in (None, 9):
        out = str(tmp_path / ("gpu%s.zip" % level))
        Z.zip_tree(root, out, ctx=gpu_ctx, compresslevel=level)
        st = same_as_extractall(gpu_ctx, out, str(tmp_path))
        assert st["gpu_members"] == st["files"] > 0 and st["stdlib_members"] == 0
        assert st["n_large"] > 0 and st["n_small"] > 0, st
    ref = shutil.make_archive(str(tmp_path / "ref"), "zip", root)
    same_as_extractall(gpu_ctx, ref, str(tmp_path))


def test_stored_members(gpu_ctx, tmp_path):
    path = str(tmp_path / "s.zip")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as zf:
        for i in range(50):
            zf.writestr("s/%d.bin" % i, os.urandom(i * 997))
        zf.writestr("s/big.bin", os.urandom(5 << 20))
    st = same_as_extractall(gpu_ctx, path, str(tmp_path))
    assert st["n_stored"] == 51


def test_numpy_scipy(gpu_ctx, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    root = tmp_path / "bundle"
    for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
        if os.path.exists(os.path.join(SITE, d)):
            shutil.copytree(os.path.join(SITE, d), root / d, symlinks=True)
    out = str(tmp_path / "ns.zip")
    Z.zip_tree(str(root), out, ctx=gpu_ctx)
    st = same_as_extractall(gpu_ctx, out, str(tmp_path))
    print("numpy+scipy unzip:", {k: st[k] for k in ("members", "gpu_members", "n_small", "n_large", "n_spans", "kernel_ms")})


def test_20000_tiny_files(gpu_ctx, tmp_path):
    path = str(tmp_path / "tiny.zip")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for d in range(20):
            for i in range(1000):
                zf.writestr("d%02d/m%04d.py" % (d, i), b"x = %d\n" % (i * d) * (i % 7))
    st = same_as_extractall(gpu_ctx, path, str(tmp_path))
    assert st["gpu_members"] == 20_000


@pytest.mark.parametrize("span_kb", [None, 1])
def test_member_over_64mb(gpu_ctx, tmp_path, monkeypatch, span_kb):
    from lambdipy_b200 import zipfile_gpu as Z
    if span_kb is not None:
        monkeypatch.setenv("LB2_INFLATE_SPAN_KB", str(span_kb))
    data = np.random.default_rng(9).integers(0, 16, 65 << 20, dtype=np.uint8).tobytes()  # 4 bits per byte
    path = str(tmp_path / "big.zip")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED, compresslevel=1) as zf:
        zf.writestr("a.txt", b"before " * 1000)
        zf.writestr("big.bin", data)
        zf.writestr("z.txt", b"after " * 1000)
    st = same_as_extractall(gpu_ctx, path, str(tmp_path))
    assert st["n_large"] >= 1 and st["n_spans"] > 1, st


def test_corruption_testzip_and_crc(gpu_ctx, tmp_path):
    from lambdipy_b200 import zipfile_gpu as Z
    good = tmp_path / "good.zip"
    with zipfile.ZipFile(good, "w", zipfile.ZIP_DEFLATED) as zf:
        for i in range(6):
            zf.writestr("m/%d.txt" % i, (b"member %d " % i) * (400 + 30000 * (i == 3)))
    for what in ("crc", "size", "body"):
        bad = corrupt(good, tmp_path / ("bad_%s.zip" % what), "m/3.txt", what)
        try:
            with zipfile.ZipFile(bad) as zf:
                want = zf.testzip()
        except (zlib.error, EOFError):
            want = "m/3.txt"  # the stdlib raises; testzip names the member
        assert Z.testzip(str(bad), ctx=gpu_ctx) == want == "m/3.txt", what
    with pytest.raises(zipfile.BadZipFile, match=r"Bad CRC-32 for file 'm/3.txt'"):
        Z.extract_zip(str(tmp_path / "bad_crc.zip"), str(tmp_path / "x"), ctx=gpu_ctx)
    with pytest.raises(Z.BadZipMember, match="m/3.txt"):
        Z.extract_zip(str(tmp_path / "bad_body.zip"), str(tmp_path / "y"), ctx=gpu_ctx)


def test_bad_member_leaves_neighbours_alone_and_deterministic(gpu_ctx):
    from lambdipy_b200 import zipfile_gpu as Z
    rng = np.random.default_rng(4)
    datas = [bytes(rng.integers(0, 30, n, dtype=np.uint8)) for n in (1000, 300_000, 50, 2_000_000, 0)]
    bodies = [zlib.compress(d, 6)[2:-4] for d in datas]
    bad = bytearray(bodies[1])
    bad[len(bad) // 2] ^= 0xFF
    bodies.insert(2, bytes(bad))
    datas.insert(2, datas[1])
    buf, members = b"", []
    for d, b in zip(datas, bodies):
        members.append((len(buf), len(b), len(d), zlib.crc32(d), 8))
        buf += b + b"\xAA" * 13
    members.append((0, 0, 0, 0, 0))                          # empty STORED
    members.append((5, 10, 9, 0, 0))                         # STORED of the wrong size
    with Z.GpuUnzipDecoder(gpu_ctx) as dec:
        runs = []
        for _ in range(2):
            view = dec.buffer(len(buf))
            view[:] = buf
            runs.append([(s, bytes(d)) for s, d in dec.run(len(buf), members)])
    assert runs[0] == runs[1]
    st = [s for s, _ in runs[0]]
    assert st[2] != Z.UNZIP_OK and st[6] == Z.UNZIP_OK and st[7] == Z.UNZIP_WRONG_SIZE
    for i in (0, 1, 3, 4, 5):
        assert st[i] == Z.UNZIP_OK and runs[0][i][1] == datas[i], i


def test_raw_api_errors(gpu_ctx):
    from lambdipy_b200 import _native as N
    lib = gpu_ctx.lib
    u = C.c_void_p()
    assert lib.lb2_unzip_create(gpu_ctx.h, 1, C.byref(u)) == N.LB2_E_ARG
    assert lib.lb2_unzip_create(gpu_ctx.h, 0, C.byref(u)) == N.LB2_OK
    try:
        assert lib.lb2_unzip_read(u, None, 0) == N.LB2_E_STATE
        buf = (C.c_uint8 * 64)()
        out_n, res, st = C.c_uint64(), (N.UnzipResult * 1)(), N.UnzipStats()

        def run(off, blen, size, method):
            m = (N.UnzipMember * 1)()
            m[0].body_off, m[0].body_len, m[0].size, m[0].crc32, m[0].method = off, blen, size, 0, method
            return lib.lb2_unzip_run(u, buf, 64, m, 1, C.byref(out_n), res, C.byref(st))

        assert run(0, 65, 10, 8) == N.LB2_E_ARG                # body past the buffer
        assert run(65, 0, 0, 8) == N.LB2_E_ARG                 # starts past it
        assert run(2 ** 64 - 1, 2, 0, 8) == N.LB2_E_ARG        # wraps around
        assert run(0, 4, 10, 12) == N.LB2_E_ARG                # bzip2
        assert run(0, 4, 2 ** 64 - 8, 8) == N.LB2_E_ARG        # output sizes overflow
        assert lib.lb2_unzip_run(u, buf, 64, None, 1, C.byref(out_n), res, C.byref(st)) == N.LB2_E_ARG
        assert lib.lb2_unzip_read(u, None, 0) == N.LB2_E_STATE  # nothing ran
        buf[0], buf[1] = 0x03, 0x00
        assert run(0, 2, 0, 8) == N.LB2_OK and res[0].status == 0 and out_n.value == 0
        assert st.n_small == 1 and st.n_members == 1
        assert lib.lb2_unzip_read(u, None, 0) == N.LB2_OK
    finally:
        lib.lb2_unzip_destroy(u)
