"""GPU checks of strip_tarball (tarball.py) and of the entry points under it (lb2_inflate_device_output,
lb2_memcpy_d2d, lb2_gzip_submit_device, lb2_tar_index in csrc/api.cu, the walk kernel in csrc/tar.cu).

Parity: extracting src and running the reference's `find -name "*.so" | xargs strip` gives the tree extracting
strip_tarball(src) gives, on gcc variants with symlinks, hard links, a directory named x.so and a non-ELF x.so, on the
golden files and on numpy + scipy, each written by tarfile "w:gz", gzip_tarball and GNU tar -czf; every TarInfo field
but a stripped member's size and checksum is the source's; gzip -t and tar -tzf accept the result; the DEFLATE body is
what GpuGzipFile writes for that tar stream, at 64 MB and 1 MB pieces and at level 9; runs are deterministic; the
index costs no miss; only the compressed source, the rewritten headers, the index and the DEFLATE bytes cross the bus;
corrupt and truncated sources raise and leave nothing; the new entry points refuse what they refuse."""
import ctypes as C
import glob
import gzip
import io
import os
import shutil
import subprocess
import tarfile
import zlib

import numpy as np
import pytest

import tar_archives as A

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LIMIT_CLASS = "c_many_sections"


def reference_line(root):
    return subprocess.run('find %s/ -name "*.so" | xargs strip' % root, shell=True, capture_output=True).returncode


def write_tgz(ctx, root, path, how):
    """root's directory as a .tar.gz written by tarfile "w:gz", gzip_tarball or GNU tar -czf"""
    from lambdipy_b200.tarball import gzip_tarball
    if how == "tarfile":
        with tarfile.open(path, "w:gz") as tar:
            tar.add(root, arcname=os.path.basename(root))
    elif how == "gpu":
        gzip_tarball([root], path, ctx=ctx)
    else:
        subprocess.run(["tar", "-czf", path, "-C", os.path.dirname(root), os.path.basename(root)], check=True)
    return path


def snapshot(root):
    out = {}
    for d, dirs, files in os.walk(root):
        for name in dirs + files:
            p = os.path.join(d, name)
            rel = os.path.relpath(p, root)
            out[rel] = ("sym", os.readlink(p)) if os.path.islink(p) else ("dir",) if os.path.isdir(p) else \
                open(p, "rb").read()
    return out


def body_of(path):
    """(gzip header, DEFLATE body, trailer) of a single-member gzip file"""
    raw = open(path, "rb").read()
    p = 10
    if raw[3] & 8:
        p = raw.index(b"\0", 10) + 1
    return raw[:p], raw[p:-8], raw[-8:]


def check(ctx, src, tmp, rc=0, piece_bytes=None, **kw):
    from lambdipy_b200 import tarball as T
    want, got, dst = os.path.join(tmp, "want"), os.path.join(tmp, "got"), os.path.join(tmp, "stripped.tar.gz")
    for d in (want, got):
        shutil.rmtree(d, ignore_errors=True)
    with tarfile.open(src, "r:gz") as t:
        t.extractall(want, filter="fully_trusted")
        src_members = t.getmembers()
    assert reference_line(want) == rc
    extra = {} if piece_bytes is None else {"piece_bytes": piece_bytes}
    st = T.strip_tarball(src, dst, ctx=ctx, **extra, **kw)
    with tarfile.open(dst, "r:gz") as t:
        t.extractall(got, filter="fully_trusted")
        dst_members = t.getmembers()
    assert snapshot(got) == snapshot(want)
    assert subprocess.run(["gzip", "-t", dst]).returncode == 0
    assert subprocess.run(["tar", "-tzf", dst], capture_output=True).returncode == 0
    assert len(src_members) == len(dst_members) == st["members"]
    for a, b in zip(src_members, dst_members):
        fa, fb = a.get_info(), b.get_info()
        if a.size != b.size:
            for k in ("size", "chksum"):
                fa.pop(k), fb.pop(k)
        assert fa == fb, a.name
    assert st["index"]["misses"] == 0
    # the DEFLATE body is GpuGzipFile's for this tar stream
    tar_stream = gzip.decompress(open(dst, "rb").read())
    assert len(tar_stream) == st["tar_bytes_out"] and len(tar_stream) % tarfile.RECORDSIZE == 0
    mtime = int.from_bytes(open(src, "rb").read()[4:8], "little")
    ref = os.path.join(tmp, "ref", os.path.basename(dst))
    os.makedirs(os.path.dirname(ref), exist_ok=True)
    with T.GpuGzipFile(ref, mtime=mtime, ctx=ctx, compresslevel=kw.get("compresslevel"), **extra) as g:
        g.write(tar_stream)
    assert open(ref, "rb").read() == open(dst, "rb").read()
    # what crossed the bus: the compressed source and the rewritten headers up; the index and the DEFLATE bytes down
    if st["fallback"] == 0:
        raw = open(src, "rb").read()
        up = 0        # each member's DEFLATE body is uploaded with the rest of the file behind it
        members = T.gzip_members(raw)
        body = next(members, None)
        while body is not None:
            up += len(raw) - body
            d = zlib.decompressobj(-15)
            d.decompress(raw[body:])
            try:
                body = members.send(len(raw) - body - len(d.unused_data))
            except StopIteration:
                body = None
        headers = st["uploaded_bytes"] - up      # the rewritten header blocks of the stripped members
        assert 512 * st["gpu"] <= headers <= 2048 * st["gpu"]
        assert st["downloaded_bytes"] == 16 * st["index"]["ranges"] + st["index"]["bytes"] + len(body_of(dst)[1]) - 2
    for d in (want, got):
        shutil.rmtree(d)
    return st, dst


def variant_tree(root, variants):
    os.makedirs(os.path.join(root, "lib", "x.so"))
    for k in sorted(variants):
        if k != LIMIT_CLASS:
            shutil.copy(variants[k], os.path.join(root, "lib", "lib%s.so.1" % k))
            os.symlink("lib%s.so.1" % k, os.path.join(root, "lib", "lib%s.so" % k))
    os.link(os.path.join(root, "lib", "libc_g.so.1"), os.path.join(root, "hard.so"))
    shutil.copy(variants["cxx_g"], os.path.join(root, "plain.so"))
    with open(os.path.join(root, "README.txt"), "wb") as f:
        f.write(b"a package built elsewhere\n" * 100)
    return root


@pytest.mark.parametrize("how", ["tarfile", "gpu", "gnu"])
def test_variants(gpu_ctx, variants, tmp_path, how):
    root = variant_tree(str(tmp_path / "pkg"), variants)
    src = write_tgz(gpu_ctx, root, str(tmp_path / "src.tar.gz"), how)
    shutil.rmtree(root)
    st, dst = check(gpu_ctx, src, str(tmp_path), rc=123)  # strip refuses the directory x.so, which is left alone
    assert st["gpu"] == st["selected"] and st["fallback"] == 0 and st["skipped"] == 1
    assert st["out_bytes"] < st["in_bytes"] and st["index"]["stop_reason"] == 1
    first = open(dst, "rb").read()
    from lambdipy_b200 import tarball as T
    T.strip_tarball(src, dst, ctx=gpu_ctx)
    assert open(dst, "rb").read() == first                                                   # deterministic
    if how == "gpu":
        check(gpu_ctx, src, str(tmp_path / "p1"), rc=123, piece_bytes=1 << 20)
        st9, dst9 = check(gpu_ctx, src, str(tmp_path / "l9"), rc=123, compresslevel=9)
        assert st9["dst_bytes"] <= st["dst_bytes"] and st9["deflate"]["n_opt_chunks"] > 0


def test_non_elf_and_fallback(gpu_ctx, variants, tmp_path):
    from lambdipy_b200 import tarball as T
    from lambdipy_b200.zipfile_gpu import StripFailed
    root = str(tmp_path / "pkg")
    A.tree(root, {"g.so": open(variants["c_g"], "rb").read(), "many.so": open(variants[LIMIT_CLASS], "rb").read(),
                  "text.so": b"this is not an ELF file\n" * 10})
    src = write_tgz(gpu_ctx, root, str(tmp_path / "s.tar.gz"), "gpu")
    shutil.rmtree(root)
    with pytest.raises(StripFailed, match="text.so"):
        T.strip_tarball(src, str(tmp_path / "no.tar.gz"), ctx=gpu_ctx)
    assert sorted(os.listdir(tmp_path)) == ["s.tar.gz"]
    st, _ = check(gpu_ctx, src, str(tmp_path), rc=123, tolerate_non_elf=True)
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    assert st["downloaded_bytes"] > os.path.getsize(variants[LIMIT_CLASS])    # the fallback member was fetched


def test_golden_files(gpu_ctx, tmp_path):
    from lambdipy_b200 import tarball as T
    ins = sorted(glob.glob(os.path.join(GOLDEN, "*.in.bin")))
    root = str(tmp_path / "golden")
    A.tree(root, {os.path.basename(p)[:-7] + ".so": open(p, "rb").read() for p in ins})
    for how in ("tarfile", "gnu"):
        src = write_tgz(gpu_ctx, root, str(tmp_path / ("g_%s.tar.gz" % how)), how)
        st, dst = check(gpu_ctx, src, str(tmp_path / how))
        assert st["gpu"] == len(ins)
        with tarfile.open(dst) as t:
            for p in ins:
                assert t.extractfile("golden/%s.so" % os.path.basename(p)[:-7]).read() == open(p[:-7] + ".gnu.bin", "rb").read()


def test_numpy_scipy(gpu_ctx, tmp_path):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    root = tmp_path / "prebuilt"
    for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
        if os.path.exists(os.path.join(SITE, d)):
            shutil.copytree(os.path.join(SITE, d), root / d, symlinks=True)
    for how in ("gpu", "gnu"):
        src = write_tgz(gpu_ctx, str(root), str(tmp_path / ("ns_%s.tar.gz" % how)), how)
        st, _ = check(gpu_ctx, src, str(tmp_path / how))
        assert st["gpu"] + st["fallback"] == st["selected"] > 50 and st["index"]["n_members"] == st["members"] > 1000
        print("numpy+scipy strip_tarball (%s):" % how, {k: st[k] for k in ("members", "selected", "gpu", "fallback",
              "in_bytes", "out_bytes", "src_bytes", "dst_bytes", "kernel_ms")}, "index ms", st["index"]["kernel_ms"])


def test_multi_member_and_errors(gpu_ctx, variants, tmp_path):
    from lambdipy_b200 import _native as N
    from lambdipy_b200 import tarball as T
    root = variant_tree(str(tmp_path / "pkg"), variants)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tar:
        tar.add(root, arcname="pkg")
    tar_stream = buf.getvalue()
    shutil.rmtree(root)
    src = str(tmp_path / "multi.tar.gz")
    with open(src, "wb") as f:
        for k in range(3):
            f.write(gzip.compress(tar_stream[k * len(tar_stream) // 3:(k + 1) * len(tar_stream) // 3], mtime=77))
    st, dst = check(gpu_ctx, src, str(tmp_path), rc=123)
    assert st["gpu"] > 10
    raw = open(src, "rb").read()
    for name, data in (("trunc.tar.gz", raw[:len(raw) // 2]), ("crc.tar.gz", raw[:-12] + bytes([raw[-12] ^ 1]) + raw[-11:]),
                       ("junk.tar.gz", gzip.compress(b"not a tar stream" * 64))):
        p = str(tmp_path / name)
        open(p, "wb").write(data)
        with pytest.raises((EOFError, gzip.BadGzipFile, tarfile.ReadError)):
            T.strip_tarball(p, str(tmp_path / "out.tar.gz"), ctx=gpu_ctx)
        assert not os.path.exists(tmp_path / "out.tar.gz")
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
    with pytest.raises(ValueError):
        T.strip_tarball(src, src, ctx=gpu_ctx)


@pytest.mark.parametrize("level", [None, 9])
def test_device_submit_equals_host_submit(gpu_ctx, level):
    from lambdipy_b200 import _native as N
    lib, rng = gpu_ctx.lib, np.random.default_rng(0x7A2)
    lens = [1, 15, 16, 17, 4097, 65536, 65537, 200_001, 3, 0, 70_000]
    datas = [bytes(rng.integers(0, 24, n, dtype=np.uint8)) for n in lens]
    pieces = [datas[:6], datas[6:]]
    arena = b"\xEE" * 3 + b"\xEE".join(datas) + b"\xEE" * 64
    d_arena = gpu_ctx.dev_alloc(len(arena))
    gpu_ctx.h2d(d_arena, arena, len(arena))
    addr, pos = [], 3
    for d in datas:
        addr.append(d_arena + pos)
        pos += len(d) + 1
    assert len({a % 16 for a in addr}) > 4
    outs, keep = [], []
    try:
        for device in (False, True):
            g = C.c_void_p()
            gpu_ctx.check(lib.lb2_gzip_create(gpu_ctx.h, N.deflate_flags(level), C.byref(g)))
            try:
                got, k0 = [], 0
                for ds in pieces:
                    if device:
                        src = (N.ZipSource * len(ds))()
                        for i, d in enumerate(ds):
                            src[i].d_ptr, src[i].len = addr[k0 + i], len(d)
                        gpu_ctx.check(lib.lb2_gzip_submit_device(g, src, len(ds)))
                    else:
                        b = b"".join(ds)
                        keep.append(b)
                        gpu_ctx.check(lib.lb2_gzip_submit(g, b, len(b)))
                    k0 += len(ds)
                for _ in pieces:
                    out, n = C.create_string_buffer(N.gzip_bound(1 << 20)), C.c_uint64()
                    gpu_ctx.check(lib.lb2_gzip_collect(g, out, len(out), C.byref(n)))
                    got.append(out.raw[:n.value])
                out, n, crc, isize = C.create_string_buffer(16), C.c_uint64(), C.c_uint32(), C.c_uint64()
                gpu_ctx.check(lib.lb2_gzip_finish(g, out, 16, C.byref(n), C.byref(crc), C.byref(isize), None))
                got.append((out.raw[:n.value], crc.value, isize.value))
                outs.append(got)
            finally:
                lib.lb2_gzip_destroy(g)
    finally:
        gpu_ctx.dev_free(d_arena)
    assert outs[0] == outs[1]
    whole = b"".join(datas)
    assert zlib.decompressobj(-15).decompress(outs[1][0] + outs[1][1] + outs[1][2][0]) == whole
    assert outs[1][2][1:] == (zlib.crc32(whole), len(whole))


def test_raw_api_errors(gpu_ctx, tmp_path):
    from lambdipy_b200 import _native as N
    lib = gpu_ctx.lib
    d, d_out, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
    gpu_ctx.check(lib.lb2_inflate_create(gpu_ctx.h, 0, C.byref(d)))
    try:
        assert lib.lb2_inflate_device_output(d, C.byref(d_out), C.byref(n)) == N.LB2_E_STATE
        assert lib.lb2_inflate_device_output(d, None, C.byref(n)) == N.LB2_E_ARG
        body = zlib.compress(b"hello, tar" * 100, 6)[2:-4]
        out_n, st = C.c_uint64(), N.InflateStats()
        gpu_ctx.check(lib.lb2_inflate_run(d, body, len(body), C.byref(out_n), C.byref(st)))
        gpu_ctx.check(lib.lb2_inflate_device_output(d, C.byref(d_out), C.byref(n)))
        assert n.value == 1000 and d_out.value % 256 == 0
        copy = gpu_ctx.dev_alloc(1000)
        try:
            assert lib.lb2_memcpy_d2d(gpu_ctx.h, None, d_out, 10) == N.LB2_E_ARG
            gpu_ctx.check(lib.lb2_memcpy_d2d(gpu_ctx.h, copy, d_out, 1000))
            back = C.create_string_buffer(1000)
            gpu_ctx.d2h(back, copy, 1000)
            assert back.raw == b"hello, tar" * 100
        finally:
            gpu_ctx.dev_free(copy)
        assert lib.lb2_inflate_run(d, b"\xff" * 64, 64, C.byref(out_n), C.byref(st)) == N.LB2_E_DATA
        assert lib.lb2_inflate_device_output(d, C.byref(d_out), C.byref(n)) == N.LB2_E_STATE
    finally:
        lib.lb2_inflate_destroy(d)
    g = C.c_void_p()
    gpu_ctx.check(lib.lb2_gzip_create(gpu_ctx.h, 0, C.byref(g)))
    buf = gpu_ctx.dev_alloc(1 << 16)
    try:
        src = (N.ZipSource * 1)()
        src[0].d_ptr, src[0].len = buf, 1 << 16
        assert lib.lb2_gzip_submit_device(g, None, 1) == N.LB2_E_ARG
        src[0].d_ptr = None
        assert lib.lb2_gzip_submit_device(g, src, 1) == N.LB2_E_ARG
        src[0].d_ptr = buf
        gpu_ctx.check(lib.lb2_gzip_submit_device(g, src, 1))
        gpu_ctx.check(lib.lb2_gzip_submit_device(g, src, 0))
        assert lib.lb2_gzip_submit_device(g, src, 1) == N.LB2_E_STATE       # two pieces in flight
    finally:
        lib.lb2_gzip_destroy(g)
        gpu_ctx.dev_free(buf)
    # the index: capacity, alignment and NULLs
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tar:
        for i in range(50):
            ti = tarfile.TarInfo("f/%02d.so" % i)
            ti.size = 1000 * i
            tar.addfile(ti, io.BytesIO(bytes(ti.size)))
    raw = buf.getvalue()
    d_tar = gpu_ctx.dev_alloc(len(raw) + 16)
    try:
        gpu_ctx.h2d(d_tar, raw, len(raw))
        nr, nb, st = C.c_uint32(), C.c_uint64(), N.TarIndexStats()
        ranges, data = (N.TarRange * 4)(), C.create_string_buffer(1024)
        assert lib.lb2_tar_index(gpu_ctx.h, d_tar, len(raw), ranges, 4, C.byref(nr), data, 1024, C.byref(nb),
                                 C.byref(st)) == N.LB2_E_CAPACITY
        assert nr.value > 4 and nb.value > 1024 and st.n_members == 50 and st.stop_reason == N.TAR_STOP_ZERO
        ranges, data = (N.TarRange * nr.value)(), C.create_string_buffer(nb.value)
        gpu_ctx.check(lib.lb2_tar_index(gpu_ctx.h, d_tar, len(raw), ranges, nr.value, C.byref(nr), data, nb.value,
                                        C.byref(nb), C.byref(st)))
        at = 0
        for r in ranges:
            assert data.raw[at:at + r.len] == raw[r.off:r.off + r.len]
            at += r.len
        t = tarfile.open(fileobj=io.BytesIO(raw))
        t.getmembers()
        assert st.stop_offset == t.offset
        assert lib.lb2_tar_index(gpu_ctx.h, d_tar + 1, 512, ranges, 1, C.byref(nr), data, 1, C.byref(nb), None) == N.LB2_E_ARG
        assert lib.lb2_tar_index(gpu_ctx.h, d_tar, 512, None, 1, C.byref(nr), data, 1, C.byref(nb), None) == N.LB2_E_ARG
        assert lib.lb2_tar_index(gpu_ctx.h, d_tar, 512, ranges, 1, None, data, 1, C.byref(nb), None) == N.LB2_E_ARG
    finally:
        gpu_ctx.dev_free(d_tar)


@pytest.mark.parametrize("name", sorted(A.crafted()) + ["gnu_sparse"])
def test_index_matches_the_walk_on_the_cpu(gpu_ctx, tmp_path, name):
    """the kernel gathers what the CPU emulator of the same walk gathers, and tarfile needs nothing else"""
    from lambdipy_b200 import tarball as T
    from test_tar_walk_emulated import TarEmu, check as cpu_check
    if name == "gnu_sparse":
        root = tmp_path / "sp"
        root.mkdir()
        with open(root / "holes.so", "wb") as f:
            f.seek(3 << 20)
            f.write(b"x" * 100)
        raw = A.gnu_tar_bytes(str(root), "posix", str(tmp_path), "--sparse")
        if raw is None:
            pytest.skip("GNU tar is not installed")
    else:
        raw = A.crafted()[name]
    emu = TarEmu()
    cpu_check(emu, raw)
    d_tar = gpu_ctx.dev_alloc(len(raw) + 16)
    try:
        gpu_ctx.h2d(d_tar, raw, len(raw))
        ranges, data, st = T.GpuTarIndex(gpu_ctx).index((d_tar, len(raw)))
    finally:
        gpu_ctx.dev_free(d_tar)
    e_ranges, e_data, (members, stop, reason) = emu.walk(raw)
    assert ranges == e_ranges and data == e_data
    assert (st["n_members"], st["stop_offset"], st["stop_reason"]) == (members, stop, reason)
